"""One lock-step sweep round with host parameters, with device parameters, and replayed from a captured CUDA graph.

The grid is tools/sweep_report.py's C1 grid: MnistNet, N = 10 users, D = 79,510 fp32 at pitch --ld, z in {0.25, 0.5,
1.0, 1.5, 2.0, 3.0} x f in {1, 2} (Bulyan: f in {0, 1}) x S seeds, B = 12 S problems.  One round is ALIE on rows
0..f_b-1 of every problem, the rule, the attack-success metrics, and the server's momentum step on [B, D] weights with
the rule's aggregate (Krum: the winning rows).  Three arms:
  host    the module-level batched calls with host arrays of f and z (batched.alie_rows, krum / bulyan / ...,
          attack_metrics, _device.momentum_step);
  device  the same round through batched.DeviceRound, run eagerly;
  graph   the DeviceRound round captured once with torch.cuda.graph and replayed.
Each arm runs --warmup rounds, then the arms alternate --reps times, each timed with CUDA events over --steps rounds;
the median is reported in ms per round and aggregations/s (B problems per round).  In the same run, from fresh copies
of the inputs, one round of every arm must give the same bits: ALIE's statistics, the attacked matrix, the rule's
outputs, the metrics, the weights and the velocity.  Prints one JSON object with the card's name and power limit;
fails without a GPU.

    python tools/device_round_throughput.py [--seeds 2,21] [--steps 20] [--warmup 3] [--reps 3] [--ld 79520] [--out FILE]
"""
import argparse
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import torch  # noqa: E402

from host_outofcore import gpu_info  # noqa: E402
from sweep_throughput import D, N, RULES, fresh, grid, time_ms  # noqa: E402

MOMENTUM, LR = 0.9, 0.01


def host_round(bt, dv, rule, G, f, z, w, v):
    B = G.shape[0]
    bt.alie_rows(G, f, z)
    if rule == "Krum":
        idx = bt.krum(G, N, f, return_index=True)
        agg = G[torch.arange(B, device=G.device), idx.long()]
        met = bt.attack_metrics(G, f, krum_index=idx)
        out = {"idx": idx}
    elif rule == "Bulyan":
        agg, sel = bt.bulyan(G, N, f, return_selection=True)
        met = bt.attack_metrics(G, f, aggregated=agg, selection=sel)
        out = {"agg": agg, "sel": sel}
    else:
        agg = bt.defend[rule](G, N, f)
        met = bt.attack_metrics(G, f, aggregated=agg)
        out = {"agg": agg}
    dv.momentum_step(w, v, agg, MOMENTUM, LR)
    return out, met


def device_round(dv, rm, rule, w, v):
    rm.alie()
    if rule == "Krum":
        agg = rm.krum()
        met = rm.attack_metrics(krum_index=rm.krum_index)
        out = {"idx": rm.krum_index}
    elif rule == "Bulyan":
        agg, sel = rm.bulyan(return_selection=True)
        met = rm.attack_metrics(aggregated=agg, selection=sel)
        out = {"agg": agg, "sel": sel}
    else:
        agg = rm.trimmed_mean() if rule == "TrimmedMean" else rm.no_defense()
        met = rm.attack_metrics(aggregated=agg)
        out = {"agg": agg}
    dv.momentum_step(w, v, agg, MOMENTUM, LR)
    return out, met


def bits_equal(a, b):
    if a.shape != b.shape or a.dtype != b.dtype:
        return False
    iv = {4: torch.int32, 8: torch.int64, 1: torch.uint8}[a.element_size()]
    return torch.equal(a.contiguous().view(iv), b.contiguous().view(iv))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--seeds", default="2,21")
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--ld", type=int, default=79_520)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("device_round_throughput.py measures on a GPU; none is visible")
    from attacking_federate_learning_b200 import _device as dv, batched as bt
    info = {"gpu": gpu_info(), "device": torch.cuda.get_device_name(), "n": N, "d": D, "ld": a.ld,
            "steps": a.steps, "warmup": a.warmup, "reps": a.reps, "timing": []}
    for S in [int(x) for x in a.seeds.split(",")]:
        B = 12 * S
        gen = torch.Generator(device="cuda").manual_seed(1000 + S)
        buf = torch.empty((B, N, a.ld), dtype=torch.float32, device="cuda")
        buf.normal_(generator=gen)
        buf.mul_(torch.exp(0.25 * torch.randn((B, N, 1), device="cuda", generator=gen)))
        buf.add_(0.1 * torch.randn((B, 1, a.ld), device="cuda", generator=gen))    # the clients' common component
        G0 = buf[:, :, :D]
        for rule in RULES:
            _, f, z = grid(rule, S)
            Gh, Gd = fresh(G0), fresh(G0)
            wh, vh, wd, vd = (torch.zeros((B, D), device="cuda") for _ in range(4))
            rm = bt.DeviceRound(Gd, rules=(rule,))
            rm.f.copy_(torch.as_tensor(f, device="cuda"))
            rm.z.copy_(torch.as_tensor(z, device="cuda"))

            # parity: one round of each arm from the same inputs
            Gg = fresh(G0)
            wg, vg = torch.zeros((B, D), device="cuda"), torch.zeros((B, D), device="cuda")
            rmg = bt.DeviceRound(Gg, rules=(rule,))
            rmg.f.copy_(rm.f)
            rmg.z.copy_(rm.z)
            res_h = host_round(bt, dv, rule, Gh, f, z, wh, vh)
            res_d = device_round(dv, rm, rule, wd, vd)
            side = torch.cuda.Stream()
            side.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(side):                          # eager warm-up of the graph arm's buffers
                device_round(dv, rmg, rule, wg, vg)
            torch.cuda.current_stream().wait_stream(side)
            Gg.copy_(G0)
            wg.zero_(), vg.zero_()
            graph = torch.cuda.CUDAGraph()
            with torch.cuda.graph(graph):
                res_g = device_round(dv, rmg, rule, wg, vg)
            Gg.copy_(G0)
            wg.zero_(), vg.zero_()
            graph.replay()
            torch.cuda.synchronize()
            agree = bits_equal(Gh, Gd) and bits_equal(Gh, Gg)
            for x, y in ((wh, wd), (wh, wg), (vh, vd), (vh, vg)):
                agree &= bits_equal(x, y)
            for (oh, mh), (o2, m2) in ((res_h, res_d), (res_h, res_g)):
                for k in oh:
                    agree &= bits_equal(oh[k], o2[k][:, :oh[k].shape[1]] if k == "sel" else o2[k])
                for k in mh:
                    agree &= bits_equal(mh[k], m2[k])
            agree &= not rm.status.any().item() and not rmg.status.any().item()

            fns = {"host": lambda: host_round(bt, dv, rule, Gh, f, z, wh, vh),
                   "device": lambda: device_round(dv, rm, rule, wd, vd),
                   "graph": graph.replay}
            for fn in fns.values():
                time_ms(fn, a.warmup)
            t = {k: [] for k in fns}
            for _ in range(a.reps):                                  # alternate the arms
                for k, fn in fns.items():
                    t[k].append(time_ms(fn, a.steps))
            med = {k: statistics.median(v) for k, v in t.items()}
            row = {"rule": rule, "S": S, "B": B, "agree": bool(agree)}
            for k in fns:
                row[f"{k}_ms"] = round(med[k], 4)
                row[f"{k}_aggs_per_s"] = round(B / med[k] * 1e3, 1)
                row[f"{k}_ms_all_reps"] = [round(x, 4) for x in t[k]]
            info["timing"].append(row)
            print(json.dumps(row), file=sys.stderr, flush=True)
            del graph, rm, rmg, Gh, Gd, Gg
            torch.cuda.empty_cache()
    info["agree_all"] = all(r["agree"] for r in info["timing"])
    text = json.dumps(info)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as fh:
            fh.write(text + "\n")
    print(text)


if __name__ == "__main__":
    main()
