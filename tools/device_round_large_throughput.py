"""Sweep rounds of up to 1000 clients per problem with host parameters, with device parameters (DeviceRound(large=True))
and replayed from a captured CUDA graph; and the trimmed mean's device-count class launches against its host-count ones.

The grid is tools/users_sweep_throughput.py's: n in {100, 250, 500, 1000} users, f = int(0.24 n) (Bulyan: the largest
f with n >= 4f + 3), z in {0.25, 0.5, 1, 1.5, 2, 3} and --seeds seeds, B = 24 * seeds problems (B = 48: one
[48, 1000, 79520] fp32 tensor, 15 GB) of D = 79,510 fp32 as one ragged batch.  One round is ALIE on rows 0..f_b-1, the
rule, the attack-success metrics and the server's momentum step on [B, D] weights with the rule's aggregate (Krum:
the winning rows).  Three arms per rule:
  host    the module-level calls with host arrays (batched.alie_rows, batched.defend[rule](G, None, f, rows=rows),
          attack_metrics, _device.momentum_step): afl_defend_batched_large, classes grouped on the host;
  device  the same round through batched.DeviceRound(rows=True, large=True), run eagerly;
  graph   the DeviceRound round captured once with torch.cuda.graph and replayed.
A second table times the trimmed mean alone for the rules that run it (TrimmedMean, and Bulyan's second stage): the
summed CUDA-event brackets of its launches (afl_profile_read("trimmed_mean")) in afl_defend_batched_large (host-count
class launches) and in afl_defend_batched_large_dev (device-count launches, all 8 classes) on the same attacked
problems.  Every figure is the median of --reps alternating runs of --steps calls, after --warmup calls.  In the same
run, from the same inputs, one round of every arm must give the same bits (ALIE's outputs, the attacked rows, the
rule's outputs, the metrics, the weights and the velocity), and both trimmed-mean arms the same output.  Prints one
JSON object with the card's name and power limit; fails without a GPU.

    python tools/device_round_large_throughput.py [--seeds 2] [--steps 3] [--warmup 1] [--reps 3] [--out FILE]
"""
import argparse
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import numpy as np  # noqa: E402
import torch  # noqa: E402

from host_outofcore import gpu_info  # noqa: E402
from users_sweep_throughput import D, LD, N, RULES, USERS, ZS, f_of, time_ms  # noqa: E402

MOMENTUM, LR = 0.9, 0.01
PROFILED = ("gram_pair", "sqdist_simt", "krum_tail", "row_sort", "bulyan_rounds", "trimmed_mean", "mean", "alie",
            "honest_deviation")


def host_round(bt, dv, rule, G, rows, rows_d, fs, zs, w, v):
    bt.alie_rows(G, fs, zs)
    if rule == "Krum":
        idx = bt.krum(G, None, fs, return_index=True, rows=rows)
        agg = G[torch.arange(G.shape[0], device=G.device), bt.krum_gather_rows(idx, rows_d, G.shape[1])]
        met = bt.attack_metrics(G, fs, krum_index=idx, rows=rows)
        out = {"idx": idx, "agg": agg}
    elif rule == "Bulyan":
        agg, sel = bt.bulyan(G, None, fs, return_selection=True, rows=rows)
        met = bt.attack_metrics(G, fs, aggregated=agg, selection=sel, rows=rows)
        out = {"agg": agg, "sel": sel}
    else:
        agg = bt.defend[rule](G, None, fs, rows=rows)
        met = bt.attack_metrics(G, fs, aggregated=agg, rows=rows)
        out = {"agg": agg}
    dv.momentum_step(w, v, agg, MOMENTUM, LR)
    return out, met


def device_round(dv, rm, rule, w, v):
    rm.alie()
    if rule == "Krum":
        agg = rm.krum()
        idx = rm.krum_index
        met = rm.attack_metrics(krum_index=idx)
        out = {"idx": idx, "agg": agg}
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


def snapshot(res, G, fmax, w, v):
    (out, met) = res
    return {k: t.clone() for k, t in out.items()}, {k: t.clone() for k, t in met.items()}, G[:, :fmax].clone(), \
        w.clone(), v.clone()


def same(a, b):
    (oa, ma, ga, wa, va), (ob, mb, gb, wb, vb) = a, b
    ok = bits_equal(ga, gb) and bits_equal(wa, wb) and bits_equal(va, vb)
    for k in oa:
        ok &= bits_equal(oa[k], ob[k][:, :oa[k].shape[1]] if k == "sel" else ob[k])
        if k == "sel":
            ok &= bool((ob[k][:, oa[k].shape[1]:] < 0).all())
    for k in ma:
        ok &= bits_equal(ma[k], mb[k])
    return ok


def tm_ms(nat, call, steps):
    """Summed trimmed-mean brackets per call (ms) over `steps` calls."""
    for name in PROFILED:
        nat.profile_read(name)
    nat.profile_enable(1)
    try:
        for _ in range(steps):
            call()
        torch.cuda.synchronize()
        ms, launches = nat.profile_read("trimmed_mean")
    finally:
        nat.profile_enable(0)
        for name in PROFILED:
            nat.profile_read(name)
    return ms / steps, launches // steps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--seeds", type=int, default=2)
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("device_round_large_throughput.py measures on a GPU; none is visible")
    from attacking_federate_learning_b200 import _device as dv, _native as nat, batched as bt

    grid = [(n, z, s) for n in USERS for z in ZS for s in range(a.seeds)]
    B = len(grid)
    rows = np.array([g[0] for g in grid], np.int32)
    zs = np.array([g[1] for g in grid], np.float64)
    gen = torch.Generator(device="cuda").manual_seed(1234)
    buf0 = torch.zeros((B, N, LD), dtype=torch.float32, device="cuda")
    for b, (n, _, _) in enumerate(grid):
        x = torch.randn((n, LD), device="cuda", generator=gen)
        buf0[b, :n] = 0.1 * torch.randn((1, LD), device="cuda", generator=gen) + \
            x * torch.exp(0.25 * torch.randn((n, 1), device="cuda", generator=gen))
    buf = torch.empty_like(buf0)                                    # the arms' working copy (ALIE writes into it)
    G = buf[:, :, :D]
    info = {"gpu": gpu_info(), "device": torch.cuda.get_device_name(), "D": D, "ld": LD, "N": N, "B": B,
            "seeds": a.seeds, "steps": a.steps, "warmup": a.warmup, "reps": a.reps, "rounds": [], "trimmed_mean": []}
    L = nat.lib()
    rows_d = torch.as_tensor(rows, device="cuda")
    for rule in RULES:
        fs = np.array([f_of(rule, n) for n in rows], np.int32)
        fmax = int(fs.max())
        w, v = (torch.zeros((B, D), device="cuda") for _ in range(2))
        rm = bt.DeviceRound(G, rows=True, large=True, rules=(rule,))
        rmg = bt.DeviceRound(G, rows=True, large=True, rules=(rule,))
        for r in (rm, rmg):
            r.f.copy_(torch.as_tensor(fs, device="cuda"))
            r.z.copy_(torch.as_tensor(zs, device="cuda"))
            r.rows.copy_(torch.as_tensor(rows, device="cuda"))

        def restart():
            buf.copy_(buf0)
            w.zero_(), v.zero_()

        # parity: one round of each arm from the same inputs
        restart()
        ref = snapshot(host_round(bt, dv, rule, G, rows, rows_d, fs, zs, w, v), G, fmax, w, v)
        restart()
        agree = same(ref, snapshot(device_round(dv, rm, rule, w, v), G, fmax, w, v))
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):                              # eager warm-up of the graph arm's buffers
            device_round(dv, rmg, rule, w, v)
        torch.cuda.current_stream().wait_stream(side)
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            res_g = device_round(dv, rmg, rule, w, v)
        restart()
        graph.replay()
        torch.cuda.synchronize()
        agree &= same(ref, snapshot(res_g, G, fmax, w, v))
        agree &= not rm.status.any().item() and not rmg.status.any().item()

        arms = {"host": lambda: host_round(bt, dv, rule, G, rows, rows_d, fs, zs, w, v),
                "device": lambda: device_round(dv, rm, rule, w, v),
                "graph": graph.replay}
        for fn in arms.values():
            time_ms(fn, a.warmup)
        t = {k: [] for k in arms}
        for _ in range(a.reps):                                     # alternate the arms
            for k, fn in arms.items():
                t[k].append(time_ms(fn, a.steps))
        row = {"rule": rule, "agree": bool(agree)}
        for k in arms:
            m = statistics.median(t[k])
            row[f"{k}_ms"] = round(m, 3)
            row[f"{k}_aggs_per_s"] = round(B / m * 1e3, 1)
            row[f"{k}_ms_all_reps"] = [round(x, 3) for x in t[k]]
        info["rounds"].append(row)
        print(json.dumps(row), file=sys.stderr, flush=True)

        if rule in ("TrimmedMean", "Bulyan"):
            # the trimmed mean alone: host-count against device-count class launches on the same attacked problems
            restart()
            bt.alie_rows(G, fs, zs)
            ucs = rows.copy()
            fs_d, ucs_d = (torch.as_tensor(x, device="cuda") for x in (fs, ucs))
            status = torch.zeros(B, dtype=torch.int32, device="cuda")
            code = 0
            out_h, out_d = torch.empty((B, D), device="cuda"), torch.empty((B, D), device="cuda")
            sel_h = torch.empty((B, int((ucs - 2 * fs).max())), dtype=torch.int32, device="cuda")
            sel_d = torch.empty((B, N), dtype=torch.int32, device="cuda")
            ws_h = torch.empty(L.afl_batched_large_workspace_bytes(rule.encode(), B, N, D, code), dtype=torch.uint8,
                               device="cuda")
            ws_d = torch.empty(L.afl_batched_large_dev_workspace_bytes(rule.encode(), B, N, D, code),
                               dtype=torch.uint8, device="cuda")
            bulyan = rule == "Bulyan"
            stream = torch.cuda.current_stream().cuda_stream

            def host_count():
                nat.check(L.afl_defend_batched_large(rule.encode(), G.data_ptr(), B, G.stride(0), N, D, LD, code,
                                                     rows.ctypes.data, ucs.ctypes.data, fs.ctypes.data,
                                                     out_h.data_ptr(), None, sel_h.data_ptr() if bulyan else None,
                                                     ws_h.data_ptr(), ws_h.numel(), stream))

            def device_count():
                nat.check(L.afl_defend_batched_large_dev(rule.encode(), G.data_ptr(), B, G.stride(0), N, D, LD, code,
                                                         rows_d.data_ptr(), 0, ucs_d.data_ptr(), fs_d.data_ptr(),
                                                         out_d.data_ptr(), None,
                                                         sel_d.data_ptr() if bulyan else None, N, ws_d.data_ptr(),
                                                         ws_d.numel(), status.data_ptr(), stream))

            host_count(), device_count()
            torch.cuda.synchronize()
            tm_agree = bits_equal(out_h, out_d) and not status.any().item()
            if bulyan:
                tm_agree &= bits_equal(sel_h, sel_d[:, :sel_h.shape[1]])
            calls = {"host_count": host_count, "device_count": device_count}
            for fn in calls.values():
                tm_ms(nat, fn, a.warmup)
            tt = {k: [] for k in calls}
            launches = {}
            for _ in range(a.reps):
                for k, fn in calls.items():
                    ms, launches[k] = tm_ms(nat, fn, a.steps)
                    tt[k].append(ms)
            trow = {"rule": rule, "agree": bool(tm_agree)}
            for k in calls:
                trow[f"{k}_ms"] = round(statistics.median(tt[k]), 4)
                trow[f"{k}_ms_all_reps"] = [round(x, 4) for x in tt[k]]
                trow[f"{k}_launches"] = launches[k]
            trow["device_over_host"] = round(trow["device_count_ms"] / trow["host_count_ms"], 4)
            info["trimmed_mean"].append(trow)
            print(json.dumps(trow), file=sys.stderr, flush=True)
            del ws_h, ws_d
        del graph, rm, rmg
        torch.cuda.empty_cache()
    info["agree_all"] = all(r["agree"] for r in info["rounds"] + info["trimmed_mean"])
    info["device_count_within_3pct"] = all(r["device_over_host"] <= 1.03 for r in info["trimmed_mean"])
    text = json.dumps(info)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as fh:
            fh.write(text + "\n")
    print(text)


if __name__ == "__main__":
    main()
