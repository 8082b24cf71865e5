"""The reference's experiment grid at C1 as one batch: per-problem counts and strengths against per-cell batches and
single calls.

The reference's results come from runs over z (--num_std, main.py:109), the malicious share (--mal-prop, main.py:106;
f = int(mal_prop * N), main.py:21) and the seed.  At C1 (MnistNet, N = 10 users, D = 79,510 fp32, pitch --ld) the
grid is z in {0.25, 0.5, 1.0, 1.5, 2.0, 3.0} x f in {1, 2} (Bulyan: f in {0, 1}, its assert N >= 4f + 3) x S seeds,
B = 12 S problems, ordered cell by cell.  One round is ALIE on rows 0..f-1 of every problem, then the rule:
  each      two per-problem calls on the whole batch: batched.alie_rows(G, f[], z[]) and batched.defend[rule](G, N, f[]);
  per_cell  one scalar batched call per (z, f) cell and stage: 24 calls on S-problem slices;
  looped    DriftAttack(z).attack_rows(G[b], f) and defences.defend[rule](G[b], N, f) for every problem (Krum with
            return_index=True, which synchronises per call as the single device call does).
Each arm is timed with CUDA events over --steps rounds after --warmup rounds, the arms alternate, --reps times, and the
median is reported as aggregations/s (B problems per round).  The rounds keep attacking the same buffer: the work per
round does not depend on the values.
Parity, in the same run, from fresh copies of the same inputs and with AFL_GRAM_SPLITS pinned for every arm (the split
count is chosen per call): the ALIE outputs, the attacked matrices and the rule's outputs (Krum's indices, Bulyan's
selections and outputs, the trimmed mean, the mean) of the three arms must be bit-identical.  Prints one JSON object
with the card's name and power limit.

    python tools/sweep_throughput.py [--seeds 2,21] [--steps 10] [--warmup 2] [--reps 3] [--ld 79520] [--out FILE]
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

N, D = 10, 79_510
ZS = [0.25, 0.5, 1.0, 1.5, 2.0, 3.0]
RULES = ["Krum", "Bulyan", "TrimmedMean", "NoDefense"]


def grid(rule, S):
    """(cells [(z, f)], per-problem f and z arrays), problems ordered cell by cell, S seeds per cell."""
    fs = (0, 1) if rule == "Bulyan" else (1, 2)
    cells = [(z, f) for z in ZS for f in fs]
    return cells, np.repeat([f for _, f in cells], S).astype(np.int32), np.repeat([z for z, _ in cells], S)


def arms(bt, D_, M, rule, G, S):
    cells, f, z = grid(rule, S)
    B = G.shape[0]
    krum = rule == "Krum"

    def rule_call(mod, Gx, fx):
        return mod.krum(Gx, N, fx, return_index=True) if krum else mod.defend[rule](Gx, N, fx)

    def each():
        a = bt.alie_rows(G, f, z)
        return a, rule_call(bt, G, f)

    def per_cell():
        outs = []
        for c, (zc, fc) in enumerate(cells):
            Gc = G[c * S:(c + 1) * S]
            outs.append((bt.alie_rows(Gc, fc, zc), rule_call(bt, Gc, fc)))
        return outs

    def looped():
        outs = []
        for b in range(B):
            crafted = M.DriftAttack(float(z[b])).attack_rows(G[b], int(f[b]))
            outs.append((crafted, rule_call(D_, G[b], int(f[b]))))
        return outs
    return {"each": each, "per_cell": per_cell, "looped": looped}


def time_ms(fn, steps):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        fn()
    e1.record()
    e1.synchronize()
    return e0.elapsed_time(e1) / steps


def same(a, b):
    if isinstance(a, int) or isinstance(b, int):             # Krum's index: a Python int from the single call
        return int(a) == int(b)
    a, b = torch.as_tensor(a).contiguous(), torch.as_tensor(b).contiguous()
    return a.shape == b.shape and a.dtype == b.dtype and torch.equal(a.view(torch.uint8), b.view(torch.uint8))


def fresh(G0):
    """A copy of G0 with its strides (the padded pitch stays, and with it the Gram path)."""
    return torch.empty_strided(G0.shape, G0.stride(), dtype=G0.dtype, device=G0.device).copy_(G0)


def parity(bt, D_, M, rule, G0, S):
    """Every arm's round on a fresh copy of G0: ALIE outputs, attacked matrix and rule outputs, bit for bit."""
    cells, f, z = grid(rule, S)
    B = G0.shape[0]
    saved = os.environ.get("AFL_GRAM_SPLITS")
    os.environ["AFL_GRAM_SPLITS"] = "4"
    try:
        res = {}
        for name in ("each", "per_cell", "looped"):
            G = fresh(G0)
            out = arms(bt, D_, M, rule, G, S)[name]()
            crafted, agg = [None] * B, [None] * B
            if name == "each":
                (c, _, _), r = out
                for b in range(B):
                    crafted[b] = c[b] if f[b] > 0 and z[b] != 0 else None
                    agg[b] = r[b]
            elif name == "per_cell":
                for ci, (alie, r) in enumerate(out):                   # alie_rows returns None for f = 0
                    for s in range(S):
                        b = ci * S + s
                        crafted[b] = alie[0][s] if f[b] > 0 and z[b] != 0 else None
                        agg[b] = r[s]
            else:
                for b, (c, r) in enumerate(out):
                    crafted[b], agg[b] = c, r
            res[name] = (G, crafted, agg)
        if rule == "Bulyan":                     # the selections too (each: padded to theta_max with -2)
            sel = bt.bulyan(res["each"][0], N, f, return_selection=True)[1].cpu()
            for b in range(B):
                theta = N - 2 * int(f[b])
                one = D_.bulyan(res["looped"][0][b], N, int(f[b]), return_selection=True)[1].cpu()
                if not (same(sel[b, :theta], one) and bool((sel[b, theta:] == -2).all())):
                    return False
        ref_G, ref_c, ref_a = res["looped"]
        for name in ("each", "per_cell"):
            G, c, a = res[name]
            if not same(G, ref_G):
                return False
            for b in range(B):
                if (c[b] is None) != (ref_c[b] is None) or (c[b] is not None and not same(c[b], ref_c[b])):
                    return False
                if not same(a[b], ref_a[b]):
                    return False
        return True
    finally:
        if saved is None:
            os.environ.pop("AFL_GRAM_SPLITS", None)
        else:
            os.environ["AFL_GRAM_SPLITS"] = saved


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--seeds", default="2,21")
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--ld", type=int, default=79_520)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("sweep_throughput.py measures on a GPU; none is visible")
    from attacking_federate_learning_b200 import batched as bt, defences as D_, malicious as M
    info = {"gpu": gpu_info(), "device": torch.cuda.get_device_name(), "n": N, "d": D, "ld": a.ld, "z": ZS,
            "steps": a.steps, "warmup": a.warmup, "reps": a.reps, "rows": []}
    for S in [int(x) for x in a.seeds.split(",")]:
        B = 12 * S
        gen = torch.Generator(device="cuda").manual_seed(1000 + S)
        buf = torch.empty((B, N, a.ld), dtype=torch.float32, device="cuda")
        buf.normal_(generator=gen)
        buf.mul_(torch.exp(0.25 * torch.randn((B, N, 1), device="cuda", generator=gen)))
        G0 = buf[:, :, :D]
        for rule in RULES:
            ok = parity(bt, D_, M, rule, G0, S)
            G = fresh(G0)
            fns = arms(bt, D_, M, rule, G, S)
            for fn in fns.values():
                time_ms(fn, a.warmup)
            t = {k: [] for k in fns}
            for _ in range(a.reps):                                  # alternate the arms
                for k, fn in fns.items():
                    t[k].append(time_ms(fn, a.steps))
            med = {k: statistics.median(v) for k, v in t.items()}
            row = {"rule": rule, "S": S, "B": B, "f": sorted(set(grid(rule, S)[1].tolist())), "parity": ok}
            for k in fns:
                row[f"{k}_ms"] = round(med[k], 4)
                row[f"{k}_aggs_per_s"] = round(B / med[k] * 1e3, 1)
                row[f"{k}_ms_all_reps"] = [round(x, 4) for x in t[k]]
            row["each_over_per_cell"] = round(med["per_cell"] / med["each"], 2)
            row["each_over_looped"] = round(med["looped"] / med["each"], 2)
            info["rows"].append(row)
            print(json.dumps(row), file=sys.stderr, flush=True)
            del G
        del buf, G0
        torch.cuda.empty_cache()
    info["parity_all"] = all(r["parity"] for r in info["rows"])
    text = json.dumps(info)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as fh:
            fh.write(text + "\n")
    print(text)


if __name__ == "__main__":
    main()
