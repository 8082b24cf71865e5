"""A sweep over the number of users up to 1000 clients as one ragged batch (afl_defend_batched_large), against one batch
per client count and against a loop of single calls.

The grid is the reference's experiment grid at MnistNet's D = 79,510 (ld 79,520, fp32) with the larger client counts:
  n in {100, 250, 500, 1000} (--users-count, main.py:118), f = int(0.24 n) (Bulyan: the largest f with n >= 4f + 3),
  z in {0.25, 0.5, 1, 1.5, 2, 3} (--num_std), and --seeds seeds,
so B = 24 * seeds problems (B = 48: one [48, 1000, 79520] fp32 tensor, 15 GB).  Each problem's rows 0..f-1 hold its
ALIE vector (batched.alie_rows).  Per rule, three arms:
  ragged  one `batched.defend[rule](G, None, f, rows=rows)` call on the [B, 1000, D] ragged tensor;
  each    one `batched.defend[rule](G_n, n, f_n)` call per client count on that count's own [B_n, n, D] tensor;
  single  `defences.defend[rule](G_n[b], n, f)` for every problem (Krum: return_index=True, which synchronises).
Each arm runs --warmup calls, then the three arms alternate --reps times, each timed with CUDA events over --steps
calls; the median is reported as aggregations/s (B problems per call).

Agreement is checked in the same run with AFL_GRAM_SPLITS pinned for every arm.  The trimmed mean and the mean read no
distance table, so the three arms must give the same bits.  The ragged batch chooses the Gram operand format for
N = 1000, which can differ from the format a call at n = 100 picks (one-tile centred bf16x2), so there Krum's indices
and Bulyan's selections are compared, and Bulyan's outputs (a trimmed mean of the selected rows) then the same bits.
Prints one JSON object with the card's name and power limit.

    python tools/users_sweep_throughput.py [--seeds 2] [--steps 3] [--warmup 1] [--reps 3] [--out FILE]
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

D, LD, N = 79_510, 79_520, 1000
USERS = [100, 250, 500, 1000]
ZS = [0.25, 0.5, 1.0, 1.5, 2.0, 3.0]
RULES = ["Krum", "Bulyan", "TrimmedMean", "NoDefense"]


def f_of(rule, n):
    return (n - 3) // 4 if rule == "Bulyan" else int(0.24 * n)


def time_ms(fn, steps):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        fn()
    e1.record()
    e1.synchronize()
    return e0.elapsed_time(e1) / steps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--seeds", type=int, default=2)
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("users_sweep_throughput.py measures on a GPU; none is visible")
    from attacking_federate_learning_b200 import batched as bt, defences as Dm

    # problem b: (n_b, z_b, seed_b); the ragged tensor [B, N, ld] holds problem b in rows 0..n_b-1, zeros past them
    grid = [(n, z, s) for n in USERS for z in ZS for s in range(a.seeds)]
    B = len(grid)
    rows = np.array([g[0] for g in grid], np.int32)
    zs = np.array([g[1] for g in grid], np.float64)
    gen = torch.Generator(device="cuda").manual_seed(1234)
    buf = torch.zeros((B, N, LD), dtype=torch.float32, device="cuda")
    assert buf.element_size() * buf.numel() < 16e9
    for b, (n, _, _) in enumerate(grid):
        x = torch.randn((n, LD), device="cuda", generator=gen)
        buf[b, :n] = 0.1 * torch.randn((1, LD), device="cuda", generator=gen) + \
            x * torch.exp(0.25 * torch.randn((n, 1), device="cuda", generator=gen))
    G = buf[:, :, :D]
    groups = {n: np.flatnonzero(rows == n) for n in USERS}
    info = {"gpu": gpu_info(), "device": torch.cuda.get_device_name(), "D": D, "ld": LD, "N": N, "B": B,
            "seeds": a.seeds, "steps": a.steps, "warmup": a.warmup, "reps": a.reps, "rules": []}
    for rule in RULES:
        fs = np.array([f_of(rule, n) for n in rows], np.int32)
        Br = buf.clone()                                           # this rule's attacked copy (ALIE with f_b, z_b)
        Gr = Br[:, :, :D]
        bt.alie_rows(Gr, fs, zs)
        per_n = {n: Br[torch.as_tensor(idx, device="cuda"), :n].contiguous()[:, :, :D] for n, idx in groups.items()}
        kw = {"return_index": True} if rule == "Krum" else {}

        def ragged():
            return bt.defend[rule](Gr, None, fs, rows=rows, **kw)

        def each():
            return {n: bt.defend[rule](Gn, n, f_of(rule, n), **kw) for n, Gn in per_n.items()}

        def single():
            return {n: [Dm.defend[rule](Gn[b], n, f_of(rule, n), **kw) for b in range(Gn.shape[0])]
                    for n, Gn in per_n.items()}

        saved = os.environ.get("AFL_GRAM_SPLITS")
        os.environ["AFL_GRAM_SPLITS"] = "4"
        try:
            sel_r = None
            if rule == "Bulyan":
                out_r, sel_r = bt.bulyan(Gr, None, fs, return_selection=True, rows=rows)
            else:
                out_r = ragged()
            out_e, out_s = each(), single()
            agree = True
            for n, idx in groups.items():
                for j, b in enumerate(idx.tolist()):
                    if rule == "Krum":
                        agree &= int(out_r[b]) == int(out_e[n][j]) == int(out_s[n][j])
                    else:
                        agree &= torch.equal(out_r[b].view(torch.int32), out_e[n][j].view(torch.int32))
                        agree &= torch.equal(out_r[b].view(torch.int32), out_s[n][j].view(torch.int32))
                    if sel_r is not None:
                        _, s1 = Dm.bulyan(per_n[n][j], n, f_of(rule, n), return_selection=True)
                        _, s2 = bt.bulyan(per_n[n][j:j + 1], n, f_of(rule, n), return_selection=True)
                        agree &= torch.equal(sel_r[b, :s1.numel()], s1) and torch.equal(s2[0], s1)
        finally:
            if saved is None:
                os.environ.pop("AFL_GRAM_SPLITS", None)
            else:
                os.environ["AFL_GRAM_SPLITS"] = saved
        arms = {"ragged": ragged, "each": each, "single": single}
        for fn in arms.values():
            time_ms(fn, a.warmup)
        times = {k: [] for k in arms}
        for _ in range(a.reps):                                   # alternate the arms
            for k, fn in arms.items():
                times[k].append(time_ms(fn, a.steps))
        row = {"rule": rule, "agree": bool(agree)}
        for k, t in times.items():
            m = statistics.median(t)
            row[f"{k}_ms"] = round(m, 3)
            row[f"{k}_aggs_per_s"] = round(B / m * 1e3, 1)
            row[f"{k}_ms_all_reps"] = [round(x, 3) for x in t]
        info["rules"].append(row)
        print(json.dumps(row), file=sys.stderr, flush=True)
        del Br, Gr, per_n
        torch.cuda.empty_cache()
    info["agree_all"] = all(r["agree"] for r in info["rules"])
    text = json.dumps(info)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as fh:
            fh.write(text + "\n")
    print(text)


if __name__ == "__main__":
    main()
