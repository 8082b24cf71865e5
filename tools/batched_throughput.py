"""Batched aggregation against a Python loop of single device calls on the same tensors.

For each rule (Krum, Bulyan, TrimmedMean, NoDefense), shape and batch size B in {1, 16, 64, 256}:
  batched  one `batched.defend[rule](G, n, f)` call on the [B, N, D] tensor (Krum: return_index=True);
  looped   `defences.defend[rule](G[b], n, f)` for b in range(B) (Krum: return_index=True, which synchronises per call,
           as the single device call does).
The two arms alternate in this process; each is timed with CUDA events over --steps calls after --warmup calls,
--reps times, and the median is reported as aggregations/s (B problems per call).  Shapes:
  10 x 79,510 with ld 79,520 (tensor-core Gram path) and unpadded (SIMT), f = 2 (Bulyan f = 1): MnistNet at the
  reference's default of 10 users (C1);  51 x 117,706, f = 12 (CIFAR10Net, Bulyan's assert holds);
  100 x 1,048,576, f = 24.  A batch whose matrix would exceed --max-gb is skipped and listed as such.
Parity is checked in the same run: batched outputs against the looped ones, bit for bit, with AFL_GRAM_SPLITS pinned
for both arms during the check (the split count is chosen per call, and a batch is one call).
Beside each time: the algorithmic bytes B*N*D*4 and the time HBM needs to stream them at the H100 SXM data-sheet
3.35 TB/s (a floor, not a measurement).  Prints one JSON object with the card's name and power limit.

    python tools/batched_throughput.py [--steps 20] [--warmup 3] [--reps 3] [--max-gb 40] [--out FILE]
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

HBM_BPS = 3.35e12
SHAPES = [  # name, n, d, ld, f (Krum / trimmed mean), f (Bulyan)
    ("C1_padded", 10, 79_510, 79_520, 2, 1),
    ("C1_unpadded", 10, 79_510, 79_510, 2, 1),
    ("cifar_51", 51, 117_706, 117_706, 12, 12),
    ("n100_d1M", 100, 1_048_576, 1_048_576, 24, 24),
]
RULES = ["Krum", "Bulyan", "TrimmedMean", "NoDefense"]


def arms(bt, D, rule, G, n, f):
    B = G.shape[0]
    if rule == "Krum":
        return (lambda: bt.krum(G, n, f, return_index=True),
                lambda: [D.krum(G[b], n, f, return_index=True) for b in range(B)])
    return (lambda: bt.defend[rule](G, n, f), lambda: [D.defend[rule](G[b], n, f) for b in range(B)])


def time_ms(fn, steps):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        fn()
    e1.record()
    e1.synchronize()
    return e0.elapsed_time(e1) / steps


def parity(bt, D, rule, G, n, f):
    """Batched outputs == looped outputs, bit for bit, with the Gram split count pinned for both."""
    saved = os.environ.get("AFL_GRAM_SPLITS")
    os.environ["AFL_GRAM_SPLITS"] = "4"
    try:
        B = G.shape[0]
        if rule == "Krum":
            return bt.krum(G, n, f, return_index=True).cpu().tolist() == [D.krum(G[b], n, f, return_index=True)
                                                                          for b in range(B)]
        if rule == "Bulyan":
            out, sel = bt.bulyan(G, n, f, return_selection=True)
            ok = True
            for b in range(B):
                o1, s1 = D.bulyan(G[b], n, f, return_selection=True)
                ok &= torch.equal(out[b].view(torch.int32), o1.view(torch.int32)) and torch.equal(sel[b], s1)
            return bool(ok)
        out = bt.defend[rule](G, n, f)
        return all(torch.equal(out[b].view(torch.int32), D.defend[rule](G[b], n, f).view(torch.int32)) for b in range(B))
    finally:
        if saved is None:
            os.environ.pop("AFL_GRAM_SPLITS", None)
        else:
            os.environ["AFL_GRAM_SPLITS"] = saved


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--batches", default="1,16,64,256")
    ap.add_argument("--max-gb", type=float, default=40.0)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("batched_throughput.py measures on a GPU; none is visible")
    from attacking_federate_learning_b200 import batched as bt, defences as D
    info = {"gpu": gpu_info(), "device": torch.cuda.get_device_name(), "steps": a.steps, "warmup": a.warmup,
            "reps": a.reps, "hbm_floor_basis": "H100 SXM data sheet 3.35 TB/s", "rows": []}
    gen = torch.Generator(device="cuda").manual_seed(1234)
    for name, n, d, ld, f, fb in SHAPES:
        for B in [int(x) for x in a.batches.split(",")]:
            nbytes = B * n * d * 4
            if B * n * ld * 4 > a.max_gb * 2**30:
                info["rows"].append({"shape": name, "B": B, "skipped": f"matrix {B * n * ld * 4 / 2**30:.1f} GiB > --max-gb"})
                continue
            buf = torch.empty((B, n, ld), dtype=torch.float32, device="cuda")
            buf.normal_(generator=gen)
            buf.mul_(torch.exp(0.25 * torch.randn((B, n, 1), device="cuda", generator=gen)))
            G = buf[:, :, :d]
            for rule in RULES:
                ff = fb if rule == "Bulyan" else f
                batched_fn, looped_fn = arms(bt, D, rule, G, n, ff)
                ok = parity(bt, D, rule, G, n, ff)
                for fn in (batched_fn, looped_fn):
                    time_ms(fn, a.warmup)
                tb, tl = [], []
                for _ in range(a.reps):                                  # alternate the arms
                    tb.append(time_ms(batched_fn, a.steps))
                    tl.append(time_ms(looped_fn, a.steps))
                mb, ml = statistics.median(tb), statistics.median(tl)
                row = {"shape": name, "n": n, "d": d, "ld": ld, "f": ff, "B": B, "rule": rule,
                       "batched_ms": round(mb, 4), "looped_ms": round(ml, 4),
                       "batched_aggs_per_s": round(B / mb * 1e3, 1), "looped_aggs_per_s": round(B / ml * 1e3, 1),
                       "speedup": round(ml / mb, 2), "bytes": nbytes, "hbm_floor_ms": round(nbytes / HBM_BPS * 1e3, 4),
                       "batched_ms_all_reps": [round(x, 4) for x in tb], "looped_ms_all_reps": [round(x, 4) for x in tl],
                       "parity": ok}
                info["rows"].append(row)
                print(json.dumps(row), file=sys.stderr, flush=True)
            del buf, G
            torch.cuda.empty_cache()
    info["parity_all"] = all(r.get("parity", True) for r in info["rows"])
    text = json.dumps(info)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as fh:
            fh.write(text + "\n")
    print(text)


if __name__ == "__main__":
    main()
