"""fp16 client matrices against fp32 and bf16 at the headline shapes, with parity checked in the same run.

  Krum          N = 100 x D = 11.2M (--krum-n, --krum-d), f = 24: the same data in fp32, rounded to bf16 and rounded
                to fp16.  Each arm is the headline's step (ShardedAggregator().krum, one FFI call and one stream
                synchronisation, world size 1); aggregations/s from CUDA events around --steps steps, and the Gram
                kernel's time per step from afl_profile_read("gram_pair").  The arms alternate, --reps times; medians.
                Parity: each arm's index equals Krum on the SIMT table of the same matrix (float64 sums of squared fp32
                differences), and the margin of that table's top-1 / top-2 scores is reported.
  TrimmedMean   N = 1000 x D = 10M (--tm-n, --tm-d), f = 240, in fp16 and bf16 (one matrix of normal values rounded
                to each), alternating.  Parity: on the first --tm-check columns the 16-bit result against the fp32 kernel
                on the upcast values (rtol 1e-5 + 1e-6 x the column's mean |value|; the number of columns whose bits
                differ is reported), and the full-width result on those columns against the same call on the slice.

Prints one JSON object with the card's name and power limit.

    python tools/f16_throughput.py [--steps 20] [--warmup 3] [--reps 3] [--tm-steps 3] [--out FILE]
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


def timed(fn, steps, nat, kernel):
    """(ms per step, dominant-kernel ms per step) over `steps` calls of fn."""
    torch.cuda.synchronize()
    nat.profile_enable(2)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        fn()
    e1.record()
    e1.synchronize()
    nat.profile_enable(False)
    k_ms, k_cnt = nat.profile_read(kernel)
    return e0.elapsed_time(e1) / steps, (k_ms / k_cnt if k_cnt else float("nan"))


def alternate(arms, steps, warmup, reps, nat, kernel):
    for fn in arms.values():
        for _ in range(warmup):
            fn()
    t = {k: [] for k in arms}
    for _ in range(reps):
        for k, fn in arms.items():
            t[k].append(timed(fn, steps, nat, kernel))
    out = {}
    for k, v in t.items():
        ms = statistics.median(x[0] for x in v)
        out[k] = {"ms_per_step": round(ms, 4), "aggs_per_s": round(1e3 / ms, 1),
                  f"{kernel}_ms": round(statistics.median(x[1] for x in v), 4),
                  "ms_all_reps": [round(x[0], 4) for x in v]}
    return out


def krum_leg(a, nat, dev):
    from attacking_federate_learning_b200.sharded import ShardedAggregator
    n, d, f = a.krum_n, a.krum_d, 24
    gen = torch.Generator(device="cuda").manual_seed(11)
    G32 = torch.empty((n, d), dtype=torch.float32, device="cuda")
    for r in range(n):                                 # heterogeneous client scales
        G32[r].normal_(generator=gen).mul_(float(torch.exp(0.25 * torch.randn((), generator=gen, device="cuda"))))
    mats = {"f32": G32, "bf16": G32.bfloat16(), "f16": G32.half()}
    agg = ShardedAggregator()
    arms = {k: (lambda G=G: agg.krum(G, n, f, return_index=True)) for k, G in mats.items()}
    res = alternate(arms, a.steps, a.warmup, a.reps, nat, "gram_pair")
    for k, G in mats.items():
        idx = agg.krum(G, n, f, return_index=True)
        d2 = dev.sqdist_partial(G, nat.GRAM_FORCE_SIMT)
        want = int(dev.krum_from_sqdist(d2, n, f).item())
        dist = dev.sqdist_to_dist(d2).double()
        dist.fill_diagonal_(float("inf"))
        score = torch.sort(dist, dim=1).values[:, :n - f].sum(1)
        top = torch.sort(score).values
        res[k].update(index=idx, simt_index=want, parity=idx == want,
                      simt_margin=float((top[1] - top[0]) / top[0]))
        del d2, dist
    del mats, G32
    torch.cuda.empty_cache()
    return {"n": n, "d": d, "f": f, "arms": res}


def tm_leg(a, nat, dev):
    from attacking_federate_learning_b200 import defences as D
    n, d, f = a.tm_n, a.tm_d, 240
    gen = torch.Generator(device="cuda").manual_seed(12)
    mats = {"f16": torch.empty((n, d), dtype=torch.float16, device="cuda"),
            "bf16": torch.empty((n, d), dtype=torch.bfloat16, device="cuda")}
    chunk = 1 << 20
    for c0 in range(0, d, chunk):                       # the same normal values, rounded to each format
        x = torch.empty((n, min(chunk, d - c0)), device="cuda").normal_(generator=gen)
        for G in mats.values():
            G[:, c0:c0 + x.shape[1]] = x
        del x
    arms = {k: (lambda G=G: D.trimmed_mean(G, n, f)) for k, G in mats.items()}
    res = alternate(arms, a.tm_steps, 1, a.reps, nat, "trimmed_mean")
    w = min(a.tm_check, d)
    for k, G in mats.items():
        full = D.trimmed_mean(G, n, f)[:w]
        part = D.trimmed_mean(G[:, :w], n, f)
        up = G[:, :w].float()
        ref = D.trimmed_mean(up, n, f)
        scale = up.abs().mean(0)
        ok = bool(((part - ref).abs() <= 1e-5 * ref.abs() + 1e-6 * scale).all())
        res[k].update(parity=ok and torch.equal(full.view(torch.int32), part.view(torch.int32)),
                      columns_checked=w, columns_differing_from_fp32_kernel=int((part.view(torch.int32) != ref.view(torch.int32)).sum()))
        del up, ref
    del mats
    torch.cuda.empty_cache()
    return {"n": n, "d": d, "f": f, "arms": res}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--tm-steps", type=int, default=3)
    ap.add_argument("--krum-n", type=int, default=100)
    ap.add_argument("--krum-d", type=int, default=11_200_000)
    ap.add_argument("--tm-n", type=int, default=1000)
    ap.add_argument("--tm-d", type=int, default=10_000_000)
    ap.add_argument("--tm-check", type=int, default=262_144)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("f16_throughput.py measures on a GPU; none is visible")
    from attacking_federate_learning_b200 import _device as dev, _native as nat
    info = {"gpu": gpu_info(), "device": torch.cuda.get_device_name(), "steps": a.steps, "warmup": a.warmup,
            "reps": a.reps, "krum": krum_leg(a, nat, dev), "trimmed_mean": tm_leg(a, nat, dev)}
    info["parity_all"] = all(r["parity"] for leg in ("krum", "trimmed_mean") for r in info[leg]["arms"].values())
    text = json.dumps(info)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as fh:
            fh.write(text + "\n")
    print(text)


if __name__ == "__main__":
    main()
