"""Float64 d2 tables of the one-tile Gram form (49 <= N <= 112, D >= 32768) from one build of libafl_b200.so, for
comparing two builds bit for bit.

    python tools/gram_tables.py --lib PATH --out DIR     # writes DIR/<shape>.npy and DIR/krum.json
    python tools/gram_tables.py --compare DIR_A DIR_B    # np.array_equal per shape, Krum index of the headline

Shapes (seeded): those of tests/test_gpu_gram_sym.py (every instantiated row count at D = 32768 + 36, N = 100 at
D = 2^20 + 4, storage that ends at the last element with d % 4 = 1, 2, 3) and the headline matrix of bench.py
(bench.synth_shard, N = 100 x D = 11.2M, f = 24).
"""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def hetero(rng, n, d):
    return (0.1 * rng.standard_normal(d) + np.exp(0.25 * rng.standard_normal((n, 1))) * rng.standard_normal((n, d))).astype(np.float32)


def shapes():
    for n in (49, 56, 57, 64, 72, 80, 88, 96, 100, 104, 112):
        yield f"n{n}_d32804", n, 32768 + 36, 4
    yield "n100_d1048580", 100, (1 << 20) + 4, 4
    for r in (1, 2, 3):
        yield f"n100_d{32768 + 64 + r}_tight", 100, 32768 + 64 + r, 0


def matrix(torch, n, d, pad, seed):
    """Rows 0 and n // 2 equal; pad = 0: the storage ends at the last element (a flat buffer of n * d floats, viewed
    with pitch ld = d rounded up to 4 and the last row cut to d)."""
    rng = np.random.default_rng(seed)
    G = hetero(rng, n, d)
    G[n // 2] = G[0]
    if pad:
        buf = torch.zeros((n, d + pad), dtype=torch.float32, device="cuda")
        buf[:, :d] = torch.from_numpy(G).cuda()
        return buf[:, :d]
    ld = (d + 3) // 4 * 4
    flat = torch.zeros(((n - 1) * ld + d,), dtype=torch.float32, device="cuda")
    view = torch.as_strided(flat, (n, d), (ld, 1))
    view.copy_(torch.from_numpy(G).cuda())
    return view


def write(args):
    import torch
    from attacking_federate_learning_b200 import _native
    _native.LIB_PATH = os.path.abspath(args.lib)
    from attacking_federate_learning_b200 import _device as dev, defences as D
    import bench
    os.makedirs(args.out, exist_ok=True)
    for i, (name, n, d, pad) in enumerate(shapes()):
        G = matrix(torch, n, d, pad, 15000 + i)
        np.save(os.path.join(args.out, name + ".npy"), dev.sqdist_partial(G).cpu().numpy())
        del G
    G = bench.synth_shard(bench.N_CLIENTS, 0, bench.DIM, "cuda")
    np.save(os.path.join(args.out, "headline.npy"), dev.sqdist_partial(G).cpu().numpy())
    idx = D.krum(G, bench.N_CLIENTS, bench.F_BYZ, return_index=True)
    with open(os.path.join(args.out, "krum.json"), "w") as fh:
        json.dump({"headline_krum_index": int(idx), "lib": args.lib}, fh)
    print(f"{args.out}: {len(list(shapes())) + 1} tables, headline Krum index {idx}")


def compare(a, b):
    ok = True
    for f in sorted(x for x in os.listdir(a) if x.endswith(".npy")):
        ta, tb = np.load(os.path.join(a, f)), np.load(os.path.join(b, f))
        eq = np.array_equal(ta, tb)
        ok &= eq
        print(f"{f[:-4]:24s} array_equal={eq}" + ("" if eq else f" max|diff|={np.nanmax(np.abs(ta - tb)):.3e}"))
    ka, kb = (json.load(open(os.path.join(x, "krum.json")))["headline_krum_index"] for x in (a, b))
    print(f"headline Krum index: {ka} / {kb}")
    return ok and ka == kb


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lib")
    ap.add_argument("--out")
    ap.add_argument("--compare", nargs=2, metavar="DIR")
    args = ap.parse_args()
    if args.compare:
        sys.exit(0 if compare(*args.compare) else 1)
    write(args)


if __name__ == "__main__":
    main()
