"""Host-buffer ALIE and distance tables on NumPy input (configuration C5 shapes).

ALIE: `DriftAttack(1.5).attack(users)` on f = 240 NumPy users of D = 25M fp32 (24 GB), each user its own array.
  new  the package's route: afl_alie_host streams column slabs of the users' arrays (one copy per row and slab);
  old  the route it replaced, restated here: np.stack of the f arrays, one upload of the stacked matrix, _device.alie.
Each route runs in a subprocess of its own (so peak host RSS is the route's own), alternating old/new/old/new.
Reported: seconds for the timed call (after a small warm-up call), peak RSS, and peak RSS above the users' arrays.
Both routes' statistics are compared bit for bit (a checksum of the crafted vector and of sigma).

Distances: `_krum_create_distances(G)` and `krum(G, n, f, return_index=True)` on N = 1000 x D = 22.1M (88 GB, larger
than an 80 GB card); the index is checked against `krum(G, n, f)`, which returns a view of the winning row.

If host RAM cannot hold a shape, D is lowered to the largest value that fits and the output says so.  Prints one
JSON object with the card name and power limit.

    python tools/host_surface.py [--f 240] [--d 25000000] [--dist-n 1000] [--dist-d 22100000] [--skip-alie] [--skip-dist]
"""
import argparse
import json
import os
import subprocess
import sys
import time
import zlib

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from host_outofcore import gpu_info, mem_available  # noqa: E402


class User:
    def __init__(self, grads):
        self.grads = grads


def make_users(f, d, seed=1234):
    """f separately allocated float32 vectors: one random base scaled and shifted per user (cheap to build at 24 GB)."""
    rng = np.random.default_rng(seed)
    base = rng.standard_normal(d, dtype=np.float32)
    users = []
    for i in range(f):
        g = np.empty(d, np.float32)
        np.multiply(base, np.float32(np.exp(0.25 * rng.standard_normal())), out=g)
        g += np.float32(0.01 * i)
        users.append(User(g))
    return users


def rss_peak():
    import resource
    return resource.getrusage(resource.RUSAGE_SELF).ru_maxrss * 1024


def alie_child(route, f, d):
    import torch
    from attacking_federate_learning_b200 import malicious as M, _device as dev

    def old_attack(att, users):                          # the replaced NumPy route: stack, upload, one device call
        rows = torch.from_numpy(np.ascontiguousarray(np.stack([np.asarray(u.grads, np.float32) for u in users]))).cuda()
        crafted, mu, sigma = dev.alie(rows, att.num_std, None, alias_mean=True)
        att.grads_mean, att.grads_stdev = mu.cpu().numpy(), sigma.cpu().numpy()
        for u in users:
            u.grads = att.grads_mean

    run = old_attack if route == "old" else (lambda att, users: att.attack(users))
    run(M.DriftAttack(1.5), make_users(f, 4096))         # warm-up: CUDA context, library, streams
    torch.cuda.synchronize()
    users = make_users(f, d)
    rss0 = rss_peak()
    att = M.DriftAttack(1.5)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    run(att, users)
    torch.cuda.synchronize()
    dt = time.perf_counter() - t0
    return {"route": route, "s_per_call": dt, "peak_rss_bytes": rss_peak(), "rss_after_users_bytes": rss0,
            "peak_above_users_bytes": rss_peak() - rss0, "h2d_GBps": f * d * 4 / dt / 1e9,
            "crc_crafted": zlib.crc32(att.grads_mean.view(np.uint8)), "crc_sigma": zlib.crc32(att.grads_stdev.view(np.uint8))}


def distances(n, d, f):
    import torch
    import bench
    from attacking_federate_learning_b200 import defences as D
    G = np.empty((n, d), np.float32)
    blk = 1 << 20
    for c0 in range(0, d, blk):                          # the matrix of host_outofcore.py (bench.synth_shard, seed 1234)
        c1 = min(d, c0 + blk)
        P = bench.synth_shard(n, c0, c1, "cuda")
        for r0 in range(0, n, 100):
            G[r0:r0 + 100, c0:c1] = P[r0:r0 + 100].cpu().numpy()
        del P
    torch.cuda.empty_cache()
    rec = {"n": n, "d": d, "f": f, "matrix_bytes": n * d * 4,
           "exceeds_card": n * d * 4 > torch.cuda.get_device_properties(0).total_memory}
    t0 = time.perf_counter()
    table = D._krum_create_distances(G)
    torch.cuda.synchronize()
    rec["krum_create_distances_s"] = time.perf_counter() - t0
    del table
    t0 = time.perf_counter()
    idx = D.krum(G, n, f, return_index=True)
    rec["krum_return_index_s"] = time.perf_counter() - t0
    t0 = time.perf_counter()
    row = D.krum(G, n, f)
    rec["krum_row_s"] = time.perf_counter() - t0
    rec["index"] = idx
    rec["index_matches_krum_row"] = bool(row.ctypes.data == G[idx].ctypes.data)
    for k in ("krum_create_distances_s", "krum_return_index_s", "krum_row_s"):
        rec[k.replace("_s", "_h2d_GBps")] = n * d * 4 / rec[k] / 1e9
    return rec


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--f", type=int, default=240)
    ap.add_argument("--d", type=int, default=25_000_000)
    ap.add_argument("--reps", type=int, default=2)
    ap.add_argument("--dist-n", type=int, default=1000)
    ap.add_argument("--dist-d", type=int, default=22_100_000)
    ap.add_argument("--dist-f", type=int, default=240)
    ap.add_argument("--skip-dist", action="store_true")
    ap.add_argument("--skip-alie", action="store_true")
    ap.add_argument("--child", choices=["old", "new"], help=argparse.SUPPRESS)
    args = ap.parse_args()
    if args.child:
        print(json.dumps(alie_child(args.child, args.f, args.d)))
        return 0

    avail = mem_available()
    rec = {"gpu": gpu_info(), "host_bytes_available": avail}
    f, d = args.f, args.d
    if 2 * f * d * 4 > avail - (8 << 30):                # the old route holds the users and their stacked copy
        d = max(32, (avail - (8 << 30)) // (2 * f * 4)) // 32 * 32
        rec["alie_note"] = f"host RAM holds D = {d} for the old route, not {args.d}"
    runs = []
    for rep in range(0 if args.skip_alie else args.reps):
        for route in ("old", "new"):
            out = subprocess.run([sys.executable, os.path.abspath(__file__), "--child", route, "--f", str(f), "--d", str(d)],
                                 capture_output=True, text=True)
            if out.returncode != 0:
                runs.append({"route": route, "error": out.stderr[-2000:]})
            else:
                runs.append(json.loads(out.stdout.strip().splitlines()[-1]))
    ok = [r for r in runs if "error" not in r]
    if runs:
        rec["alie"] = {"f": f, "d": d, "users_bytes": f * d * 4, "runs": runs,
                       "bit_identical": len({(r["crc_crafted"], r["crc_sigma"]) for r in ok}) == 1 and len(ok) == len(runs)}

    if not args.skip_dist:
        n, dd = args.dist_n, args.dist_d
        if n * dd * 4 > avail - (10 << 30):
            dd = max(32, (avail - (10 << 30)) // (n * 4)) // 32 * 32
            rec["dist_note"] = f"host RAM holds D = {dd}, not {args.dist_d}"
        try:
            rec["distances"] = distances(n, dd, args.dist_f)
        except Exception as ex:                           # report, do not hide, a failure at this size
            rec["distances"] = {"n": n, "d": dd, "error": f"{type(ex).__name__}: {str(ex)[:500]}"}
    print(json.dumps(rec))
    ok = rec.get("alie", {}).get("bit_identical", True) and ("distances" not in rec or rec["distances"].get("index_matches_krum_row", False))
    return 0 if ok else 1


if __name__ == "__main__":
    sys.exit(main())
