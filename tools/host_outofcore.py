"""Host-buffer defences on a client matrix larger than the GPU (configuration C5: N = 1000 x D = 25M fp32, 100 GB).

The matrix is an ordinary pageable NumPy array, as server.py:35 allocates it, filled column block by column block
with bench.synth_shard (seed 1234).  Krum (f = 240), TrimmedMean, NoDefense and Bulyan (f = 240) run through the
NumPy API (afl_defend_host), and every output is checked bit for bit against a slab-wise device route: the same
matrix regenerated on the device in two pieces split at a slab boundary, d2 = sum over slabs of afl_sqdist_partial
in slab order, then afl_krum_from_sqdist / afl_sqdist_to_dist -> afl_bulyan_select -> afl_trimmed_mean, and the
column rules on each piece.

If host RAM cannot hold 100 GB, D is lowered to the largest value that fits (and the output says whether the matrix
still exceeds the card's memory).  Prints one JSON object: seconds per call, the effective H2D rate of each call
(one pass over the matrix divided by the call time; Bulyan also re-streams its selected rows), a plain H2D copy of
the same bytes from pageable and from pinned memory, and the card name and power limit.

    python tools/host_outofcore.py [--n 1000] [--d 25000000] [--f 240]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def mem_available():
    """Host bytes this process may use: MemAvailable, lowered to the cgroup's memory limit when there is one."""
    avail = 0
    with open("/proc/meminfo") as fh:
        for line in fh:
            if line.startswith("MemAvailable:"):
                avail = int(line.split()[1]) * 1024
    try:
        with open("/sys/fs/cgroup/memory.max") as fh:
            v = fh.read().strip()
        if v.isdigit():
            avail = min(avail, int(v))
    except OSError:
        pass
    return avail


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power = [x.strip() for x in out.split(",")]
        return {"name": name, "power_limit": power}
    except Exception as ex:  # pragma: no cover
        return {"error": str(ex)[:200]}


def slab_width(n, d):
    w = max(32, ((96 << 20) // (n * 4) + 31) // 32 * 32)          # afl_defend_host's default (slab_cols = 0)
    return min(w, (d + 31) // 32 * 32)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=1000)
    ap.add_argument("--d", type=int, default=25_000_000)
    ap.add_argument("--f", type=int, default=240)
    ap.add_argument("--host-bytes", type=float, default=0, help="host memory the run may use (default: what is available)")
    args = ap.parse_args()
    import torch
    import bench
    from attacking_federate_learning_b200 import defences as D, _device as dev

    n, f = args.n, args.f
    card = torch.cuda.get_device_properties(0).total_memory
    d = args.d
    avail = int(args.host_bytes) or mem_available()
    note = None
    if n * d * 4 > avail - (10 << 30):                               # leave room for torch, the output vectors and staging
        d = max(1, (avail - (10 << 30)) // (n * 4)) // 32 * 32
        note = f"host RAM ({avail / 1e9:.1f} GB available) holds D = {d}, not {args.d}"
    nbytes = n * d * 4
    rec = {"n": n, "d": d, "f": f, "matrix_bytes": nbytes, "card_bytes": card, "exceeds_card": nbytes > card,
           "gpu": gpu_info(), "note": note}

    w = slab_width(n, d)
    nslab = -(-d // w)
    split = (nslab // 2) * w                                        # a slab boundary: no slab spans both pieces
    pieces = [(0, split), (split, d)]

    # ---- slab-wise device route (before the host calls, so that both never hold device memory at once)
    d2 = None
    want_tm = np.empty(d, np.float32)
    want_mean = np.empty(d, np.float32)
    for c0, c1 in pieces:
        P = bench.synth_shard(n, c0, c1, "cuda")
        for s0 in range(0, c1 - c0, w):
            part = dev.sqdist_partial(P[:, s0:min(c1 - c0, s0 + w)])
            d2 = part if d2 is None else d2 + part
        want_tm[c0:c1] = dev.trimmed_mean(P, f).cpu().numpy()
        want_mean[c0:c1] = dev.mean(P).cpu().numpy()
        del P
        torch.cuda.empty_cache()
    want_krum = int(dev.krum_from_sqdist(d2, n, f).item())
    sel = dev.bulyan_select(dev.sqdist_to_dist(d2), n, f)
    want_bulyan = np.empty(d, np.float32)
    for c0, c1 in pieces:
        P = bench.synth_shard(n, c0, c1, "cuda")
        want_bulyan[c0:c1] = dev.trimmed_mean(P, 2 * f, row_index=sel).cpu().numpy()
        del P
        torch.cuda.empty_cache()
    del d2, sel
    torch.cuda.empty_cache()

    # ---- the pageable host matrix, column block by column block
    t0 = time.perf_counter()
    G = np.empty((n, d), np.float32)
    blk = 1 << 20
    for c0 in range(0, d, blk):
        c1 = min(d, c0 + blk)
        P = bench.synth_shard(n, c0, c1, "cuda")
        for r0 in range(0, n, 100):                                  # bounded host temporaries
            G[r0:r0 + 100, c0:c1] = P[r0:r0 + 100].cpu().numpy()
        del P
    torch.cuda.empty_cache()
    rec["fill_s"] = time.perf_counter() - t0

    # ---- the four rules through the NumPy API
    calls = {}
    match = {}
    for rule in ("Krum", "TrimmedMean", "NoDefense", "Bulyan"):
        t0 = time.perf_counter()
        if rule == "Krum":
            row = D.krum(G, n, f)
            dt = time.perf_counter() - t0
            match[rule] = bool(np.shares_memory(row, G) and (row.ctypes.data - G.ctypes.data) == want_krum * G.strides[0])
        else:
            out = {"TrimmedMean": D.trimmed_mean, "NoDefense": D.no_defense, "Bulyan": D.bulyan}[rule](G, n, f)
            dt = time.perf_counter() - t0
            want = {"TrimmedMean": want_tm, "NoDefense": want_mean, "Bulyan": want_bulyan}[rule]
            match[rule] = bool(np.array_equal(out.view(np.uint32), want.view(np.uint32)))
        calls[rule] = {"s_per_call": dt, "h2d_GBps": nbytes / dt / 1e9}
    rec["calls"] = calls
    rec["bit_identical_to_device_route"] = match
    rec["krum_index"] = want_krum

    # ---- plain H2D copies of the same bytes: pageable (the matrix itself) and pinned (one buffer, repeated)
    chunk = 1 << 30
    dbuf = torch.empty(chunk // 4, dtype=torch.float32, device="cuda")
    flat = G.reshape(-1)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for e0 in range(0, flat.size, chunk // 4):
        src = torch.from_numpy(flat[e0:e0 + chunk // 4])
        dbuf[:src.numel()].copy_(src)
    torch.cuda.synchronize()
    dt = time.perf_counter() - t0
    rec["memcpy_pageable"] = {"s": dt, "GBps": nbytes / dt / 1e9}
    pinned = torch.empty(chunk // 4, dtype=torch.float32).pin_memory()
    pinned.copy_(torch.from_numpy(flat[:chunk // 4]))
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for e0 in range(0, flat.size, chunk // 4):
        m = min(chunk // 4, flat.size - e0)
        dbuf[:m].copy_(pinned[:m], non_blocking=True)
    torch.cuda.synchronize()
    dt = time.perf_counter() - t0
    rec["memcpy_pinned"] = {"s": dt, "GBps": nbytes / dt / 1e9, "note": "one 1 GiB pinned buffer copied repeatedly"}
    print(json.dumps(rec))
    return 0 if all(match.values()) else 1


if __name__ == "__main__":
    sys.exit(main())
