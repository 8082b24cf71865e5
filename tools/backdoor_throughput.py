"""The backdoor attack over the reference's experiment grid at C1: one batched call against per-problem loops.

The grid is tools/sweep_throughput.py's: MnistNet, N = 10 users, D = 79,510 fp32 at pitch --ld, z in {0.25, 0.5, 1.0,
1.5, 2.0, 3.0} x f in {1, 2} x S seeds, B = 12 S problems (B = 24 and 252 for the default seeds), each with its own
global model w_b and learning rate 0.1.  The malicious-network training is the golden fixtures' stand-in (p * 0.9 +
0.01, one element-wise pass), so the figures are the engine's cost around the caller's training.  One round crafts
and writes the malicious rows of every problem:
  batched      batched.backdoor_rows(G, f[], z[], W, 0.1, train): one call, the training called once for all problems;
  attack_rows  BackdoorAttack(z_b, train).attack_rows(G[b], f_b, W[b], 0.1) for every problem;
  attack       BackdoorAttack(z_b, train).attack(users) on the f_b per-user row vectors of every problem, then the
               crafted vector copied into rows 0..f_b-1 (server.py:82-83).
Each arm is timed with CUDA events over --steps rounds after --warmup rounds, the arms alternate, --reps times, and the
median is reported.  The rounds keep attacking the same buffer: the work per round does not depend on the values.
Parity, in the same run, from fresh copies of the same inputs: the crafted vectors, the statistics and the attacked
matrices of the three arms must be bit-identical (the script fails otherwise).  Prints one JSON object with the card's
name and power limit.

    python tools/backdoor_throughput.py [--seeds 2,21] [--steps 10] [--warmup 2] [--reps 3] [--ld 79520] [--out FILE]
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
from sweep_throughput import D, N, ZS, time_ms  # noqa: E402

LR = 0.1


def train(p):                                    # tests/golden/make_golden_backdoor.py's stand-in for backdoor.py:108
    return p * 0.9 + 0.01


class User:
    def __init__(self, g, w):
        self.grads, self.original_params, self.learning_rate = g, w, LR


def inputs(S, ld, seed):
    """(G [B, N, D] at pitch ld, W [B, D], f [B], z [B]): problems ordered cell by cell, S seeds per cell."""
    cells = [(z, f) for z in ZS for f in (1, 2)]
    f = np.repeat([c[1] for c in cells], S).astype(np.int32)
    z = np.repeat([c[0] for c in cells], S)
    B = len(f)
    gen = torch.Generator(device="cuda").manual_seed(seed)
    buf = torch.empty((B, N, ld), device="cuda").normal_(generator=gen)
    buf *= torch.exp(0.25 * torch.randn((B, N, 1), generator=gen, device="cuda"))     # heterogeneous client scales
    W = torch.empty((B, D), device="cuda").normal_(generator=gen)
    return buf[:, :, :D], W, f, z


def arms(bt, M, G, W, f, z):
    B = G.shape[0]

    def batched():
        crafted, mu, sigma = bt.backdoor_rows(G, f, z, W, LR, lambda x, problems: train(x))
        return [(crafted[b], mu[b], sigma[b]) for b in range(B)]

    def attack_rows():
        outs = []
        for b in range(B):
            att = M.BackdoorAttack(float(z[b]), train)
            outs.append((att.attack_rows(G[b], int(f[b]), W[b], LR), att.grads_mean, att.grads_stdev))
        return outs

    def attack():
        outs = []
        for b in range(B):
            users = [User(G[b, i], W[b]) for i in range(int(f[b]))]
            att = M.BackdoorAttack(float(z[b]), train)
            att.attack(users)
            G[b, :int(f[b])] = users[0].grads                                  # server.py:82-83
            outs.append((users[0].grads, att.grads_mean, att.grads_stdev))
        return outs
    return {"batched": batched, "attack_rows": attack_rows, "attack": attack}


def same(a, b):
    a, b = a.contiguous(), b.contiguous()
    return a.shape == b.shape and torch.equal(a.view(torch.int32), b.view(torch.int32))


def leg(bt, M, S, a):
    G, W, f, z = inputs(S, a.ld, 100 + S)
    B = G.shape[0]
    # parity: one round of every arm on fresh copies of the same inputs
    results, mats = {}, {}
    for k in ("batched", "attack_rows", "attack"):
        Gk = G.clone()
        results[k] = arms(bt, M, Gk, W, f, z)[k]()
        mats[k] = Gk
    parity = all(same(mats[k], mats["batched"]) and
                 all(same(x, y) for r, q in zip(results[k], results["batched"]) for x, y in zip(r, q))
                 for k in ("attack_rows", "attack"))
    assert parity, f"B = {B}: the arms' crafted vectors, statistics or attacked matrices differ"
    fns = arms(bt, M, G, W, f, z)
    for fn in fns.values():
        for _ in range(a.warmup):
            fn()
    t = {k: [] for k in fns}
    for _ in range(a.reps):
        for k, fn in fns.items():
            t[k].append(time_ms(fn, a.steps))
    out = {}
    for k, v in t.items():
        ms = statistics.median(v)
        out[k] = {"ms_per_round": round(ms, 4), "problems_per_s": round(B * 1e3 / ms, 1),
                  "ms_all_reps": [round(x, 4) for x in v]}
    for k in ("attack_rows", "attack"):
        out[k]["batched_speedup"] = round(out[k]["ms_per_round"] / out["batched"]["ms_per_round"], 2)
    return {"B": B, "S": S, "parity": parity, "arms": out}


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
        sys.exit("backdoor_throughput.py measures on a GPU; none is visible")
    from attacking_federate_learning_b200 import batched as bt, malicious as M
    info = {"gpu": gpu_info(), "device": torch.cuda.get_device_name(), "n": N, "d": D, "ld": a.ld, "steps": a.steps,
            "warmup": a.warmup, "reps": a.reps,
            "legs": [leg(bt, M, int(S), a) for S in a.seeds.split(",")]}
    text = json.dumps(info)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as fh:
            fh.write(text + "\n")
    print(text)


if __name__ == "__main__":
    main()
