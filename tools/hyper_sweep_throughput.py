"""Learning-rate x batch-size sweep throughput: one mixed sweep of 8-tuple experiments against one scalar sweep per
(lr, c) cell, both captured.

Grid: the C1 grid of tools/training_sweep_throughput.py (MnistNet, N = 10 users, z in {0.25, 0.5, 1, 1.5, 2, 3} x
mal_prop in {0.1, 0.24} x Krum, TrimmedMean, NoDefense, and Bulyan where main.py accepts it) x lr in {0.05, 0.1, 0.2}
x c in {32, 83, 128} x S seeds: 42 S x 9 experiments.  The mixed arm is one `sweep.run` of every 8-tuple (per-problem
m and lr on the device); the scalar arm is nine `sweep.run` calls, one per (lr, c), each over that cell's 5-tuples at
learning_rate = lr, batch_size = c, which is what a user ran before.  Each arm trains every experiment for --epochs
epochs (a test every 5 epochs and at the last), setup included; the arms alternate --reps times and the median wall
time gives experiment-epochs per second.

Parity, in the same run: AFL_GRAM_SPLITS is pinned so that the Krum and Bulyan distance tables do not follow the batch
size, and every experiment's final weights, accuracies and losses must be bit for bit the same in both arms.  Prints
one JSON object with the card's name and power limit; fails without a GPU.

    python tools/hyper_sweep_throughput.py [--seeds 2] [--epochs 10] [--reps 3] [--out FILE]
"""
import argparse
import json
import os
import statistics
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import torch  # noqa: E402

from host_outofcore import gpu_info  # noqa: E402

ZS = (0.25, 0.5, 1.0, 1.5, 2.0, 3.0)
MALS = (0.1, 0.24)
RULES = ("Krum", "TrimmedMean", "NoDefense", "Bulyan")
LRS = (0.05, 0.1, 0.2)
CS = (32, 83, 128)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--seeds", type=int, default=2)
    ap.add_argument("--epochs", type=int, default=10)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--train-size", type=int, default=20000)
    ap.add_argument("--test-size", type=int, default=4000)
    ap.add_argument("--out")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("hyper_sweep_throughput needs a GPU")
    os.environ["AFL_GRAM_SPLITS"] = "4"
    import __graft_entry__ as g
    g.build()
    from attacking_federate_learning_b200 import sweep
    info = gpu_info()
    seeds = list(range(args.seeds))
    mixed, dropped = sweep.grid(RULES, ZS, MALS, [10], seeds, train_size=args.train_size, learning_rates=list(LRS),
                                batch_sizes=list(CS))
    cells = {(lr, c): [e for e in mixed if e.learning_rate == lr and e.batch_size == c] for lr in LRS for c in CS}
    B, E = len(mixed), args.epochs
    kw = dict(train_size=args.train_size, test_size=args.test_size)
    tmp = tempfile.mkdtemp()
    out = {}

    def arm_mixed():
        out["mixed"] = sweep.run(mixed, E, out_dir=tmp, capture=True, **kw)

    def arm_scalar():
        res = {}
        for (lr, c), exps in cells.items():
            for e, r in zip(exps, sweep.run([tuple(e[:5]) for e in exps], E, learning_rate=lr, batch_size=c,
                                            out_dir=tmp, capture=True, **kw)):
                res[e] = r
        out["scalar"] = [res[e] for e in mixed]

    arms = {"mixed": arm_mixed, "scalar_per_cell": arm_scalar}
    for fn in arms.values():                                                       # warm-up: every shape once
        fn()
    times = {k: [] for k in arms}
    for _ in range(args.reps):
        for k, fn in arms.items():
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            fn()
            torch.cuda.synchronize()
            times[k].append(time.perf_counter() - t0)
    rate = {k: B * E / statistics.median(v) for k, v in times.items()}

    # parity between the arms of the last repetition: accuracies, losses and (from one more pair of Sweeps) weights
    same_results = all(a["error"] is None and b["error"] is None and a["accuracies"] == b["accuracies"] and
                       a["losses"] == b["losses"] for a, b in zip(out["mixed"], out["scalar"]))
    sw = sweep.Sweep(mixed, E, **kw)
    for e in range(E):
        sw.step(e)
    same_w = 0
    for (lr, c), exps in cells.items():
        one = sweep.Sweep([tuple(e[:5]) for e in exps], E, learning_rate=lr, batch_size=c, **kw)
        for e in range(E):
            one.step(e)
        for i, e in enumerate(exps):
            p, q = sw.order.index(mixed.index(e)), one.order.index(i)
            same_w += bool(torch.equal(sw.W[p].view(torch.int32), one.W[q].view(torch.int32)) and
                           torch.equal(sw.V[p].view(torch.int32), one.V[q].view(torch.int32)))
    res = {"gpu": info, "experiments": B, "dropped": [str(c) for c, _ in dropped], "epochs": E, "seeds": args.seeds,
           "learning_rates": LRS, "batch_sizes": CS, "train_size": args.train_size, "test_size": args.test_size,
           "experiment_epochs_per_s": rate, "wall_s": times,
           "median_wall_s": {k: statistics.median(v) for k, v in times.items()},
           "speedup_mixed_vs_scalar": rate["mixed"] / rate["scalar_per_cell"],
           "parity_results_bit_equal": same_results, "parity_weights_bit_equal": f"{same_w}/{B}"}
    s = json.dumps(res)
    print(s)
    if args.out:
        with open(args.out, "w") as fh:
            fh.write(s + "\n")
    assert same_results and same_w == B, (same_results, same_w)


if __name__ == "__main__":
    main()
