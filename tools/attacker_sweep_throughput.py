"""Backdoor α × malicious-epochs sweep throughput: one mixed sweep of 10-tuple experiments against one sweep per
(α, mal_epochs) cell, both captured, for MnistNet and (with --cifar10-backdoor) Cifar10Net.

Grid: main.py -d Krum Bulyan TrimmedMean NoDefense -z 1.0 -m 0.1 0.24 -b pattern 1 --seeds 0 1 (28 experiments: Bulyan
at mal_prop 0.24 needs more than 10 users) × α in {0.2, 1, 4} × mal_epochs in {1, 5}: 168 experiments, 20,000
training and 4,000 test rows.  The mixed arm is one `sweep.run` of every 10-tuple (per-problem α and epoch count in the
trainer kernel); the per-cell arm is six `sweep.run` calls, one per (α, mal_epochs), each over that cell's 6-tuples at
alpha = α, mal_epochs = k, which is what a user ran before.  Each arm trains every experiment for --epochs epochs (10
for MNIST, --cifar-epochs = 5 for CIFAR10; a test every 5 epochs and at the last), setup included; the arms alternate
--reps times and the median wall time gives experiment-epochs per second.

The trainer kernel's time per epoch, from CUDA events over --steps launches at the second epoch's starting points: the
mixed sweep's one launch, and the sum of the six per-cell launches.  Parity, in the same run: AFL_GRAM_SPLITS is pinned
so that the Krum and Bulyan distance tables do not follow the batch size, and every experiment's accuracies, backdoor
accuracies, final weights and velocities must be bit for bit the same in both arms.  Prints one JSON object with the
card's name and power limit; fails without a GPU.

    python tools/attacker_sweep_throughput.py [--epochs 10] [--cifar-epochs 5] [--reps 3] [--steps 5] [--no-cifar10]
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

RULES = ("Krum", "Bulyan", "TrimmedMean", "NoDefense")
ZS = (1.0,)
MALS = (0.1, 0.24)
BACKDOORS = ("pattern", 1)
SEEDS = (0, 1)
ALPHAS = (0.2, 1.0, 4.0)
MAL_EPOCHS = (1, 5)


def bits(t):
    return t.contiguous().view(torch.int32)


def compare(sweep, dataset, epochs, reps, steps, kw):
    """Both arms for one net: wall times, trainer times and parity."""
    mixed, dropped = sweep.grid(RULES, ZS, MALS, [10], list(SEEDS), kw["batch_size"], kw["train_size"],
                                backdoors=BACKDOORS, alphas=list(ALPHAS), mal_epochs=list(MAL_EPOCHS), **kw["grid"])
    cells = {(a, k): [e for e in mixed if e.alpha == a and e.mal_epochs == k] for a in ALPHAS for k in MAL_EPOCHS}
    B, E = len(mixed), epochs
    run_kw = {k: v for k, v in kw.items() if k != "grid"}
    tmp = tempfile.mkdtemp()
    out = {}

    def arm_mixed():
        out["mixed"] = sweep.run(mixed, E, out_dir=tmp, capture=True, **run_kw)

    def arm_cells():
        res = {}
        for (a, k), exps in cells.items():
            for e, r in zip(exps, sweep.run([tuple(e[:6]) for e in exps], E, alpha=a, mal_epochs=k, out_dir=tmp,
                                            capture=True, **run_kw)):
                res[e] = r
        out["cells"] = [res[e] for e in mixed]

    arms = {"mixed": arm_mixed, "one_run_per_cell": arm_cells}
    for fn in arms.values():                                                       # warm-up: every shape once
        fn()
    times = {k: [] for k in arms}
    for _ in range(reps):
        for k, fn in arms.items():
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            fn()
            torch.cuda.synchronize()
            times[k].append(time.perf_counter() - t0)
    rate = {k: B * E / statistics.median(v) for k, v in times.items()}
    keys = ("accuracies", "losses", "backdoor_accuracies", "backdoor_losses")
    same_results = all(a["error"] is None and b["error"] is None and all(a[k] == b[k] for k in keys)
                       for a, b in zip(out["mixed"], out["cells"]))

    def timed(fn):
        fn()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(steps):
            fn()
        b.record()
        torch.cuda.synchronize()
        return a.elapsed_time(b) / steps

    def after_one_epoch(exps, **extra):
        sw = sweep.Sweep(exps, E, capture=False, **run_kw, **extra)
        sw.step(0)
        sw.client_grads()
        sw.aggregate()                                                  # bd_initial of epoch 1
        return sw
    trainer_ms = {"mixed": timed(after_one_epoch(mixed).backdoor_train),
                  "one_run_per_cell": sum(timed(after_one_epoch([tuple(e[:6]) for e in exps], alpha=a,
                                                                mal_epochs=k).backdoor_train)
                                          for (a, k), exps in cells.items())}

    # final weights and velocities of both arms
    sw = sweep.Sweep(mixed, E, **run_kw)
    for e in range(E):
        sw.step(e)
    same_w = 0
    for (a, k), exps in cells.items():
        one = sweep.Sweep([tuple(e[:6]) for e in exps], E, alpha=a, mal_epochs=k, **run_kw)
        for e in range(E):
            one.step(e)
        for i, e in enumerate(exps):
            p, q = sw.order.index(mixed.index(e)), one.order.index(i)
            same_w += bool(torch.equal(bits(sw.W[p]), bits(one.W[q])) and torch.equal(bits(sw.V[p]), bits(one.V[q])))
    return {"dataset": dataset, "experiments": B, "dropped": len(dropped), "epochs": E,
            "experiment_epochs_per_s": rate, "wall_s": times,
            "median_wall_s": {k: statistics.median(v) for k, v in times.items()},
            "speedup_mixed_vs_cells": rate["mixed"] / rate["one_run_per_cell"],
            "trainer_ms_per_epoch": trainer_ms,
            "parity_results_bit_equal": same_results, "parity_weights_bit_equal": f"{same_w}/{B}",
            "ok": same_results and same_w == B}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--epochs", type=int, default=10)
    ap.add_argument("--cifar-epochs", type=int, default=5)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--train-size", type=int, default=20000)
    ap.add_argument("--test-size", type=int, default=4000)
    ap.add_argument("--no-cifar10", action="store_true")
    ap.add_argument("--out")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("attacker_sweep_throughput needs a GPU")
    os.environ["AFL_GRAM_SPLITS"] = "4"
    import __graft_entry__ as g
    g.build()
    from attacking_federate_learning_b200 import sweep
    torch.backends.cudnn.allow_tf32 = False
    info = gpu_info()
    kw = dict(batch_size=83, train_size=args.train_size, test_size=args.test_size)
    res = {"gpu": info, "alphas": ALPHAS, "mal_epochs": MAL_EPOCHS,
           "mnist": compare(sweep, "MNIST", args.epochs, args.reps, args.steps, dict(kw, grid={}))}
    if not args.no_cifar10:
        ckw = dict(kw, dataset="CIFAR10", fading_rate=2000, cifar10_backdoor=True,
                   grid=dict(dataset="CIFAR10", cifar10_backdoor=True))
        res["cifar10"] = compare(sweep, "CIFAR10", args.cifar_epochs, args.reps, max(1, args.steps // 2), ckw)
    s = json.dumps(res)
    print(s)
    if args.out:
        with open(args.out, "w") as fh:
            fh.write(s + "\n")
    assert all(res[k]["ok"] for k in ("mnist", "cifar10") if k in res)


if __name__ == "__main__":
    main()
