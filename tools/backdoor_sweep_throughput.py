"""Backdoor-sweep throughput: a C1 grid of main.py -b experiments as sweep.run with captured epochs, as sweep.run
eagerly, and (on a subset) as a loop of harness.main(..., backdoor=...).

Grid: MnistNet (D = 79,510 fp32), N = 10 users, z in {0.5, 1, 1.5} x mal_prop in {0.1, 0.24} x the rules Krum,
TrimmedMean, NoDefense, and Bulyan where main.py accepts it (mal_prop 0.1 only at N = 10) x backdoor in {pattern, 1} x
S seeds: 42 S experiments.  Each sweep arm trains every experiment
for --epochs epochs (test every 5 epochs and at the last), setup included; the harness arm runs the first
--harness-subset experiments.  The arms alternate --reps times and the median wall time gives experiment-epochs per
second.

Then, from one Sweep of the same grid after one epoch, CUDA events over --steps launches time the trainer kernel
(afl_mnist_backdoor_train) on the epoch's starting points, and the client gradients, the whole aggregation (the
crafting, the trainer, the rules, the momentum steps) and the evaluation with the backdoor test.  The trainer's FLOP
count comes from the set lengths: per problem the BEFORE test's forward pass, 2 (784 100 + 100 10) per row, and for a
problem that trains, mal_epochs passes of forward and backward, 2 (784 100 + 100 10) + 2 (784 100 + 2 100 10) per row
(a problem whose trained vector is its initial one exited after the BEFORE test and counts the test only).  Parity, in
the same run: the sweep's first weight step against harness.main's for the seed-0, z = 1, mal_prop 0.24 TrimmedMean and
NoDefense experiments (f = 2: with f = 1, sigma is 0 and the crafted row is the mean whatever the training gives), as
the norm-wise relative difference.  Prints one JSON object with the card's name and power limit; fails without a GPU.

    python tools/backdoor_sweep_throughput.py [--seeds 2] [--epochs 10] [--reps 3] [--steps 10] [--out FILE]
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

ZS = (0.5, 1.0, 1.5)
RULES = ("Krum", "Bulyan", "TrimmedMean", "NoDefense")
MALS = (0.1, 0.24)
BACKDOORS = ("pattern", 1)
FP32_PEAK = 67e12
FWD, BWD = 2 * (784 * 100 + 100 * 10), 2 * (784 * 100 + 2 * 100 * 10)


def harness_first_step(harness, e, kw):
    """harness.main's global weights before and after its first epoch (main.py:64-71)."""
    seen = []
    orig = harness.AggregationServer.defend

    def defend(self, *a, **k):
        out = orig(self, *a, **k)
        seen.append(self.current_weights.clone())
        return out
    harness.AggregationServer.defend = defend
    try:
        tmp = tempfile.mkdtemp()
        harness.main(e.mal_prop, e.num_std, e.defense, users_count=e.users_count, epochs=1, seed=e.seed, out_dir=tmp,
                     output=os.path.join(tmp, "log.txt"), backdoor=e.backdoor, **kw)
    finally:
        harness.AggregationServer.defend = orig
    return seen[0]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--seeds", type=int, default=2)
    ap.add_argument("--epochs", type=int, default=10)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--harness-subset", type=int, default=4)
    ap.add_argument("--batch-size", type=int, default=83)
    ap.add_argument("--train-size", type=int, default=20000)
    ap.add_argument("--test-size", type=int, default=4000)
    ap.add_argument("--out")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("backdoor_sweep_throughput needs a GPU")
    import __graft_entry__ as g
    g.build()
    from attacking_federate_learning_b200 import harness, sweep
    info = gpu_info()
    exps, dropped = sweep.grid(RULES, ZS, MALS, [10], list(range(args.seeds)), args.batch_size, args.train_size,
                               backdoors=BACKDOORS)
    B, E = len(exps), args.epochs
    sub = exps[:args.harness_subset]
    kw = dict(batch_size=args.batch_size, train_size=args.train_size, test_size=args.test_size)
    tmp = tempfile.mkdtemp()

    def arm_harness():
        for e in sub:
            harness.main(e.mal_prop, e.num_std, e.defense, users_count=e.users_count, epochs=E, seed=e.seed,
                         out_dir=tmp, output=os.path.join(tmp, "log.txt"), backdoor=e.backdoor, **kw)

    def arm_sweep(capture):
        return lambda: sweep.run(exps, E, out_dir=tmp, capture=capture, **kw)
    arms = {"harness_loop": (arm_harness, len(sub)), "sweep_eager": (arm_sweep(False), B),
            "sweep_captured": (arm_sweep(True), B)}
    harness.main(0.1, 1.0, "Krum", epochs=1, out_dir=tmp, output=os.path.join(tmp, "log.txt"), backdoor="pattern",
                 **kw)                                                  # warm-up
    sweep.run(exps, 2, out_dir=tmp, capture=True, **kw)
    times = {k: [] for k in arms}
    for _ in range(args.reps):
        for k, (fn, _) in arms.items():
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            fn()
            torch.cuda.synchronize()
            times[k].append(time.perf_counter() - t0)
    rate = {k: arms[k][1] * E / statistics.median(v) for k, v in times.items()}

    # component times of one epoch, from CUDA events, at the second epoch's starting points
    sw = sweep.Sweep(exps, E, capture=False, **kw)
    sw.step(0)
    sw.client_grads()
    sw.aggregate()                                                      # bd_initial and bd_mal of epoch 1

    def timed(fn):
        fn()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(args.steps):
            fn()
        b.record()
        torch.cuda.synchronize()
        return a.elapsed_time(b) / args.steps
    t_train = timed(sw.backdoor_train)
    trained = [not torch.equal(sw.bd_mal[k], sw.bd_initial[k]) for k in range(sw.n_backdoor)]
    lens = sw.bd_len.cpu().tolist()
    idx = sw.bd_index.cpu().tolist()
    flops = sum(FWD * lens[idx[k]] + (sw.mal_epochs * (FWD + BWD) * lens[idx[k]] if trained[k] else 0)
                for k in range(sw.n_backdoor))
    t_grad = timed(sw.client_grads)
    t_agg = timed(sw.aggregate)
    sw.test_slot.zero_()
    t_eval = timed(lambda: (sw.test_epoch(), sw.test_slot.zero_()))
    epoch_ms = t_grad + t_agg + t_eval / 5

    # parity of the first weight step with harness.main
    parity = {}
    ps = sweep.Sweep(exps, 1, capture=False, **kw)
    w0 = ps.W.clone()
    ps.step(0)
    for i, e in enumerate(ps.experiments):
        if e.defense in ("TrimmedMean", "NoDefense") and e.seed == 0 and e.num_std == 1.0 and e.mal_prop == 0.24:
            w = harness_first_step(harness, e, kw)
            step = w.double() - w0[i].double()
            parity[f"{e.defense} z={e.num_std} b={e.backdoor}"] = float(
                ((ps.W[i].double() - w0[i].double()) - step).norm() / step.norm())
    out = {"gpu": info, "experiments": B, "dropped": [str(c) for c, _ in dropped], "epochs": E, "seeds": args.seeds,
           "harness_subset": len(sub), "batch_size": args.batch_size, "train_size": args.train_size,
           "test_size": args.test_size, "experiment_epochs_per_s": rate, "wall_s": times,
           "speedup_captured_vs_harness": rate["sweep_captured"] / rate["harness_loop"],
           "trainer_ms": t_train, "trainer_problems_trained": sum(trained), "trainer_gflop": flops / 1e9,
           "trainer_tflops": flops / t_train / 1e9, "trainer_share_of_fp32_peak": flops / (t_train * 1e-3) / FP32_PEAK,
           "client_grad_ms": t_grad, "aggregation_ms": t_agg, "evaluation_ms": t_eval,
           "epoch_share": {"client_grad": t_grad / epoch_ms, "aggregation": t_agg / epoch_ms,
                           "trainer_in_aggregation": t_train / epoch_ms, "evaluation": t_eval / 5 / epoch_ms},
           "first_step_rel_diff_vs_harness": parity}
    s = json.dumps(out)
    print(s)
    if args.out:
        with open(args.out, "w") as fh:
            fh.write(s + "\n")
    assert all(v < 1e-3 for v in parity.values()), parity


if __name__ == "__main__":
    main()
