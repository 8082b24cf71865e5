"""Training-sweep throughput: a C1 grid of main.py experiments as a loop of harness.main, as sweep.run eagerly, and as
sweep.run with captured epochs.

Grid: MnistNet (D = 79,510 fp32), N = 10 users, z in {0.25, 0.5, 1, 1.5, 2, 3} x mal_prop in {0.1, 0.24} x the rules
Krum, TrimmedMean, NoDefense, and Bulyan where main.py accepts it (mal_prop 0.1 only at N = 10), x S seeds: 42 S
experiments.  Each arm trains every experiment for --epochs epochs (test every 5 epochs and at the last), setup
included; the arms alternate --reps times and the median wall time gives experiment-epochs per second.

Then, from one Sweep of the same grid, CUDA events over --steps launches each time the client-gradient kernel, the
aggregation (ALIE, rules, momentum steps) and the evaluation; the kernel's FLOP/s come from the minibatch shapes
(forward 2 m (784 100 + 100 10), backward 2 m (784 100 + 2 100 10), per client) against the 67 TFLOP/s FP32 data-sheet
figure, and the epoch shares count the evaluation once every 5 epochs.  Parity, in the same run: the sweep's weights
after epoch 0 against harness.main's epoch 0 (the same code path, stopped after one epoch) for TrimmedMean and
NoDefense, as the norm-wise relative difference of the two weight steps.  Prints one JSON object with the card's name and power limit; fails
without a GPU.

    python tools/training_sweep_throughput.py [--seeds 2] [--epochs 10] [--reps 3] [--steps 20] [--out FILE]
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
FP32_PEAK = 67e12


def harness_epoch0_weights(harness, malicious, e, batch_size, train_size, test_size):
    """harness.main's setup and its first epoch body (main.py:64-71): the global weights before and after it."""
    from attacking_federate_learning_b200.server import AggregationServer
    defense, mal_prop, num_std, n, seed = e
    f = int(mal_prop * n)
    (xtr, ytr), _, net = harness.experiment_setup(seed, train_size, test_size, "cuda")
    layout = harness.ParamLayout(net.parameters())
    w0 = layout.flatten(list(net.parameters()))
    srv = AggregationServer(n, layout.dim, mal_prop, 0.1, 0.9, device="cuda", initial_weights=w0)
    users = [harness.Client(u, u < f, xtr[u::n], ytr[u::n], batch_size, layout, "cuda") for u in range(n)]
    for u in users:
        u.step(srv.current_weights, 0.1, srv.users_grads[u.user_id])
    malicious.DriftAttack(num_std).attack_rows(srv.users_grads, f)
    srv.defend(defense, 0)
    return w0, srv.current_weights


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--seeds", type=int, default=2)
    ap.add_argument("--epochs", type=int, default=10)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--batch-size", type=int, default=83)
    ap.add_argument("--train-size", type=int, default=20000)
    ap.add_argument("--test-size", type=int, default=4000)
    ap.add_argument("--out")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("training_sweep_throughput needs a GPU")
    import __graft_entry__ as g
    g.build()
    from attacking_federate_learning_b200 import harness, malicious, sweep
    info = gpu_info()
    exps, dropped = sweep.grid(RULES, ZS, MALS, [10], list(range(args.seeds)), args.batch_size, args.train_size)
    B, E = len(exps), args.epochs
    kw = dict(batch_size=args.batch_size, train_size=args.train_size, test_size=args.test_size)
    tmp = tempfile.mkdtemp()

    def arm_harness():
        for e in exps:
            harness.main(e.mal_prop, e.num_std, e.defense, users_count=e.users_count, epochs=E, seed=e.seed,
                         out_dir=tmp, output=os.path.join(tmp, "log.txt"), **kw)

    def arm_sweep(capture):
        return lambda: sweep.run(exps, E, out_dir=tmp, capture=capture, **kw)
    arms = {"harness_loop": arm_harness, "sweep_eager": arm_sweep(False), "sweep_captured": arm_sweep(True)}
    harness.main(0.1, 1.0, "Krum", epochs=2, out_dir=tmp, output=os.path.join(tmp, "log.txt"), **kw)   # warm-up
    sweep.run(exps, 2, out_dir=tmp, capture=True, **kw)
    times = {k: [] for k in arms}
    for _ in range(args.reps):
        for k, fn in arms.items():
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            fn()
            torch.cuda.synchronize()
            times[k].append(time.perf_counter() - t0)
    rate = {k: B * E / statistics.median(v) for k, v in times.items()}

    # component times of one epoch, from CUDA events
    sw = sweep.Sweep(exps, E, capture=False, **kw)
    sw.step(0)

    def timed(fn):
        fn()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(args.steps):
            fn()
        b.record()
        torch.cuda.synchronize()
        return a.elapsed_time(b) / args.steps
    t_kernel = timed(sw.client_grads)
    t_agg = timed(sw.aggregate)
    sw.test_slot.zero_()
    t_eval = timed(lambda: (sw.test_epoch(), sw.test_slot.zero_()))
    e_now = int(sw.epoch_counter)
    flops = 0
    for e in sw.experiments:
        for u in range(e.users_count):
            lo, hi = sweep.minibatch(args.train_size, e.users_count, u, args.batch_size, e_now)
            flops += 2 * (hi - lo) * (784 * 100 + 100 * 10) + 2 * (hi - lo) * (784 * 100 + 2 * 100 * 10)
    epoch_ms = t_kernel + t_agg + t_eval / 5

    # parity of the first epoch with harness.main, continuous rules
    parity = {}
    ps = sweep.Sweep(exps, 1, capture=False, **kw)
    ps.step(0)
    for i, e in enumerate(ps.experiments):
        if e.defense in ("TrimmedMean", "NoDefense") and e.seed == 0 and e.num_std in (0.5, 2.0):
            w0, w = harness_epoch0_weights(harness, malicious, e, **kw)
            step = (w.double() - w0.double())
            rel = float(((ps.W[i].double() - w0.double()) - step).norm() / step.norm())
            parity[f"{e.defense} z={e.num_std} m={e.mal_prop}"] = rel
    out = {"gpu": info, "experiments": B, "dropped": [str(c) for c, _ in dropped], "epochs": E, "seeds": args.seeds,
           "batch_size": args.batch_size, "train_size": args.train_size, "test_size": args.test_size,
           "experiment_epochs_per_s": rate, "wall_s": times,
           "speedup_captured_vs_harness": rate["sweep_captured"] / rate["harness_loop"],
           "client_grad_ms": t_kernel, "client_grad_tflops": flops / t_kernel / 1e9,
           "client_grad_share_of_fp32_peak": flops / (t_kernel * 1e-3) / FP32_PEAK,
           "aggregation_ms": t_agg, "evaluation_ms": t_eval,
           "epoch_share": {"client_grad": t_kernel / epoch_ms, "aggregation": t_agg / epoch_ms,
                           "evaluation": t_eval / 5 / epoch_ms},
           "epoch0_weight_rel_diff_vs_harness": parity}
    s = json.dumps(out)
    print(s)
    if args.out:
        with open(args.out, "w") as fh:
            fh.write(s + "\n")
    assert all(v < 1e-3 for v in parity.values()), parity


if __name__ == "__main__":
    main()
