"""CIFAR10 training-sweep throughput: a C1 grid of main.py -s CIFAR10 experiments as a loop of
harness.main(dataset='CIFAR10'), as sweep.run(dataset='CIFAR10') eagerly, and with captured epochs.

Grid: Cifar10Net (D = 117,706 fp32), N = 10 users, z in {0.25, 0.5, 1, 1.5, 2, 3} x mal_prop in {0.1, 0.24} x the rules
Krum, TrimmedMean, NoDefense, and Bulyan where main.py accepts it (mal_prop 0.1 only at N = 10), x S seeds: 42 S
experiments.  Each arm trains for --epochs epochs (test every 5 epochs and at the last), setup included; the harness
loop runs the first --harness-exps experiments only (it takes about a second per experiment-epoch), the sweeps the
whole grid.  The arms alternate --reps times and the median wall time gives experiment-epochs per second.

Then, from one Sweep of the same grid, CUDA events over --steps launches each time the client-gradient kernel, the
aggregation (ALIE, rules, momentum steps) and the evaluation.  The kernel's FLOP/s count 2 FLOP per multiply-add it
computes, per minibatch row: the forward pass on the 23x23 corner (conv1 21 21 16 27 + conv2 4 4 64 256 + fc 64 384 +
384 192 + 192 10 = 552,880) and the backward (the fc weight and input gradients 2 (192 10 + 384 192 + 64 384), conv2's
weight and input gradients at each channel's pool2 index 2 (64 256), conv1's weight gradient at each pool1 index
49 432 = 254,384); against the 67 TFLOP/s FP32 data-sheet figure.  The epoch shares count the evaluation once every 5
epochs.  Parity, in the same run: the sweep's weights
after epoch 0 against harness.main's epoch 0 (the same code path, stopped after one epoch) for TrimmedMean and
NoDefense, as the norm-wise relative difference of the two weight steps.  cuDNN's TF32 convolutions are switched off
so that harness.main computes in fp32 as the kernel does (with torch's default TF32 the two steps differ by about 1e-2).  Prints one JSON object with the card's name and power limit; fails
without a GPU.

    python tools/cifar_sweep_throughput.py [--seeds 2] [--epochs 10] [--reps 3] [--harness-exps 4] [--steps 20]
                                           [--out FILE]
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
MACS_PER_ROW = (21 * 21 * 16 * 27 + 4 * 4 * 64 * 256 + 64 * 384 + 384 * 192 + 192 * 10) + \
    (2 * (192 * 10 + 384 * 192 + 64 * 384) + 2 * 64 * 256 + 49 * 432)


def harness_epoch0_weights(harness, malicious, e, batch_size, train_size, test_size):
    """harness.main's setup and its first epoch body (main.py:64-71): the global weights before and after it."""
    from attacking_federate_learning_b200.server import AggregationServer
    defense, mal_prop, num_std, n, seed = e
    f = int(mal_prop * n)
    (xtr, ytr), _, net = harness.experiment_setup(seed, train_size, test_size, "cuda", "CIFAR10")
    layout = harness.ParamLayout(net.parameters())
    w0 = layout.flatten(list(net.parameters()))
    srv = AggregationServer(n, layout.dim, mal_prop, 0.1, 0.9, device="cuda", initial_weights=w0)
    users = [harness.Client(u, u < f, xtr[u::n], ytr[u::n], batch_size, layout, "cuda", "CIFAR10") for u in range(n)]
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
    ap.add_argument("--harness-exps", type=int, default=4)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--batch-size", type=int, default=83)
    ap.add_argument("--train-size", type=int, default=20000)
    ap.add_argument("--test-size", type=int, default=4000)
    ap.add_argument("--out")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("cifar_sweep_throughput needs a GPU")
    import __graft_entry__ as g
    g.build()
    from attacking_federate_learning_b200 import harness, malicious, sweep
    torch.backends.cudnn.allow_tf32 = False          # harness.main's convolutions in fp32, as the kernel computes them
    info = gpu_info()
    exps, dropped = sweep.grid(RULES, ZS, MALS, [10], list(range(args.seeds)), args.batch_size, args.train_size,
                               dataset="CIFAR10")
    B, E = len(exps), args.epochs
    kw = dict(batch_size=args.batch_size, train_size=args.train_size, test_size=args.test_size)
    skw = dict(kw, dataset="CIFAR10", fading_rate=2000)
    tmp = tempfile.mkdtemp()
    h_exps = exps[:args.harness_exps]

    def arm_harness():
        for e in h_exps:
            harness.main(e.mal_prop, e.num_std, e.defense, users_count=e.users_count, epochs=E, seed=e.seed,
                         out_dir=tmp, output=os.path.join(tmp, "log.txt"), fading_rate=2000, dataset="CIFAR10", **kw)

    def arm_sweep(capture):
        return lambda: sweep.run(exps, E, out_dir=tmp, capture=capture, **skw)
    arms = {"harness_loop": arm_harness, "sweep_eager": arm_sweep(False), "sweep_captured": arm_sweep(True)}
    arm_exps = {"harness_loop": len(h_exps), "sweep_eager": B, "sweep_captured": B}
    harness.main(0.1, 1.0, "Krum", epochs=2, out_dir=tmp, output=os.path.join(tmp, "log.txt"), dataset="CIFAR10",
                 **kw)                                                                        # warm-up
    sweep.run(exps, 2, out_dir=tmp, capture=True, **skw)
    times = {k: [] for k in arms}
    for _ in range(args.reps):
        for k, fn in arms.items():
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            fn()
            torch.cuda.synchronize()
            times[k].append(time.perf_counter() - t0)
    rate = {k: arm_exps[k] * E / statistics.median(v) for k, v in times.items()}

    # component times of one epoch, from CUDA events
    sw = sweep.Sweep(exps, E, capture=False, **skw)
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
            flops += 2 * (hi - lo) * MACS_PER_ROW
    epoch_ms = t_kernel + t_agg + t_eval / 5

    # parity of the first epoch with harness.main, continuous rules
    parity = {}
    ps = sweep.Sweep(exps, 1, capture=False, **skw)
    ps.step(0)
    for i, e in enumerate(ps.experiments):
        if e.defense in ("TrimmedMean", "NoDefense") and e.seed == 0 and e.num_std in (0.5, 2.0):
            w0, w = harness_epoch0_weights(harness, malicious, e, **kw)
            step = (w.double() - w0.double())
            rel = float(((ps.W[i].double() - w0.double()) - step).norm() / step.norm())
            parity[f"{e.defense} z={e.num_std} m={e.mal_prop}"] = rel
    out = {"gpu": info, "dataset": "CIFAR10", "experiments": B, "harness_loop_experiments": len(h_exps), "dropped": [str(c) for c, _ in dropped], "epochs": E, "seeds": args.seeds,
           "batch_size": args.batch_size, "train_size": args.train_size, "test_size": args.test_size,
           "experiment_epochs_per_s": rate, "wall_s": times,
           "speedup_captured_vs_harness": rate["sweep_captured"] / rate["harness_loop"],
           "client_grad_ms": t_kernel, "client_grad_gflop": flops / 1e9, "client_grad_tflops": flops / t_kernel / 1e9,
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
    # The trimmed mean's steps differ by more than 1e-3 at 20,000 training rows (measured 1.3e-3 to 2.1e-3 on an
    # H100, README), against 4e-5 for NoDefense on the same client gradients; only the mean's steps are held here.
    assert all(v < 1e-3 for k, v in parity.items() if k.startswith("NoDefense")), parity


if __name__ == "__main__":
    main()
