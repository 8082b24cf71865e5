"""What the attack trace costs a captured training sweep: the C1 grid (MnistNet, N = 10, z in {0.25, 0.5, 1, 1.5, 2,
3} x mal_prop in {0.1, 0.24} x Krum, TrimmedMean, NoDefense and Bulyan where main.py accepts it, x 2 seeds: 84
experiments, 10 epochs) and its CIFAR10 counterpart (Cifar10Net, fading rate 2000), each as Sweep(capture=True) with
trace off and on.

Per dataset the two arms alternate --reps times; each arm builds its Sweep, runs epoch 0 eagerly (which captures the
epoch graphs), and the timed window is the replayed epochs 1..E-1 ending in a device synchronise, so the figure is
milliseconds per captured epoch (test epochs included as the sweep runs them).  The median of the reps is reported.
Then, on one traced Sweep after its epochs, CUDA events over --steps repetitions of one epoch's attack_trace launches
(every rule's slice) give the trace's own kernel time, and the bytes it reads (every problem's honest rows, its
aggregate and, when f_b > 0, row 0, D fp32 each) give its achieved bandwidth.  In the same run the two arms' accuracies,
W and V are compared bit for bit (AFL_GRAM_SPLITS pinned, so the Krum and Bulyan distance tables split alike).  Prints
one JSON object with the card's name and power limit; fails without a GPU.

    python tools/trace_sweep_throughput.py [--seeds 2] [--epochs 10] [--reps 3] [--steps 20] [--out FILE]
"""
import argparse
import json
import os
import statistics
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
os.environ.setdefault("AFL_GRAM_SPLITS", "4")

import torch  # noqa: E402

from host_outofcore import gpu_info  # noqa: E402

ZS = (0.25, 0.5, 1.0, 1.5, 2.0, 3.0)
MALS = (0.1, 0.24)
RULES = ("Krum", "TrimmedMean", "NoDefense", "Bulyan")
DATASETS = {"MNIST": dict(fading_rate=10000), "CIFAR10": dict(dataset="CIFAR10", fading_rate=2000)}


def trace_bytes(sw):
    """Bytes one traced epoch reads: per problem its honest rows, the aggregate and row 0 when f_b > 0."""
    rows = sum((e.users_count - e.corrupted_count) + 1 + (e.corrupted_count > 0) for e in sw.experiments)
    return rows * sw.D * 4


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--seeds", type=int, default=2)
    ap.add_argument("--epochs", type=int, default=10)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--out")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("trace_sweep_throughput needs a GPU")
    import __graft_entry__ as g
    g.build()
    from attacking_federate_learning_b200 import sweep
    info = gpu_info()
    E = args.epochs
    kw = dict(batch_size=83, train_size=20000, test_size=4000)
    out = {"gpu": info, "epochs": E, "seeds": args.seeds, "reps": args.reps, "gram_splits": os.environ["AFL_GRAM_SPLITS"]}
    for name, dkw in DATASETS.items():
        exps, _ = sweep.grid(RULES, ZS, MALS, [10], list(range(args.seeds)), 83, 20000, dataset=dkw.get("dataset", "MNIST"))

        def arm(trace):
            sw = sweep.Sweep(exps, E, capture=True, trace=trace, **kw, **dkw)
            with torch.cuda.device(sw.device):
                sw.step(0)
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                for e in range(1, E):
                    sw.step(e)
                torch.cuda.synchronize()
            return sw, (time.perf_counter() - t0) * 1e3 / (E - 1)
        arm(False)                                                # warm-up: modules, allocator
        times, last = {False: [], True: []}, {}
        for _ in range(args.reps):
            for trace in (False, True):
                sw, ms = arm(trace)
                times[trace].append(ms)
                last[trace] = sw
        a, b = last[False], last[True]
        same = (all(torch.equal(getattr(a, t).view(torch.int32), getattr(b, t).view(torch.int32)) for t in ("W", "V"))
                and [r["accuracies"] for r in a.results()] == [r["accuracies"] for r in b.results()])

        slot = torch.zeros(1, dtype=torch.int32, device="cuda")
        calls = []
        for rounds in (b.rounds, b.backdoor_rounds):
            for r, (sl, rnd) in rounds.items():
                agg = rnd.krum_rows if r == "Krum" else rnd.out[r]
                names = ["agg_deviation", "malicious_deviation"] + (
                    ["krum_index"] if r == "Krum" else ["bulyan_malicious", "bulyan_selected"] if r == "Bulyan" else [])
                calls.append((rnd, agg, {k: b.trace[k][:, sl] for k in names},
                              rnd.krum_index if r == "Krum" else None, rnd.selection if r == "Bulyan" else None))

        def epoch_trace():
            for rnd, agg, tabs, idx, sel in calls:
                rnd.attack_trace(agg, slot, tabs, krum_index=idx, selection=sel)
        epoch_trace()
        ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        ev0.record()
        for _ in range(args.steps):
            epoch_trace()
        ev1.record()
        torch.cuda.synchronize()
        k_ms = ev0.elapsed_time(ev1) / args.steps
        off, on = statistics.median(times[False]), statistics.median(times[True])
        nbytes = trace_bytes(b)
        out[name] = {"experiments": b.B, "D": b.D, "ms_per_captured_epoch": {"trace_off": off, "trace_on": on},
                     "all_ms": {"trace_off": times[False], "trace_on": times[True]},
                     "overhead": on / off - 1.0, "trace_kernel_ms_per_epoch": k_ms,
                     "trace_launches_per_epoch": 3 * len(calls),     # table, deviation pass, finish
                     "trace_bytes_per_epoch": nbytes, "trace_gb_per_s": nbytes / (k_ms * 1e-3) / 1e9,
                     "trace_share_of_epoch": k_ms / off, "bit_identical_W_V_accuracies": same}
        del a, b, last, calls
        torch.cuda.empty_cache()
    s = json.dumps(out)
    print(s)
    if args.out:
        with open(args.out, "w") as fh:
            fh.write(s + "\n")
    assert all(out[n]["bit_identical_W_V_accuracies"] for n in DATASETS), "trace changed the training"


if __name__ == "__main__":
    main()
