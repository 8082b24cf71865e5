"""Real-data training sweeps: the cost of data.load and of each epoch part on full-size MNIST- and CIFAR10-format
files, against the synthetic sweep at the same sizes.

The files are generated from a seed (uniform random pixels and labels) into a temporary directory: MNIST's four IDX
files (60,000 / 10,000 rows) and CIFAR10's six batch pickles (50,000 / 10,000 rows).  Per dataset: the wall time of
data.load, then the C1 grid (z in {0.25, 0.5, 1, 1.5, 2, 3} x mal_prop in {0.1, 0.24} x Krum, TrimmedMean, NoDefense
and Bulyan where main.py accepts it, N = 10) x --seeds seeds, built once with data_dir and once on the synthetic
problem at the files' sizes.  For each: the Sweep set-up time, the wall time of --epochs captured epochs (test every
5 epochs and at the last), and CUDA events over --steps replays of the captured training epoch and of the test epoch.
Prints one JSON object with the card's name and power limit; fails without a GPU.

    python tools/real_data_sweep_throughput.py [--seeds 2] [--epochs 10] [--steps 20] [--out FILE]
"""
import argparse
import json
import os
import pickle
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import numpy as np  # noqa: E402
import torch  # noqa: E402

from host_outofcore import gpu_info  # noqa: E402

ZS = (0.25, 0.5, 1.0, 1.5, 2.0, 3.0)
MALS = (0.1, 0.24)
RULES = ("Krum", "TrimmedMean", "NoDefense", "Bulyan")


def idx(a):
    return (0x800 | a.ndim).to_bytes(4, 'big') + b''.join(int(d).to_bytes(4, 'big') for d in a.shape) + a.tobytes()


def write_files(base, rng):
    mnist = os.path.join(base, 'mnist_data', 'MNIST', 'raw')
    os.makedirs(mnist)
    for pre, n in (('train', 60000), ('t10k', 10000)):
        with open(os.path.join(mnist, f'{pre}-images-idx3-ubyte'), 'wb') as f:
            f.write(idx(rng.integers(0, 256, (n, 28, 28), dtype=np.uint8)))
        with open(os.path.join(mnist, f'{pre}-labels-idx1-ubyte'), 'wb') as f:
            f.write(idx(rng.integers(0, 10, n, dtype=np.uint8)))
    cifar = os.path.join(base, 'cifar10_data', 'cifar-10-batches-py')
    os.makedirs(cifar)
    for name in [f'data_batch_{i}' for i in range(1, 6)] + ['test_batch']:
        with open(os.path.join(cifar, name), 'wb') as f:
            pickle.dump({'data': rng.integers(0, 256, (10000, 3072), dtype=np.uint8),
                         'labels': [int(v) for v in rng.integers(0, 10, 10000)]}, f, protocol=4)
    return {'MNIST': os.path.join(base, 'mnist_data'), 'CIFAR10': os.path.join(base, 'cifar10_data')}


def events_ms(fn, steps):
    fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(steps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / steps


def measure(sweep, exps, dataset, epochs, steps, **kw):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    sw = sweep.Sweep(exps, epochs, batch_size=83, test_step=5, capture=True, dataset=dataset,
                     fading_rate=sweep.FADING_RATE[dataset], **kw)
    torch.cuda.synchronize()
    t1 = time.perf_counter()
    for e in range(epochs):
        sw.step(e)
    torch.cuda.synchronize()
    t2 = time.perf_counter()
    acc = [max(r['accuracies']) for r in sw.results()]
    return dict(setup_s=t1 - t0, run_s=t2 - t1, experiment_epochs_per_s=len(exps) * epochs / (t2 - t1),
                train_epoch_ms=events_ms(sw._graphs[0].replay, steps),
                test_epoch_ms=events_ms(sw._graphs[1].replay, steps), train_sets=list(sw.x_train.shape[:2]),
                test_sets=list(sw.x_test.shape[:2]), max_accuracy_range=[min(acc), max(acc)])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--seeds", type=int, default=2)
    ap.add_argument("--epochs", type=int, default=10)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--out")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("real_data_sweep_throughput needs a GPU")
    import __graft_entry__ as g
    g.build()
    from attacking_federate_learning_b200 import data, sweep
    out = dict(gpu=gpu_info(), seeds=args.seeds, epochs=args.epochs, steps=args.steps)
    with tempfile.TemporaryDirectory() as tmp:
        t0 = time.perf_counter()
        roots = write_files(tmp, np.random.default_rng(0))
        out['write_files_s'] = time.perf_counter() - t0
        for dataset, (n_train, n_test) in (('MNIST', (60000, 10000)), ('CIFAR10', (50000, 10000))):
            t0 = time.perf_counter()
            (xtr, _), (xte, _) = data.load(dataset, roots[dataset])
            res = dict(load_s=time.perf_counter() - t0, rows=[len(xtr), len(xte)])
            exps, _ = sweep.grid(RULES, ZS, MALS, [10], list(range(args.seeds)), 83, n_train, dataset=dataset)
            res['experiments'] = len(exps)
            res['real'] = measure(sweep, exps, dataset, args.epochs, args.steps, data_dir=roots[dataset])
            res['synthetic'] = measure(sweep, exps, dataset, args.epochs, args.steps, train_size=n_train,
                                       test_size=n_test)
            out[dataset] = res
            torch.cuda.empty_cache()
    line = json.dumps(out)
    print(line)
    if args.out:
        with open(args.out, 'w') as f:
            f.write(line + '\n')


if __name__ == "__main__":
    main()
