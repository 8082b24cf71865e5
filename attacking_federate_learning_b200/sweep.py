"""Training sweeps: a grid of `harness.main` experiments trained side by side as one batch on the GPU.

An experiment is `(defense, mal_prop, num_std, users_count, seed[, backdoor])`, what main.py:104-131 takes: a drift
experiment (ALIE) is the 5-tuple, a backdoor experiment (`-b pattern|1|2|3`) adds 'pattern', 1, 2 or 3.  Experiment b
starts from exactly the data and weights `harness.main(mal_prop, num_std, defense, users_count, seed=seed,
backdoor=backdoor)` starts from (`harness.experiment_setup`) and runs main.py's epoch loop (main.py:64-71,
server.py:86-90):

  1. every client's MnistNet gradient on its minibatch (user.py:76-92), for every experiment in one launch of the
     client-gradient kernel (C ABI `afl_mnist_client_grads`), written straight into the experiment's rows of one
     [B, N_max, ld] client matrix;
  2. per (defence, attack), on the contiguous slice of experiments that use it (`batched.DeviceRound` with the
     experiments' own f_b = int(mal_prop * n_b), z_b and row counts): the attack on rows 0..f_b-1, the rule, and the
     server's momentum step on the slice's [B_r, D] weights at the base learning rate (server.py:89).  The drift attack
     is ALIE.  The backdoor attack is `DeviceRound.backdoor_start` at lr_t = learning_rate * fading_rate / (epoch +
     fading_rate) (server.py:50-52, float64 on the device from the epoch counter), then one launch of the trainer
     kernel (C ABI `afl_mnist_backdoor_train`, harness.BackdoorTrainer.train) for every backdoor experiment of the
     batch, then `DeviceRound.backdoor_finish`;
  3. the device epoch counter advances (the kernel reads it, so a replayed graph moves every client's minibatch on);
  4. every `test_step` epochs and at the last epoch, every experiment's test loss and accuracy (`afl_mnist_evaluate`,
     harness.main's test loop) into the next slot of a device table, and every backdoor experiment's backdoor test
     (`afl_mnist_backdoor_test`, main.py:91-95's 'POST') into the same slot of its own tables.

Nothing synchronises the host until the run ends.  With capture=True epoch 0 runs eagerly and the later epochs replay
a captured training epoch and test epoch; both paths give the same bits.  A client's gradient depends only on its own
weights and rows, so an experiment's trajectory does not depend on which other experiments share its batch (the
Krum and Bulyan distance tables aside, whose split count follows the batch unless AFL_GRAM_SPLITS pins it).  A
failure that only the data can show (a Bulyan round with no eligible user) lands in the rule's `DeviceRound.status`:
that experiment is reported as failed with the error `raise_for_status` gives, and the others complete.  So is a
backdoor experiment whose malicious training meets a NaN loss: Exception('...: Got nan loss'), as backdoor.py raises.

Outputs per experiment: the accuracy list and the CSV `harness.main` writes (np.savetxt(..., delimiter=',') in
out_dir/logs, with `_seed_<s>` before `.csv` so that seeds do not overwrite one another), and one summary CSV with the
parameters, max and final accuracy and status (and, when the run has a backdoor experiment, the backdoor and its max
and final backdoor accuracy; when it has an 8-tuple, every experiment's learning rate and batch size).  No checkpoint
is written: main.py's checkpoint path has no experiment key, so the experiments of a batch would overwrite one file.

    python -m attacking_federate_learning_b200.sweep -d Krum TrimmedMean -z 0.5 1.5 -m 0.1 0.24 -n 10 --seeds 0 1 -e 30
    python -m attacking_federate_learning_b200.sweep -d Krum NoDefense -z 1.0 -b No pattern 1 --seeds 0 1 -e 30
    python -m attacking_federate_learning_b200.sweep -s CIFAR10 -d Krum TrimmedMean -z 0.5 1.5 --seeds 0 1 -e 30
    python -m attacking_federate_learning_b200.sweep -s CIFAR10 -d Krum NoDefense -z 1.0 -b pattern 1 --cifar10-backdoor
    python -m attacking_federate_learning_b200.sweep -d Krum NoDefense -z 1.0 -l 0.05 0.1 0.2 -c 32 83 128 -e 30

dataset='CIFAR10' (main.py -s CIFAR10) runs the same loop on harness.Cifar10Net and `synthetic_cifar_problem`, with
the CIFAR10 kernels (C ABI `afl_cifar10_client_grads` and `afl_cifar10_evaluate`) in steps 1 and 4 and SYNTH-CIFAR10
log names.  A batch holds one dataset: the two models have different D.  CIFAR10 backdoor experiments
(main.py -s CIFAR10 -b ...) are batched with cifar10_backdoor=True (--cifar10-backdoor): the attacker's Cifar10Net
trains in the CIFAR10 trainer kernel (C ABI `afl_cifar10_backdoor_train`) and its backdoor test is
`afl_cifar10_backdoor_test`.  Without the switch `check` raises NotImplementedError for them, as before.

data_dir (--data-dir) trains on the real dataset's files there, as `harness.main(..., data_dir=...)` does: data.load's
rows, each client's DistributedSampler shard (user.py:49-54) and the backdoor loaders' rows (backdoor.py:30-42), with
main.py's log names (MNIST_..., CIFAR10_...).  The training data are one sampler-ordered copy per distinct padded
length ceil(N / n) * n (users counts 10, 100, 250, 500 and 1000 share the 60,000 rows of MNIST), and the kernel reads
each problem's set length from the device (C ABI `afl_*_client_grads_sets`); the test set is one copy for all seeds.

    python -m attacking_federate_learning_b200.sweep --data-dir ./mnist_data -d Krum NoDefense -z 1.0 -n 10 51 -e 30

Learning rate and batch size per experiment (main.py -l and -c; several values on the CLI, `grid(learning_rates=...,
batch_sizes=...)`): the 8-tuple experiments carry their own, and experiments of any (lr, c) train in one batch.  The
kernels take problem b's minibatch and test batch size from a device array (C ABI `afl_*_client_grads_each` and
`afl_*_evaluate_each`) and the momentum step its learning rate (`afl_momentum_step_batched`), and the backdoor's lr_t
starts from its own learning_rate * fading_rate; each problem's bits equal a sweep of its own (lr, c).  The backdoor
trainer keeps its own batch (200) and lr (0.1); epochs, momentum and fading rate stay per run.  An 8-tuple's CSV
takes its own learning rate and adds `_batch_<c>` before the seed, since main.py's name has no batch size.

trace=True (--trace) records why accuracy moves: in every epoch, after each rule, one `DeviceRound.attack_trace`
call (C ABI `afl_attack_trace_dev`) per (defence, attack) slice writes each experiment's ||aggregate - honest mean|| /
||honest mean||, the same for its first malicious row (the crafted vector when the attack wrote one), Krum's index and
Bulyan's malicious and selected counts into row `epoch` of [epochs, B] device tables, inside the captured epoch and
with no host synchronisation.  It reads G and the aggregates and writes only its tables, so every other output keeps
its bits.  `results()` gains `trace` per experiment (metrics.trace_record), and `run` writes one
`..._seed_<s>_trace.csv` per experiment (metrics.TRACE_HEADER) and four more summary columns (metrics.TRACE_SUMMARY).

    python -m attacking_federate_learning_b200.sweep -d Krum Bulyan TrimmedMean NoDefense -z 0.5 1.5 -m 0.1 0.24 -e 10 --trace
"""
from __future__ import annotations

import argparse
import csv as _csv
import itertools
import os
from operator import itemgetter

import numpy as np
import torch

from . import _native as nat
from . import batched
from . import data as _data
from . import harness
from . import metrics
from ._device import momentum_step_batched
from .defences import DefenseTypes

RULES = (DefenseTypes.Krum, DefenseTypes.Bulyan, DefenseTypes.TrimmedMean, DefenseTypes.NoDefense)
MAX_USERS = batched.MAX_CLIENTS          # clients per experiment (DeviceRound with large=True)
MAX_BATCH_SIZE = 128                     # minibatch rows of the client-gradient kernel
BACKDOOR_BATCH = 200                     # BackdoorTrainer's minibatch and test batch (the trainer kernel's limit)
SUMMARY = 'sweep_summary.csv'
FADING_RATE = {'MNIST': 10000, 'CIFAR10': 2000}         # main.py:144-147
TRACE_UNSET = -9                         # a trace table entry no epoch has written


class Experiment(tuple):
    """(defense, mal_prop, num_std, users_count, seed[, backdoor]): a drift experiment (backdoor False) is the 5-tuple,
    so it equals, prints and writes as before; a backdoor experiment carries 'pattern', 1, 2 or 3 as a sixth element.
    An experiment with its own learning rate and batch size (main.py's -l and -c) is the 8-tuple (defense, mal_prop,
    num_std, users_count, seed, backdoor, learning_rate, batch_size), backdoor False for a drift experiment; the short
    forms take the run's and return None for both."""
    __slots__ = ()
    _fields = ('defense', 'mal_prop', 'num_std', 'users_count', 'seed')     # a drift experiment's
    _hyper = ('backdoor', 'learning_rate', 'batch_size')

    def __new__(cls, defense, mal_prop, num_std, users_count, seed, backdoor=False, learning_rate=None,
                batch_size=None):
        t = (defense, mal_prop, num_std, users_count, seed)
        if learning_rate is None and batch_size is None:
            return tuple.__new__(cls, t if backdoor is False else t + (backdoor,))
        if learning_rate is None or batch_size is None:
            raise ValueError("an experiment gives both learning_rate and batch_size, or neither")
        return tuple.__new__(cls, t + (backdoor, learning_rate, batch_size))

    def __getnewargs__(self):
        return tuple(self)

    def __repr__(self):
        return 'Experiment(' + ', '.join(f'{n}={v!r}' for n, v in zip(self._fields + self._hyper, self)) + ')'

    defense, mal_prop, num_std, users_count, seed = (property(itemgetter(i)) for i in range(5))

    @property
    def backdoor(self):
        return self[5] if len(self) > 5 else False

    @property
    def learning_rate(self):
        return self[6] if len(self) == 8 else None

    @property
    def batch_size(self):
        return self[7] if len(self) == 8 else None

    @property
    def corrupted_count(self):
        return int(self.mal_prop * self.users_count)                      # main.py:21


def normalise_backdoor(bd):
    """main.py's -b value as harness.main takes it: False (also 'No'), 'pattern' or the sample 1, 2 or 3 (also '1'..'3').
    Raises ValueError for anything else."""
    if bd is False or (isinstance(bd, str) and bd == 'No'):
        return False
    if isinstance(bd, str) and bd == 'pattern':
        return bd
    if isinstance(bd, (str, int, np.integer)) and not isinstance(bd, bool) and str(bd) in ('1', '2', '3'):
        return int(bd)
    raise ValueError(f"unknown backdoor {bd!r} (expected False, 'pattern', 1, 2 or 3)")


def minibatch(n_train, users_count, user, batch_size, epoch):
    """Shard positions [lo, hi) of `user`'s minibatch at `epoch`: harness.Client.step's cycling position in closed form
    (the kernel computes the same).  The shard is training rows user, user + n, ...; row = user + n * position."""
    length = (n_train - user + users_count - 1) // users_count
    k = epoch % ((length + batch_size - 1) // batch_size)
    return k * batch_size, min(k * batch_size + batch_size, length)


def check(exp, batch_size=83, train_size=20000, dataset='MNIST', cifar10_backdoor=False):
    """Raise what main.py would raise for this experiment at its first `defend` (AssertionError for the reference's
    asserts), or for what the sweep's kernels do not take.  A CIFAR10 backdoor experiment is taken only with
    cifar10_backdoor=True.  batch_size is the run's, which an 8-tuple's own replaces.  Returns the normalised
    Experiment."""
    if len(exp) not in (5, 6, 8):
        raise ValueError(f"{exp}: an experiment has 5, 6 or 8 elements")
    exp = Experiment(str(exp[0]), float(exp[1]), float(exp[2]), int(exp[3]), int(exp[4]),
                     normalise_backdoor(exp[5]) if len(exp) > 5 else False,
                     *((float(exp[6]), int(exp[7])) if len(exp) == 8 else ()))
    if exp.batch_size is not None:
        batch_size = exp.batch_size
    if harness.check_dataset(dataset) == 'CIFAR10' and exp.backdoor is not False and not cifar10_backdoor:
        raise NotImplementedError(f"{exp}: CIFAR10 backdoor experiments need cifar10_backdoor=True "
                                  "(--cifar10-backdoor)")
    if exp.backdoor not in (False, 'pattern') and exp.backdoor > train_size:
        raise ValueError(f"{exp}: backdoor sample {exp.backdoor} lies past the training set ({train_size} rows)")
    if exp.defense not in RULES:
        raise KeyError(f"{exp}: unknown defence {exp.defense!r} (expected one of {', '.join(RULES)})")
    if not 1 <= exp.users_count <= MAX_USERS:
        raise (ValueError if exp.users_count < 1 else NotImplementedError)(
            f"{exp}: users_count must lie in 1..{MAX_USERS}")
    if exp.users_count > train_size:
        raise ValueError(f"{exp}: {exp.users_count} users need at least as many training samples (got {train_size})")
    n, f = exp.users_count, exp.corrupted_count
    if exp.defense == DefenseTypes.Krum and not n >= 2 * f + 1:           # defences.py:24
        raise AssertionError(f"{exp}: Krum needs users_count >= 2 * corrupted_count + 1 ({n}, {f})")
    if exp.defense == DefenseTypes.Bulyan and not n >= 4 * f + 3:         # defences.py:56
        raise AssertionError(f"{exp}: Bulyan needs users_count >= 4 * corrupted_count + 3 ({n}, {f})")
    if not 1 <= batch_size <= MAX_BATCH_SIZE:
        raise (ValueError if batch_size < 1 else NotImplementedError)(
            f"batch_size must lie in 1..{MAX_BATCH_SIZE} (got {batch_size})")
    return exp


def grid(defenses, num_stds, mal_props, users_counts, seeds, batch_size=83, train_size=20000, backdoors=(False,),
         dataset='MNIST', cifar10_backdoor=False, learning_rates=None, batch_sizes=None, learning_rate=0.1):
    """The Cartesian grid (defence-major, backdoor-minor) as (kept experiments, [(experiment, rejection), ...]): a cell
    main.py would reject is dropped with the exception `check` raises for it.  A drift cell (backdoor False) has 5
    elements, a backdoor cell 6.  When learning_rates or batch_sizes is given, every cell is an 8-tuple over the product
    with the learning rate and then the batch size as the innermost axes; the one not given is [learning_rate] or
    [batch_size]."""
    hyper = learning_rates is not None or batch_sizes is not None
    axes = (defenses, mal_props, num_stds, users_counts, seeds, backdoors)
    if hyper:
        axes += ([learning_rate] if learning_rates is None else learning_rates,
                 [batch_size] if batch_sizes is None else batch_sizes)
    kept, dropped = [], []
    for cell in itertools.product(*axes):
        if cell[5] is False and not hyper:
            cell = cell[:5]
        try:
            kept.append(check(cell, batch_size, train_size, dataset, cifar10_backdoor))
        except (AssertionError, KeyError, ValueError, NotImplementedError) as e:
            dropped.append((cell, e))
    return kept, dropped


def csv_name(exp, learning_rate, alpha=4, dataset='MNIST', data_dir=None):
    """harness.main's log name for this experiment, with `_seed_<s>` before `.csv`.  An 8-tuple's name takes its own
    learning rate and adds `_batch_<c>` before the seed: main.py's name has no batch size."""
    if exp.learning_rate is not None:
        learning_rate = exp.learning_rate
    name = harness.csv_name(exp.num_std, exp.defense, exp.backdoor, exp.mal_prop, exp.users_count, alpha, learning_rate,
                            dataset, data_dir)
    batch = '' if exp.batch_size is None else f'_batch_{exp.batch_size}'
    return name[:-len('.csv')] + f'{batch}_seed_{exp.seed}.csv'


def test_epochs(epochs, test_step):
    return [e for e in range(epochs) if e % test_step == 0 or e == epochs - 1]


def fading_lr(epoch, learning_rate, fading_rate, out=None):
    """harness.main's client learning rate lr_t = learning_rate * fading_rate / (epoch + fading_rate) (server.py:50-52)
    as float64 tensor arithmetic on `epoch` (an integer tensor), in the Python expression's order: one product, one
    sum and one IEEE division, so each value is the harness's Python double.  learning_rate: a float, or a float64
    tensor of per-problem products learning_rate * fading_rate already taken in Python (`lr_products`), which the
    epoch broadcasts against."""
    if isinstance(learning_rate, torch.Tensor):
        num = learning_rate
    else:
        num = torch.full(epoch.shape, learning_rate * fading_rate, dtype=torch.float64, device=epoch.device)
    return torch.div(num, epoch.to(torch.float64) + fading_rate, out=out)


def lr_products(learning_rates, fading_rate, device):
    """float64 [len(learning_rates)]: each learning_rate * fading_rate as the Python double `fading_lr` starts from."""
    return torch.tensor([lr * fading_rate for lr in learning_rates], dtype=torch.float64, device=device)


def backdoor_sets(specs, sampled=False):
    """The trainer kernel's backdoor sets from [(backdoor, x_train, y_train, seed), ...]: harness.backdoor_set (what
    BackdoorTrainer trains and tests on, from the reference's sampler rows when sampled) per spec, as x fp32
    [n_sets, max_len, *row shape] ([.., 784] for MNIST, [.., 3, 32, 32] for CIFAR10) and y int64 [n_sets, max_len],
    each set zero-padded to the longest, and set_len int32 [n_sets], on the training sets' device."""
    sets = [harness.backdoor_set(bd, x, y, seed, BACKDOOR_BATCH, sampled) for bd, x, y, seed in specs]
    dev, max_len = sets[0][0].device, max(len(x) for x, _ in sets)
    xs = torch.zeros((len(sets), max_len) + tuple(sets[0][0].shape[1:]), dtype=torch.float32, device=dev)
    ys = torch.zeros((len(sets), max_len), dtype=torch.int64, device=dev)
    for k, (x, y) in enumerate(sets):
        xs[k, :len(x)] = x
        ys[k, :len(y)] = y
    return xs, ys, torch.tensor([len(x) for x, _ in sets], dtype=torch.int32, device=dev)


def summary_header(with_backdoor, with_hyper=False, with_trace=False):
    """The summary CSV's columns; the backdoor ones only when the run has a backdoor experiment, the learning rate and
    batch size only when it has an 8-tuple, the trace's (metrics.TRACE_SUMMARY) only when the run traces."""
    bd = with_backdoor
    return list(Experiment._fields) + (['backdoor'] if bd else []) + \
        (['learning_rate', 'batch_size'] if with_hyper else []) + ['max_accuracy', 'final_accuracy'] + \
        (['max_backdoor_accuracy', 'final_backdoor_accuracy'] if bd else []) + \
        (metrics.TRACE_SUMMARY if with_trace else []) + ['status']


def trace_csv_name(name):
    """The trace CSV beside the accuracy CSV `name`: `..._seed_<s>_trace.csv`."""
    return name[:-len('.csv')] + '_trace.csv'


def write_logs(res, logs, names, with_backdoor=False, hyper=None, trace=False):
    """`run`'s files under `logs` from `results()`-style dicts: each successful experiment's accuracy CSV names[k]
    (np.savetxt, main.py:100) and, with trace, its trace CSV; then the summary CSV.  hyper: None, or [learning_rate,
    batch_size] per result for the summary.  Sets each dict's `csv` (and with trace `trace_csv`), None when it failed."""
    with_bd, with_hyper = with_backdoor, hyper is not None
    with open(os.path.join(logs, SUMMARY), 'w', newline='') as fh:
        w = _csv.writer(fh)
        w.writerow(summary_header(with_bd, with_hyper, trace))
        for k, r in enumerate(res):
            e = r['experiment']
            r['csv'] = None
            if trace:
                r['trace_csv'] = None
            head = list(e[:5]) + ([e.backdoor] if with_bd else []) + (hyper[k] if with_hyper else [])
            if r['error'] is None:
                r['csv'] = os.path.join(logs, names[k])
                np.savetxt(r['csv'], r['accuracies'], delimiter=',')     # main.py:100
                bd = r.get('backdoor_accuracies')
                tail = ([max(bd), bd[-1]] if bd else ['', '']) if with_bd else []
                if trace:
                    r['trace_csv'] = os.path.join(logs, trace_csv_name(names[k]))
                    metrics.write_trace_csv(r['trace_csv'], r['trace'])
                    tail += metrics.trace_summary(r['trace'])
                w.writerow(head + [max(r['accuracies']), r['accuracies'][-1]] + tail + ['ok'])
            else:
                w.writerow(head + ['', ''] + (['', ''] if with_bd else []) +
                           ([''] * len(metrics.TRACE_SUMMARY) if trace else []) +
                           [f"failed: {type(r['error']).__name__}: {r['error']}"])


def status_error(code, name):
    """The exception DeviceRound.raise_for_status raises for a status code, naming the experiment; for the backdoor
    trainer's NaN codes, the Exception backdoor.py raises."""
    if code in (nat.AFL_ERR_NAN_LOSS, nat.AFL_ERR_NAN_DIST_LOSS):
        return Exception(f"{name}: Got nan {'dist loss' if code == nat.AFL_ERR_NAN_DIST_LOSS else 'loss'}")
    if code == nat.AFL_ERR_NO_WINNER:
        e = KeyError(-1)
        e.add_note(f"{name}: a Bulyan selection round found no eligible user (defences.py:66)")
        return e
    exc, what = batched._STATUS_ERRORS.get(code, (nat.NativeError, None))
    return nat.NativeError(code, name) if what is None else exc(f"{name}: {what}")


class Sweep:
    """The device state of a batch of experiments and its epoch.  `run` drives it; tests and tools may drive it
    directly: `train_epoch()` and `test_epoch()` enqueue one epoch's work, `step(epoch)` runs epoch `epoch` (captured
    after epoch 0 when capture=True), `results()` synchronises and reads the tables back.

    Batch order: the drift experiments grouped by defence in RULES order, then the backdoor experiments grouped the
    same way, each group in the given order; `order[i]` is the position in `experiments` of batch problem i.  W, V:
    fp32 [B, D] weights and velocity; G: the [B, N_max, ld] client matrix (ld a multiple of 32, as AggregationServer
    pads); `rounds`: {defence: (slice, DeviceRound)} of the drift groups, `backdoor_rounds` the same for the backdoor
    groups, which occupy batch problems `bd0`..B-1.  Their DeviceRounds hold views of one f, z, lr and status over
    those problems, so the trainer reads every backdoor experiment in one launch.  `dataset` picks the model, the data
    and the kernels: x_train and x_test are [n_sets, n, 784] for MNIST and [n_sets, n, 3, 32, 32] for CIFAR10.
    Problem b trains on the first set_len[data_index[b]] rows of x_train[data_index[b]] and is tested on
    x_test[test_index[b]]: one set per seed for the synthetic data; with data_dir one training set per padded length
    (data.sampler_order) and one test set.  train_size and test_size: None (20,000 and 4,000 synthetic rows, or the
    files' row counts), or those sizes.  cifar10_backdoor: take CIFAR10 backdoor experiments (see `check`).

    Per problem: `batch_sizes` and `learning_rates` (an 8-tuple's own, else the run's batch_size and learning_rate),
    on the device as m (int32: the client minibatches and the test batches), lr (fp32: the momentum step) and
    lr_fading (float64: learning_rate * fading_rate, the backdoor's lr_t numerator), allocated once so that captured
    graphs keep their pointers.  trace=True: `trace` holds the [epochs, B] tables of DeviceRound.TRACE_TABLES (TRACE_UNSET
    until an epoch writes them), filled after each rule at row epoch_counter; None otherwise."""

    def __init__(self, experiments, epochs, learning_rate=0.1, momentum=0.9, batch_size=83, train_size=None,
                 test_size=None, test_step=5, capture=True, device='cuda', alpha=4, mal_epochs=5, fading_rate=10000,
                 dataset='MNIST', data_dir=None, cifar10_backdoor=False, trace=False):
        self.dataset = harness.check_dataset(dataset)
        self.data_dir = data_dir
        real = None
        if data_dir is not None:
            real = harness.real_sizes(dataset, data_dir, train_size, test_size)
            train_size, test_size = len(real[0][0]), len(real[1][0])
        train_size = 20000 if train_size is None else train_size
        test_size = 4000 if test_size is None else test_size
        exps = [check(e, batch_size, train_size, dataset, cifar10_backdoor) for e in experiments]
        if not exps:
            raise ValueError("sweep: no experiment")
        if epochs < 1 or test_step < 1 or test_size < 1:
            raise ValueError(f"sweep: epochs, test_step and test_size must be >= 1 (got {epochs}, {test_step}, "
                             f"{test_size})")
        if mal_epochs < 0 or fading_rate <= 0:
            raise ValueError(f"sweep: mal_epochs must be >= 0 and fading_rate > 0 (got {mal_epochs}, {fading_rate})")
        self.order = [i for bd in (False, True) for r in RULES for i, e in enumerate(exps)
                      if e.defense == r and (e.backdoor is not False) == bd]
        self.experiments = [exps[i] for i in self.order]
        self.epochs, self.learning_rate, self.momentum = epochs, learning_rate, momentum
        self.batch_size, self.train_size, self.test_size, self.test_step = batch_size, train_size, test_size, test_step
        self.alpha, self.mal_epochs, self.fading_rate = alpha, mal_epochs, fading_rate
        self.capture = capture
        dev = self.device = torch.device(device)
        seeds = list(dict.fromkeys(e.seed for e in self.experiments))
        i32 = dict(dtype=torch.int32, device=dev)
        xtr, ytr, xte, yte, w0 = [], [], [], [], {}
        for s in seeds:                                                   # harness.main's start, seed by seed
            if real is None:
                (a, b), (c, d), net = harness.experiment_setup(s, train_size, test_size, dev, dataset)
                xtr.append(a); ytr.append(b); xte.append(c); yte.append(d)
            else:                                                         # experiment_setup's weights, data loaded once
                torch.manual_seed(s)
                net = harness.model(dataset).to(dev)
            w0[s] = harness.ParamLayout(net.parameters()).flatten(list(net.parameters()))
        if real is None:
            self.x_train, self.y_train = torch.stack(xtr).contiguous(), torch.stack(ytr).contiguous()
            self.x_test, self.y_test = torch.stack(xte).contiguous(), torch.stack(yte).contiguous()
            self.set_len = torch.full((len(seeds),), train_size, **i32)
            self.data_index = torch.tensor([seeds.index(e.seed) for e in self.experiments], **i32)
            self.test_index = self.data_index
        else:
            (a, b), (c, d) = real
            a, b = a.to(dev), b.to(dev)
            xtr, ytr = [a] * len(seeds), [b] * len(seeds)                 # the backdoor sets' source, per seed
            users = {}                                                    # padded length -> a users count with it
            for e in self.experiments:
                users.setdefault(_data.padded_length(train_size, e.users_count), e.users_count)
            lengths = list(users)
            self.x_train = torch.zeros((len(lengths), max(lengths)) + tuple(a.shape[1:]), dtype=a.dtype, device=dev)
            self.y_train = torch.zeros((len(lengths), max(lengths)), dtype=b.dtype, device=dev)
            for k, T in enumerate(lengths):
                order = _data.sampler_order(train_size, users[T]).to(dev)
                self.x_train[k, :T], self.y_train[k, :T] = a[order], b[order]
            self.x_test, self.y_test = c.to(dev)[None].contiguous(), d.to(dev)[None].contiguous()
            self.set_len = torch.tensor(lengths, **i32)
            self.data_index = torch.tensor([lengths.index(_data.padded_length(train_size, e.users_count))
                                            for e in self.experiments], **i32)
            self.test_index = torch.zeros(len(self.experiments), **i32)
        B, self.D = len(self.experiments), w0[seeds[0]].numel()
        self.B = B
        self.N = max(e.users_count for e in self.experiments)
        self.batch_sizes = [batch_size if e.batch_size is None else e.batch_size for e in self.experiments]
        self.learning_rates = [learning_rate if e.learning_rate is None else e.learning_rate for e in self.experiments]
        self.m = torch.tensor(self.batch_sizes, **i32)
        self.lr = torch.tensor(self.learning_rates, dtype=torch.float32, device=dev)
        self.lr_fading = lr_products(self.learning_rates, fading_rate, dev)
        self.rows = torch.tensor([e.users_count for e in self.experiments], **i32)
        self.W = torch.stack([w0[e.seed] for e in self.experiments]).contiguous()
        self.V = torch.zeros_like(self.W)
        ld = (self.D + 31) // 32 * 32
        self._storage = torch.zeros((B, self.N, ld), dtype=torch.float32, device=dev)
        self.G = self._storage[:, :, :self.D]
        self.epoch_counter = torch.zeros(1, **i32)                       # the kernel's epoch
        self.test_slot = torch.zeros(1, **i32)                           # the next row of the test tables
        self.n_tests = len(test_epochs(epochs, test_step))
        self.loss_sum = torch.zeros((self.n_tests, B), dtype=torch.float64, device=dev)
        self.correct = torch.zeros((self.n_tests, B), **i32)
        L = nat.lib()
        cifar = self.dataset == 'CIFAR10'
        self._grads_fn = L.afl_cifar10_client_grads_each if cifar else L.afl_mnist_client_grads_each
        self._evaluate_fn = L.afl_cifar10_evaluate_each if cifar else L.afl_mnist_evaluate_each
        ws_bytes = (L.afl_cifar10_evaluate_workspace_bytes if cifar else L.afl_mnist_evaluate_workspace_bytes)
        self._eval_ws = torch.empty(max(ws_bytes(B, test_size, min(self.batch_sizes)), 256),
                                    dtype=torch.uint8, device=dev)
        self.bd0 = sum(e.backdoor is False for e in self.experiments)
        self._setup_backdoor(xtr, ytr, seeds)
        self.rounds, self.backdoor_rounds = {}, {}
        for r in RULES:
            for bd, rounds in ((False, self.rounds), (True, self.backdoor_rounds)):
                idx = [i for i, e in enumerate(self.experiments) if e.defense == r and (e.backdoor is not False) == bd]
                if not idx:
                    continue
                sl = slice(idx[0], idx[-1] + 1)
                rnd = batched.DeviceRound(self.G[sl], rows=True, rules=(r,), large=self.N > batched.ONE_TILE)
                if bd:                                                    # views of the batch-wide backdoor arrays
                    k = slice(sl.start - self.bd0, sl.stop - self.bd0)
                    rnd.f, rnd.z, rnd.lr, rnd.status = self._bd_f[k], self._bd_z[k], self._bd_lr[k], self._bd_status[k]
                sub = self.experiments[sl]
                rnd.f.copy_(torch.tensor([e.corrupted_count for e in sub], dtype=torch.int32))
                rnd.z.copy_(torch.tensor([e.num_std for e in sub], dtype=torch.float64))
                rnd.rows.copy_(torch.tensor([e.users_count for e in sub], dtype=torch.int32))
                rounds[r] = (sl, rnd)
        self.trace = None
        if trace:                                                         # [epochs, B] per DeviceRound.TRACE_TABLES
            self.trace = {k: torch.full((epochs, B), TRACE_UNSET, dtype=t, device=dev)
                          for k, t in batched.DeviceRound.TRACE_TABLES.items()}
        self._graphs = None

    def _setup_backdoor(self, xtr, ytr, seeds):
        """The backdoor experiments' sets (harness.backdoor_set, one per (backdoor, seed), padded to the longest),
        their trainer state and their backdoor-test tables; for CIFAR10 also the trainer's gradient rows and the
        backdoor test's batch tables, allocated once so that captured graphs keep their pointers."""
        bds = self.experiments[self.bd0:]
        self.n_backdoor = nb = len(bds)
        if not nb:
            return
        dev, i32 = self.device, dict(dtype=torch.int32, device=self.device)
        keys = list(dict.fromkeys((e.backdoor, e.seed) for e in bds))
        self.bd_x, self.bd_y, self.bd_len = backdoor_sets(
            [(bd, xtr[seeds.index(s)], ytr[seeds.index(s)], s) for bd, s in keys], sampled=self.data_dir is not None)
        self.bd_index = torch.tensor([keys.index((e.backdoor, e.seed)) for e in bds], **i32)
        self._bd_f = torch.zeros(nb, **i32)
        self._bd_z = torch.zeros(nb, dtype=torch.float64, device=dev)
        self._bd_lr = torch.zeros(nb, dtype=torch.float64, device=dev)
        self._bd_status = torch.zeros(nb, **i32)
        self.bd_initial = torch.empty((nb, self.D), dtype=torch.float32, device=dev)
        self.bd_mal = torch.empty((nb, self.D), dtype=torch.float32, device=dev)
        self.bd_loss_sum = torch.zeros((self.n_tests, nb), dtype=torch.float64, device=dev)
        self.bd_correct = torch.zeros((self.n_tests, nb), **i32)
        if self.dataset == 'CIFAR10':
            L = nat.lib()
            self._bd_train_ws = torch.empty(L.afl_cifar10_backdoor_train_workspace_bytes(nb), dtype=torch.uint8,
                                            device=dev)
            self._bd_test_ws = torch.empty(
                L.afl_cifar10_backdoor_test_workspace_bytes(nb, self.bd_x.shape[1], BACKDOOR_BATCH), dtype=torch.uint8,
                device=dev)

    def client_grads(self):
        """Step 1: every client's gradient into G at the current device epoch."""
        G = self._storage
        with torch.cuda.device(self.device):
            nat.check(self._grads_fn(
                self.W.data_ptr(), self.B, self.D, self.x_train.data_ptr(), self.y_train.data_ptr(),
                self.x_train.shape[0], self.x_train.shape[1], self.set_len.data_ptr(), self.data_index.data_ptr(),
                self.rows.data_ptr(), self.N, self.m.data_ptr(), max(self.batch_sizes), self.epoch_counter.data_ptr(),
                G.data_ptr(), G.stride(0), G.stride(1), torch.cuda.current_stream(self.device).cuda_stream))

    def backdoor_train(self, k=None):
        """The malicious networks of the backdoor experiments bd0 + k (all of them by default) in one launch
        (BackdoorTrainer.train), from bd_initial[k] into bd_mal[k]."""
        k = slice(0, self.n_backdoor) if k is None else k
        args = (self.bd_initial[k].data_ptr(), self.bd_mal[k].data_ptr(), k.stop - k.start, self.D,
                self.bd_x.data_ptr(), self.bd_y.data_ptr(), self.bd_x.shape[0], self.bd_x.shape[1],
                self.bd_len.data_ptr(), self.bd_index[k].data_ptr(), self._bd_f[k].data_ptr(), self._bd_z[k].data_ptr(),
                self._bd_status[k].data_ptr(), float(self.alpha), self.mal_epochs, BACKDOOR_BATCH)
        stream = torch.cuda.current_stream(self.device).cuda_stream
        with torch.cuda.device(self.device):
            if self.dataset == 'CIFAR10':                                 # problem b's gradient row: D floats at b D
                L = nat.lib()
                nat.check(L.afl_cifar10_backdoor_train(
                    *args, self._bd_train_ws.data_ptr() + k.start * self.D * 4,
                    L.afl_cifar10_backdoor_train_workspace_bytes(k.stop - k.start), stream))
            else:
                nat.check(nat.lib().afl_mnist_backdoor_train(*args, stream))

    def _defend(self, r, sl, rnd):
        agg = {DefenseTypes.Krum: rnd.krum, DefenseTypes.Bulyan: rnd.bulyan,
               DefenseTypes.TrimmedMean: rnd.trimmed_mean, DefenseTypes.NoDefense: rnd.no_defense}[r]()
        if self.trace is not None:       # reads G, agg and the rule's indices; the counter is still this epoch's
            names = ['agg_deviation', 'malicious_deviation'] + (
                ['krum_index'] if r == DefenseTypes.Krum else
                ['bulyan_malicious', 'bulyan_selected'] if r == DefenseTypes.Bulyan else [])
            rnd.attack_trace(agg, self.epoch_counter, {k: self.trace[k][:, sl] for k in names},
                             krum_index=rnd.krum_index if r == DefenseTypes.Krum else None,
                             selection=rnd.selection if r == DefenseTypes.Bulyan else None)
        momentum_step_batched(self.W[sl], self.V[sl], agg, self.momentum, self.lr[sl])

    def aggregate(self, rule=None):
        """Step 2 for one defence (every defence when rule is None): the attack, the rule and the momentum step."""
        for r, (sl, rnd) in self.rounds.items():
            if rule is not None and r != rule:
                continue
            rnd.alie()
            self._defend(r, sl, rnd)
        bd = [(r, sl, rnd) for r, (sl, rnd) in self.backdoor_rounds.items() if rule is None or r == rule]
        if not bd:
            return
        fading_lr(self.epoch_counter, self.lr_fading[self.bd0:], self.fading_rate, out=self._bd_lr)
        for r, sl, rnd in bd:
            rnd.backdoor_start(self.W[sl], initial=self.bd_initial[sl.start - self.bd0:sl.stop - self.bd0])
        self.backdoor_train(None if rule is None else slice(bd[0][1].start - self.bd0, bd[0][1].stop - self.bd0))
        for r, sl, rnd in bd:
            rnd.backdoor_finish(self.bd_mal[sl.start - self.bd0:sl.stop - self.bd0])
            self._defend(r, sl, rnd)

    def train_epoch(self):
        self.client_grads()
        self.aggregate()
        self.epoch_counter.add_(1)

    def test_epoch(self):
        """Step 4: every experiment's test loss sum and correct count into the next slot of the tables, and every
        backdoor experiment's backdoor test into the same slot of its tables."""
        stream = torch.cuda.current_stream(self.device).cuda_stream
        with torch.cuda.device(self.device):
            nat.check(self._evaluate_fn(
                self.W.data_ptr(), self.B, self.D, self.x_test.data_ptr(), self.y_test.data_ptr(),
                self.x_test.shape[0], self.test_size, self.test_index.data_ptr(), self.m.data_ptr(),
                min(self.batch_sizes), max(self.batch_sizes), self.test_slot.data_ptr(), self.n_tests, self.loss_sum.data_ptr(), self.correct.data_ptr(),
                self._eval_ws.data_ptr(), self._eval_ws.numel(), stream))
            if self.n_backdoor:
                args = (self.W[self.bd0:].data_ptr(), self.n_backdoor, self.D, self.bd_x.data_ptr(),
                        self.bd_y.data_ptr(), self.bd_x.shape[0], self.bd_x.shape[1], self.bd_len.data_ptr(),
                        self.bd_index.data_ptr(), BACKDOOR_BATCH, self.test_slot.data_ptr(), self.n_tests,
                        self.bd_loss_sum.data_ptr(), self.bd_correct.data_ptr())
                if self.dataset == 'CIFAR10':
                    nat.check(nat.lib().afl_cifar10_backdoor_test(*args, self._bd_test_ws.data_ptr(),
                                                                  self._bd_test_ws.numel(), stream))
                else:
                    nat.check(nat.lib().afl_mnist_backdoor_test(*args, stream))
        self.test_slot.add_(1)

    def is_test_epoch(self, epoch):
        return epoch % self.test_step == 0 or epoch == self.epochs - 1

    def step(self, epoch):
        """Epoch `epoch` (host bookkeeping only: the device counters advance on their own).  With capture, epoch 0 runs
        eagerly and captures the training and test epochs, which every later epoch replays."""
        if not self.capture or self._graphs is None:
            self.train_epoch()
            if self.is_test_epoch(epoch):
                self.test_epoch()
            if self.capture:
                self._graphs = (torch.cuda.CUDAGraph(), torch.cuda.CUDAGraph())
                with torch.cuda.device(self.device):
                    with torch.cuda.graph(self._graphs[0]):
                        self.train_epoch()
                    with torch.cuda.graph(self._graphs[1]):
                        self.test_epoch()
            return
        self._graphs[0].replay()
        if self.is_test_epoch(epoch):
            self._graphs[1].replay()

    def status(self):
        """Per batch problem: 0, or the first error code its rule's DeviceRound flagged or the backdoor trainer set
        (synchronises)."""
        st = torch.zeros(self.B, dtype=torch.int32, device=self.device)
        for sl, rnd in list(self.rounds.values()) + list(self.backdoor_rounds.values()):
            st[sl] = rnd.status
        return st.cpu().numpy()

    def results(self):
        """Synchronise and return, in the order of `experiments` as given, one dict per experiment: experiment,
        accuracies, accuracies_epochs, losses (harness.main's test loss), error (None, or the exception), and for a
        backdoor experiment backdoor_accuracies and backdoor_losses (BackdoorTrainer.test('POST') at each test epoch).
        With trace, also `trace`: metrics.trace_record's dict over epochs, None for a failed experiment."""
        st = self.status()
        tables = None if self.trace is None else {k: v.cpu().numpy() for k, v in self.trace.items()}
        correct = self.correct.cpu().numpy()
        loss = self.loss_sum.cpu().numpy()
        if self.n_backdoor:
            bd_correct, bd_loss = self.bd_correct.cpu().numpy(), self.bd_loss_sum.cpu().numpy()
            bd_len = self.bd_len.cpu().numpy()
            bd_index = self.bd_index.cpu().numpy()
        epochs = test_epochs(self.epochs, self.test_step)
        out = [None] * self.B
        for i, (pos, e) in enumerate(zip(self.order, self.experiments)):
            acc = [100. * float(correct[t, i]) / self.test_size for t in range(self.n_tests)]
            err = status_error(int(st[i]), f"experiment {tuple(e)}") if st[i] else None
            out[pos] = dict(experiment=e, accuracies=acc, accuracies_epochs=epochs,
                            losses=[float(loss[t, i]) / self.test_size for t in range(self.n_tests)], error=err)
            if tables is not None:
                out[pos]['trace'] = None if err is not None else metrics.trace_record(
                    e.defense, e.corrupted_count, *(tables[k][:, i] for k in batched.DeviceRound.TRACE_TABLES))
            if i >= self.bd0:
                k = i - self.bd0
                n = int(bd_len[bd_index[k]])
                out[pos]['backdoor_accuracies'] = [100. * int(bd_correct[t, k]) / n for t in range(self.n_tests)]
                out[pos]['backdoor_losses'] = [float(bd_loss[t, k]) / n for t in range(self.n_tests)]
        return out


def run(experiments, epochs, learning_rate=0.1, momentum=0.9, batch_size=83, train_size=None, test_size=None,
        test_step=5, out_dir='.', capture=True, device='cuda', alpha=4, mal_epochs=5, fading_rate=10000, dataset='MNIST',
        data_dir=None, cifar10_backdoor=False, trace=False):
    """Train every experiment for `epochs` epochs as one batch; write each one's accuracy CSV and the summary CSV under
    out_dir/logs.  Returns `Sweep.results()` with `csv` (None for a failed experiment) added to each dict.  Raises
    before any GPU work for an experiment main.py would reject (see `check`).  alpha, mal_epochs and fading_rate are
    harness.main's (the backdoor experiments' malicious training and client learning rate), and so is dataset ('MNIST'
    or 'CIFAR10', main.py -s).  data_dir: the real dataset's files (see the module docstring); train_size and test_size
    are then None or the files' row counts, and None means 20,000 and 4,000 synthetic rows otherwise.
    cifar10_backdoor=True takes CIFAR10 backdoor experiments (main.py -s CIFAR10 -b ...).  trace=True records every
    epoch's attack figures (see the module docstring) and adds `trace_csv` to each dict."""
    sw = Sweep(experiments, epochs, learning_rate, momentum, batch_size, train_size, test_size, test_step, capture,
               device, alpha, mal_epochs, fading_rate, dataset, data_dir, cifar10_backdoor, trace)
    with torch.cuda.device(sw.device):
        for epoch in range(epochs):
            sw.step(epoch)
    res = sw.results()
    logs = os.path.join(out_dir, 'logs')
    os.makedirs(logs, exist_ok=True)
    with_hyper = any(e.batch_size is not None for e in sw.experiments)
    hyper = {pos: [sw.learning_rates[i], sw.batch_sizes[i]] for i, pos in enumerate(sw.order)}
    names = [csv_name(r['experiment'], learning_rate, alpha, sw.dataset, sw.data_dir) for r in res]
    write_logs(res, logs, names, sw.n_backdoor > 0, [hyper[k] for k in range(len(res))] if with_hyper else None,
               trace)
    return res


def parser():
    """The command line of `python -m attacking_federate_learning_b200.sweep`."""
    p = argparse.ArgumentParser(description="A grid of main.py experiments as one batched training run.")
    p.add_argument('-d', '--defense', nargs='+', default=['NoDefense'], choices=list(RULES))
    p.add_argument('-z', '--num_std', nargs='+', type=float, default=[1.5])
    p.add_argument('-m', '--mal-prop', nargs='+', type=float, default=[0.24])
    p.add_argument('-n', '--users-count', nargs='+', type=int, default=[10])
    p.add_argument('--seeds', nargs='+', type=int, default=[0])
    p.add_argument('-b', '--backdoor', nargs='+', default=['No'], choices=['No', 'pattern', '1', '2', '3'])
    p.add_argument('-s', '--dataset', default='MNIST', choices=list(harness.DATASETS))
    p.add_argument('-e', '--epochs', type=int, default=300)
    p.add_argument('-c', '--batch_size', nargs='+', type=int, default=[83])
    p.add_argument('-l', '--learning_rate', nargs='+', type=float, default=[0.1])
    p.add_argument('--out-dir', default='.')
    p.add_argument('--no-capture', action='store_true')
    p.add_argument('--data-dir', default=None, help="the directory holding torchvision's MNIST or CIFAR10 files (the "
                   "reference's ./mnist_data or ./cifar10_data); without it the synthetic stand-in is trained")
    p.add_argument('--cifar10-backdoor', action='store_true', help="train CIFAR10 backdoor experiments (-s CIFAR10 "
                   "-b pattern|1|2|3) in the CIFAR10 trainer kernel; without it they are skipped")
    p.add_argument('--trace', action='store_true', help="record every epoch's attack figures (aggregate and malicious "
                   "row deviation from the honest mean, Krum's pick, Bulyan's malicious share) into a _trace.csv per "
                   "experiment and four more summary columns")
    return p


def main(argv=None):
    a = parser().parse_args(argv)
    train_size = 20000 if a.data_dir is None else len(harness.real_sizes(a.dataset, a.data_dir)[0][0])
    lrs, cs = list(dict.fromkeys(a.learning_rate)), list(dict.fromkeys(a.batch_size))
    hyper = dict(learning_rates=lrs, batch_sizes=cs) if len(lrs) > 1 or len(cs) > 1 else {}   # 8-tuple cells
    kept, dropped = grid(a.defense, a.num_std, a.mal_prop, a.users_count, a.seeds, cs[0], train_size,
                         backdoors=[normalise_backdoor(b) for b in dict.fromkeys(a.backdoor)], dataset=a.dataset,
                         cifar10_backdoor=a.cifar10_backdoor, **hyper)
    for cell, e in dropped:
        print(f"skipped {cell}: {type(e).__name__}: {e}")
    if not kept:
        print("no experiment left to run")
        return []
    res = run(kept, a.epochs, lrs[0], batch_size=cs[0], out_dir=a.out_dir, capture=not a.no_capture,
              fading_rate=FADING_RATE[a.dataset], dataset=a.dataset, data_dir=a.data_dir,
              cifar10_backdoor=a.cifar10_backdoor, trace=a.trace)
    for r in res:
        e = r['experiment']
        if r['error'] is None:
            bd = r.get('backdoor_accuracies')
            extra = f", backdoor max {max(bd):.2f}, final {bd[-1]:.2f}" if bd else ""
            print(f"{tuple(e)}: max accuracy {max(r['accuracies']):.2f}, final {r['accuracies'][-1]:.2f}{extra} -> "
                  f"{r['csv']}")
        else:
            print(f"{tuple(e)}: failed: {type(r['error']).__name__}: {r['error']}")
    return res


if __name__ == '__main__':
    main()
