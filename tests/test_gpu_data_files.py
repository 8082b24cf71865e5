"""The real-data path on an H100 (afl_*_client_grads_sets, sweep.run and harness.main with data_dir), on small seeded
MNIST- and CIFAR10-format files written into a temporary directory.

1. `_sets` with every set length equal to the pitch equals the old entry point bit for bit (both nets).
2. In a batch whose sets have different lengths, every problem's rows equal the old entry point run on its set alone,
   bit for bit, including a length that cuts the last minibatch short; out-of-range lengths leave sentinels untouched.
3. Padded-shard gradients against float64 autograd within the existing tolerances.
4. sweep.run(data_dir=...): captured equals eager; a grid mixing n = 7, 10 and 51 equals each experiment run alone.
5. The first weight step against harness.main(data_dir=...)'s: MNIST drift, pattern and 1, and CIFAR10 drift.
"""
import os

import pytest
import torch

from test_data_files import write_cifar10, write_mnist
from test_gpu_cifar_sweep import check_against_autograd as cifar_check
from test_gpu_sweep import BOUND, i32, pinned_splits, rel_errors  # noqa: F401
from test_gpu_sweep import autograd as mnist_autograd

pytestmark = pytest.mark.gpu

NETS = {'MNIST': (79_510, 79_520), 'CIFAR10': (117_706, 117_728)}


@pytest.fixture(scope="module")
def env():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    import __graft_entry__ as g
    g.build()
    from attacking_federate_learning_b200 import _native, data, harness, sweep
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    return _native, data, harness, sweep


@pytest.fixture(scope="module")
def roots(tmp_path_factory):
    base = tmp_path_factory.mktemp("data")
    return {'MNIST': write_mnist(base / 'mnist_data', n_train=2000, n_test=500, seed=1),
            'CIFAR10': write_cifar10(base / 'cifar10_data', per_batch=400, n_test=300, seed=2)}


_LOADED = {}


def loaded(data, roots, dataset):
    if dataset not in _LOADED:
        (xtr, ytr), (xte, yte) = data.load(dataset, roots[dataset])
        _LOADED[dataset] = xtr.cuda(), ytr.cuda(), xte.cuda(), yte.cuda()
    return _LOADED[dataset]


def weights(harness, dataset, B, seed=0):
    torch.manual_seed(seed)
    net = harness.model(dataset).cuda()
    w = harness.ParamLayout(net.parameters()).flatten(list(net.parameters()))
    g = torch.Generator("cuda").manual_seed(seed + 1)
    return torch.stack([w + 0.01 * torch.randn(w.numel(), device="cuda", generator=g) for _ in range(B)]).contiguous()


def grads(nat, dataset, W, x, y, set_len, data_index, rows, n, m, epoch, G):
    """The _sets entry point when set_len is given, else the old one with n_train = x.shape[1]."""
    L = nat.lib()
    fn = {'MNIST': (L.afl_mnist_client_grads, L.afl_mnist_client_grads_sets),
          'CIFAR10': (L.afl_cifar10_client_grads, L.afl_cifar10_client_grads_sets)}[dataset]
    head = (W.data_ptr(), W.shape[0], NETS[dataset][0], x.data_ptr(), y.data_ptr(), x.shape[0], x.shape[1])
    tail = (data_index.data_ptr(), rows.data_ptr(), n, m, epoch.data_ptr(), G.data_ptr(), G.stride(0), G.stride(1),
            torch.cuda.current_stream().cuda_stream)
    nat.check(fn[0](*head, *tail) if set_len is None else fn[1](*head, set_len.data_ptr(), *tail))


@pytest.mark.parametrize("dataset", list(NETS))
def test_full_length_sets_equal_the_old_entry_point(env, roots, dataset):
    nat, data, harness, _ = env
    xtr, ytr, _, _ = loaded(data, roots, dataset)
    x, y = torch.stack([xtr, xtr.flip(0)]).contiguous(), torch.stack([ytr, ytr.flip(0)]).contiguous()
    W = weights(harness, dataset, 3)
    rows, idx = i32([10, 7, 10]), i32([0, 1, 1])
    for epoch in (0, 5, 24):
        out = []
        for sl in (None, i32([2000, 2000])):
            G = torch.full((3, 10, NETS[dataset][1]), 7.0, device="cuda")
            grads(nat, dataset, W, x, y, sl, idx, rows, 10, 83, i32([epoch]), G)
            out.append(G)
        assert torch.equal(out[0].view(torch.int32), out[1].view(torch.int32)), epoch


@pytest.mark.parametrize("dataset", list(NETS))
def test_sets_of_different_lengths_equal_each_set_alone(env, roots, dataset):
    """Sets padded for n = 7 (2002 rows), 10 (2000) and 51 (2040) in one [3, 2040] batch.  Shard lengths 286, 200 and
    40 at m = 83: epoch 3 takes 37 rows for n = 7, epoch 2 34 rows for n = 10, epoch 0 40 rows for n = 51.  Problems 3
    and 4 point at a set whose length is below their n or above the pitch and must write nothing."""
    nat, data, harness, _ = env
    xtr, ytr, _, _ = loaded(data, roots, dataset)
    ns, pitch = (7, 10, 51), 2040
    sets = [data.sampler_order(2000, n).cuda() for n in ns]
    x = torch.zeros((5, pitch) + tuple(xtr.shape[1:]), device="cuda")
    y = torch.zeros((5, pitch), dtype=torch.int64, device="cuda")
    for k, o in enumerate(sets):
        x[k, :len(o)], y[k, :len(o)] = xtr[o], ytr[o]
    set_len = i32([2002, 2000, 2040, 40, 2041])
    rows, idx = i32([7, 10, 51, 51, 7]), i32([0, 1, 2, 3, 4])
    W = weights(harness, dataset, 5, seed=3)
    D, ld = NETS[dataset]
    for epoch in (0, 2, 3):
        G = torch.full((5, 51, ld), 7.0, device="cuda")
        grads(nat, dataset, W, x, y, set_len, idx, rows, 51, 83, i32([epoch]), G)
        for b, n in enumerate(ns):
            T = len(sets[b])
            want = torch.full((1, n, ld), 7.0, device="cuda")
            grads(nat, dataset, W[b:b + 1].contiguous(), x[b:b + 1, :T].contiguous(), y[b:b + 1, :T].contiguous(),
                  None, i32([0]), i32([n]), n, 83, i32([epoch]), want)
            assert torch.equal(G[b, :n].view(torch.int32), want[0].view(torch.int32)), (epoch, n)
            assert (G[b, n:] == 7.0).all()
        assert (G[3:] == 7.0).all()                                       # out-of-range lengths: untouched


@pytest.mark.parametrize("dataset, n, u, epoch", [('MNIST', 7, 6, 3), ('MNIST', 51, 50, 0), ('CIFAR10', 7, 0, 3),
                                                  ('CIFAR10', 51, 17, 0)])
def test_padded_shard_gradients_against_float64_autograd(env, roots, dataset, n, u, epoch):
    """User u's minibatch is a chunk of DistributedSampler's shard; for n = 7 the shard's last rows repeat the
    permutation's first two."""
    nat, data, harness, sweep = env
    xtr, ytr, _, _ = loaded(data, roots, dataset)
    order = data.sampler_order(2000, n).cuda()
    W = weights(harness, dataset, 1, seed=5)
    D, ld = NETS[dataset]
    G = torch.full((1, n, ld), 7.0, device="cuda")
    grads(nat, dataset, W, xtr[order][None].contiguous(), ytr[order][None].contiguous(), i32([len(order)]), i32([0]),
          i32([n]), n, 83, i32([epoch]), G)
    lo, hi = sweep.minibatch(len(order), n, u, 83, epoch)
    rows = order[u::n][lo:hi]
    got = G[0, u, :D]
    if dataset == 'MNIST':
        _, g64 = mnist_autograd(harness, W[0], xtr[rows], ytr[rows], torch.float64)
        assert all(e < BOUND for e in rel_errors(got, g64)), rel_errors(got, g64)
    else:
        cifar_check(harness, got, W[0], xtr[rows], ytr[rows])


def real_sweep(sweep, root, exps, dataset='MNIST', epochs=4, capture=False):
    return sweep.Sweep(exps, epochs, batch_size=83, test_step=2, capture=capture, dataset=dataset, data_dir=root)


def tables(sw):
    out = [sw.W, sw.V, sw.loss_sum, sw.correct]
    if sw.n_backdoor:
        out += [sw.bd_loss_sum, sw.bd_correct]
    return [t.clone() for t in out]


@pytest.mark.parametrize("dataset", list(NETS))
def test_captured_sweep_equals_eager(env, roots, pinned_splits, dataset):
    _, _, _, sweep = env
    exps = [("Krum", 0.1, 1.0, 10, 0), ("TrimmedMean", 0.24, 0.5, 7, 1), ("NoDefense", 0.24, 1.5, 51, 0)]
    if dataset == 'MNIST':
        exps += [("NoDefense", 0.24, 1.0, 10, 0, 'pattern'), ("Krum", 0.24, 1.0, 7, 1, 1)]
    runs = []
    for capture in (False, True):
        sw = real_sweep(sweep, roots[dataset], exps, dataset, epochs=5, capture=capture)
        assert sw.x_train.shape[:2] == (3, 2040) and sw.x_test.shape[:2] == (1, 500 if dataset == 'MNIST' else 300)
        for e in range(5):
            sw.step(e)
        torch.cuda.synchronize()
        runs.append(tables(sw))
    for a, b in zip(*runs):
        assert torch.equal(a, b)


def test_mixed_users_grid_equals_each_experiment_alone(env, roots, pinned_splits, tmp_path):
    _, _, _, sweep = env
    exps = [("NoDefense", 0.24, 1.0, 7, 0), ("Krum", 0.1, 1.0, 10, 1), ("TrimmedMean", 0.24, 1.5, 51, 0),
            ("NoDefense", 0.24, 1.0, 51, 1, 'pattern')]
    res = sweep.run(exps, 4, test_step=2, out_dir=str(tmp_path), data_dir=roots['MNIST'])
    for e, r in zip(exps, res):
        alone = sweep.run([e], 4, test_step=2, out_dir=str(tmp_path / 'alone'), data_dir=roots['MNIST'])[0]
        assert r['error'] is None and r['accuracies'] == alone['accuracies'] and r['losses'] == alone['losses'], e
        assert r.get('backdoor_accuracies') == alone.get('backdoor_accuracies')
        assert os.path.basename(r['csv']).startswith('MNIST_stdev_')


FIRST_STEP = [('MNIST', ("TrimmedMean", 0.24, 1.5, 10, 0)), ('MNIST', ("NoDefense", 0.24, 1.0, 7, 1)),
              ('MNIST', ("NoDefense", 0.24, 1.0, 10, 0, 'pattern')), ('MNIST', ("Krum", 0.24, 1.0, 10, 1, 1)),
              ('CIFAR10', ("NoDefense", 0.24, 1.5, 10, 0)), ('CIFAR10', ("TrimmedMean", 0.24, 1.5, 7, 1))]


@pytest.mark.parametrize("dataset, e", FIRST_STEP)
def test_first_weight_step_against_harness_main(env, roots, dataset, e, monkeypatch, tmp_path):
    _, _, harness, sweep = env
    from attacking_federate_learning_b200.server import AggregationServer
    seen = {}

    class Recording(AggregationServer):
        def __init__(self, *a, initial_weights=None, **k):
            super().__init__(*a, initial_weights=initial_weights, **k)
            seen['w0'] = initial_weights.clone()

        def defend(self, *a, **k):
            super().defend(*a, **k)
            seen.setdefault('w1', self.current_weights.clone())
    monkeypatch.setattr(harness, 'AggregationServer', Recording)
    exp = sweep.check(e, dataset=dataset, train_size=2000)
    harness.main(exp.mal_prop, exp.num_std, exp.defense, users_count=exp.users_count, epochs=1, seed=exp.seed,
                 backdoor=exp.backdoor, dataset=dataset, data_dir=roots[dataset], out_dir=str(tmp_path),
                 output=str(tmp_path / 'log.txt'), fading_rate=sweep.FADING_RATE[dataset])
    sw = real_sweep(sweep, roots[dataset], [e], dataset, epochs=1)
    assert torch.equal(sw.W[0], seen['w0'])                               # the same initial weights
    sw.step(0)
    step = seen['w1'].double() - seen['w0'].double()
    rel = float(((sw.W[0].double() - seen['w0'].double()) - step).norm() / step.norm())
    print(f"first weight step {dataset} {e}: relative difference {rel:.3e}")
    assert rel < 1e-3, (e, rel)
