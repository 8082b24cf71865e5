"""CPU checks of the real-data path (data.py, harness.main and sweep.run with data_dir, the _sets entry points): the
loader against torchvision's datasets element for element, the client shards, minibatch sequences and backdoor sets
against the DistributedSampler loaders user.py and backdoor.py build, the rejection of malformed files before any GPU
work, the new entry points' argument checks, and harness.main on real-format files on the CPU.  Every fixture is a
small seeded file written into tmp_path."""
import ctypes
import gzip
import os
import pickle

import numpy as np
import pytest
import torch

from attacking_federate_learning_b200 import data, harness, sweep
from test_cifar_args import CpuServer

P = ctypes.c_void_p(256)                 # a non-NULL pointer that is never dereferenced


def idx_bytes(a):
    """An IDX file of unsigned bytes holding the uint8 array a."""
    return (0x800 | a.ndim).to_bytes(4, 'big') + b''.join(int(d).to_bytes(4, 'big') for d in a.shape) + a.tobytes()


def write_mnist(root, n_train=70, n_test=23, seed=0, sub=os.path.join('MNIST', 'raw'), gz=False):
    """The four MNIST IDX files of a seeded random dataset under root/sub; returns root."""
    rng = np.random.default_rng(seed)
    d = os.path.join(root, sub)
    os.makedirs(d, exist_ok=True)
    for pre, n in (('train', n_train), ('t10k', n_test)):
        for kind, a in (('images-idx3', rng.integers(0, 256, (n, 28, 28), dtype=np.uint8)),
                        ('labels-idx1', rng.integers(0, 10, n, dtype=np.uint8))):
            path = os.path.join(d, f'{pre}-{kind}-ubyte')
            with (gzip.open(path + '.gz', 'wb') if gz else open(path, 'wb')) as f:
                f.write(idx_bytes(a))
    return str(root)


def write_cifar10(root, per_batch=7, n_test=9, seed=0):
    """data_batch_1..5, test_batch and batches.meta of a seeded random CIFAR10 under root/cifar-10-batches-py."""
    rng = np.random.default_rng(seed)
    d = os.path.join(root, data.CIFAR10_DIR)
    os.makedirs(d, exist_ok=True)
    for name, n in [(b, per_batch) for b in data.CIFAR10_TRAIN] + [('test_batch', n_test)]:
        entry = {'batch_label': name, 'data': rng.integers(0, 256, (n, 3072), dtype=np.uint8),
                 'labels': [int(v) for v in rng.integers(0, 10, n)], 'filenames': [f'{i}.png' for i in range(n)]}
        with open(os.path.join(d, name), 'wb') as f:
            pickle.dump(entry, f, protocol=4)
    with open(os.path.join(d, 'batches.meta'), 'wb') as f:
        pickle.dump({'label_names': [str(i) for i in range(10)]}, f, protocol=4)
    return str(root)


def tv_dataset(dataset, root, train, monkeypatch=None):
    tv = pytest.importorskip('torchvision')
    from torchvision import transforms
    mean, std = data.NORMALIZE[dataset]
    t = transforms.Compose([transforms.ToTensor(), transforms.Normalize(mean, std)])       # data_sets.py:27-28, 57-58
    if dataset == 'MNIST':
        return tv.datasets.MNIST(root, train=train, download=False, transform=t)
    import torchvision.datasets.cifar as cifar
    monkeypatch.setattr(tv.datasets.CIFAR10, '_check_integrity', lambda self: True)
    monkeypatch.setattr(cifar, 'check_integrity', lambda path, md5=None: os.path.isfile(path))   # the md5 checks
    return tv.datasets.CIFAR10(root, train=train, download=False, transform=t)


def assert_loads_like_torchvision(dataset, root, monkeypatch=None):
    got = data.load(dataset, root)
    for k, train in enumerate((True, False)):
        ds = tv_dataset(dataset, root, train, monkeypatch)
        x, y = got[k]
        assert len(x) == len(ds) and x.dtype == torch.float32 and y.dtype == torch.int64
        for i in range(len(ds)):
            xi, yi = ds[i]
            assert torch.equal(x[i], xi.view(-1) if dataset == 'MNIST' else xi), (train, i)
            assert int(y[i]) == yi
    return got


def test_mnist_loads_like_torchvision(tmp_path):
    (xtr, _), (xte, _) = assert_loads_like_torchvision('MNIST', write_mnist(tmp_path))
    assert xtr.shape == (70, 784) and xte.shape == (23, 784)


def test_mnist_old_layout_and_gzip_load_the_same_rows(tmp_path):
    want = data.load('MNIST', write_mnist(tmp_path / 'new'))
    for sub, gz in ((os.path.join('MNIST', 'raw'), True), ('raw', False), ('raw', True)):
        root = write_mnist(tmp_path / f'{sub.replace(os.sep, "_")}_{gz}', sub=sub, gz=gz)
        got = data.load('MNIST', root)
        for a, b in zip(got, want):
            assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])


def test_cifar10_loads_like_torchvision(tmp_path, monkeypatch):
    (xtr, ytr), (xte, _) = assert_loads_like_torchvision('CIFAR10', write_cifar10(tmp_path), monkeypatch)
    assert xtr.shape == (35, 3, 32, 32) and xte.shape == (9, 3, 32, 32)


def test_missing_files_name_what_was_looked_for(tmp_path):
    with pytest.raises(FileNotFoundError, match='does not exist'):
        data.load('MNIST', str(tmp_path / 'nowhere'))
    with pytest.raises(FileNotFoundError, match='train-images-idx3-ubyte'):
        data.load('MNIST', str(tmp_path))
    root = write_cifar10(tmp_path)
    os.remove(os.path.join(root, data.CIFAR10_DIR, 'data_batch_3'))
    with pytest.raises(FileNotFoundError, match='data_batch_3'):
        data.load('CIFAR10', root)


def corrupt(path, fn):
    with open(path, 'rb') as f:
        b = f.read()
    with open(path, 'wb') as f:
        f.write(fn(b))


@pytest.mark.parametrize('case', ['magic', 'truncated', 'long', 'label10', 'dims', 'count'])
def test_malformed_mnist_raises_before_any_gpu_work(tmp_path, case):
    root = write_mnist(tmp_path)
    raw = os.path.join(root, 'MNIST', 'raw')
    img, lab = os.path.join(raw, 'train-images-idx3-ubyte'), os.path.join(raw, 'train-labels-idx1-ubyte')
    if case == 'magic':
        corrupt(img, lambda b: (0x0801).to_bytes(4, 'big') + b[4:])
    elif case == 'truncated':
        corrupt(img, lambda b: b[:-1])
    elif case == 'long':
        corrupt(lab, lambda b: b + b'\0')
    elif case == 'label10':
        corrupt(lab, lambda b: b[:-1] + bytes([10]))
    elif case == 'dims':
        corrupt(img, lambda b: idx_bytes(np.zeros((70, 28, 27), np.uint8)))
    else:
        corrupt(lab, lambda b: idx_bytes(np.zeros(69, np.uint8)))
    with pytest.raises(ValueError):
        data.load('MNIST', root)
    with pytest.raises(ValueError):                                        # on a CPU-only machine, before CUDA
        sweep.Sweep([('NoDefense', 0.0, 1.0, 10, 0)], 1, data_dir=root)


class Foreign:
    pass


@pytest.mark.parametrize('case', ['global', 'shape', 'dtype', 'labels', 'label10', 'not_dict', 'garbage'])
def test_malformed_cifar10_raises(tmp_path, case):
    root = write_cifar10(tmp_path)
    path = os.path.join(root, data.CIFAR10_DIR, 'data_batch_2')
    x, y = np.zeros((7, 3072), np.uint8), [0] * 7
    entry = {'global': {'data': x, 'labels': y, 'extra': Foreign()},
             'shape': {'data': np.zeros((7, 3071), np.uint8), 'labels': y},
             'dtype': {'data': x.astype(np.int16), 'labels': y},
             'labels': {'data': x, 'labels': y[:-1]},
             'label10': {'data': x, 'labels': y[:-1] + [10]},
             'not_dict': [x, y]}.get(case)
    with open(path, 'wb') as f:
        f.write(b'not a pickle' if entry is None else pickle.dumps(entry, protocol=4))
    with pytest.raises(ValueError) as e:
        data.load('CIFAR10', root)
    if case == 'global':
        assert 'Foreign' in str(e.value)


def test_old_numpy_pickle_names_are_accepted(tmp_path):
    """The CIFAR10 distribution's pickles name numpy.core.multiarray._reconstruct; numpy 2 writes numpy._core."""
    root = write_cifar10(tmp_path)
    path = os.path.join(root, data.CIFAR10_DIR, 'test_batch')
    with open(path, 'rb') as f:
        b = pickle.dumps(pickle.load(f), protocol=3)                       # GLOBAL opcodes: names as plain text
    new, old = b'numpy._core.multiarray', b'numpy.core.multiarray'
    assert (new in b) != (old in b)
    with open(path, 'wb') as f:
        f.write(b.replace(new, old) if new in b else b.replace(old, new))
    assert torch.equal(data.load('CIFAR10', root)[1][0], data.load('CIFAR10', write_cifar10(tmp_path / 'b'))[1][0])


def loader_batches(n_rows, n, u, batch_size):
    """user.py:49-54's training loader for user u of n, as index batches (n = 1 uses num_replicas=1)."""
    from torch.utils.data import DataLoader, DistributedSampler, TensorDataset
    ds = TensorDataset(torch.arange(n_rows))
    return [b[0] for b in DataLoader(ds, sampler=DistributedSampler(ds, num_replicas=n, rank=u), batch_size=batch_size)]


@pytest.mark.parametrize('n_rows,n', [(60, 10), (61, 7), (23, 5), (5, 7), (30, 1), (13, 13)])
def test_shards_and_minibatches_are_the_reference_loaders(n_rows, n):
    order = data.sampler_order(n_rows, n)
    T = data.padded_length(n_rows, n)
    assert len(order) == T
    for u in range(n):
        for m in (1, 4, 83):
            want = loader_batches(n_rows, n, u, m)
            assert torch.equal(torch.cat(want), order[u::n])
            for e in range(2 * len(want) + 1):                            # cycle(train_loader)
                lo, hi = sweep.minibatch(T, n, u, m, e)                   # the kernel's closed form, n_train = T
                assert torch.equal(order[u::n][lo:hi], want[e % len(want)])


def test_harness_clients_hold_the_sampler_shards(tmp_path, monkeypatch):
    root = write_mnist(tmp_path, n_train=61)
    seen = []
    real_init = harness.Client.__init__

    def spy(self, user_id, is_malicious, x, y, *a, **k):
        seen.append((x, y))
        real_init(self, user_id, is_malicious, x, y, *a, **k)
    monkeypatch.setattr(harness.Client, '__init__', spy)
    monkeypatch.setattr(harness, 'AggregationServer', CpuServer)
    harness.main(0.0, 1.0, 'NoDefense', users_count=7, epochs=1, device='cpu', batch_size=4, data_dir=root,
                 out_dir=str(tmp_path), output=str(tmp_path / 'log.txt'))
    (xtr, ytr), _ = data.load('MNIST', root)
    for u, (x, y) in enumerate(seen):
        idx = torch.cat(loader_batches(61, 7, u, 4))
        assert torch.equal(x, xtr[idx]) and torch.equal(y, ytr[idx])


@pytest.mark.parametrize('n_rows', [61, 4000, 60000])
def test_backdoor_sets_are_backdoor_py_loaders(n_rows):
    from torch.utils.data import DistributedSampler
    ds = range(n_rows)
    for seed in (0, 1, 7):
        u = max(n_rows // 200 // 10, 1)
        r = int(np.random.default_rng(seed).integers(u))
        assert data.backdoor_indices('pattern', n_rows, seed).tolist() == \
            list(DistributedSampler(ds, num_replicas=u, rank=r))
    for b in (1, 2, 3):
        assert data.backdoor_indices(b, n_rows).tolist() == list(DistributedSampler(ds, num_replicas=n_rows, rank=b - 1))


def test_backdoor_set_sampled_applies_the_pattern_and_labels():
    g = torch.Generator().manual_seed(3)
    x, y = torch.randn(4100, 784, generator=g), torch.randint(0, 10, (4100,), generator=g)
    bx, by = harness.backdoor_set('pattern', x, y, seed=1, sampled=True)
    i = data.backdoor_indices('pattern', 4100, 1)
    want = x[i].clone()
    want.view(-1, 28, 28)[:, :5, :5] = 2.8
    assert torch.equal(bx, want) and torch.equal(by, torch.zeros(len(i), dtype=torch.int64))
    for b in (1, 2, 3):
        bx, by = harness.backdoor_set(b, x, y, sampled=True)
        j = data.backdoor_indices(b, 4100)
        assert torch.equal(bx, x[j]) and torch.equal(by, (y[j] + 1) % 5)
    xc = torch.randn(3000, 3, 32, 32, generator=g)
    bx, _ = harness.backdoor_set('pattern', xc, y[:3000], sampled=True)
    assert (bx[:, :, :5, :5] == 2.8).all()


@pytest.fixture(scope="module")
def lib():
    import __graft_entry__ as g
    g.build()
    from attacking_federate_learning_b200 import _native
    return _native.lib()


@pytest.mark.parametrize('name,D', [('afl_mnist_client_grads_sets', 79_510), ('afl_cifar10_client_grads_sets', 117_706)])
def test_sets_entry_points_reject_bad_arguments_before_any_cuda_call(lib, name, D):
    from attacking_federate_learning_b200 import _native as nat
    ld = (D + 31) // 32 * 32

    def call(**kw):
        a = dict(weights=P, batch=2, d=D, x=P, y=P, n_sets=1, n_rows=100, set_len=P, data_index=P, rows=P, n=10, m=83,
                 epoch=P, G=P, batch_stride=10 * ld, ld=ld, stream=None)
        a.update(kw)
        return getattr(lib, name)(*a.values())
    for p in ('weights', 'x', 'y', 'set_len', 'data_index', 'rows', 'epoch', 'G'):
        assert call(**{p: None}) == nat.AFL_ERR_BAD_ARG, p
    assert call(d=D + 1) == nat.AFL_ERR_UNSUPPORTED
    assert call(m=129) == nat.AFL_ERR_UNSUPPORTED
    assert call(m=0) == nat.AFL_ERR_BAD_ARG
    assert call(n=1025) == nat.AFL_ERR_UNSUPPORTED
    assert call(n=0) == nat.AFL_ERR_BAD_ARG
    assert call(n=101) == nat.AFL_ERR_BAD_ARG                             # more clients than the set pitch
    assert call(n_rows=0) == nat.AFL_ERR_BAD_ARG
    assert call(n_sets=0) == nat.AFL_ERR_BAD_ARG
    assert call(ld=D - 1) == nat.AFL_ERR_BAD_ARG
    assert call(batch_stride=9 * ld) == nat.AFL_ERR_BAD_ARG
    assert call(batch=65536) == nat.AFL_ERR_UNSUPPORTED
    assert name.encode() in lib.afl_last_error()


def test_harness_main_writes_the_reference_named_csv(tmp_path, monkeypatch):
    monkeypatch.setattr(harness, 'AggregationServer', CpuServer)
    root = write_mnist(tmp_path / 'mnist_data', n_train=200, n_test=30)
    out = tmp_path / 'out'
    acc, epochs, csv = harness.main(0.0, 1.0, 'NoDefense', users_count=7, epochs=2, device='cpu', data_dir=root,
                                    out_dir=str(out), output=str(tmp_path / 'log.txt'), test_step=1)
    assert os.path.basename(csv) == 'MNIST_stdev_1.0_NoDefense_backdoor-False_mal_prop_0.0_users_7_alpha_None_lr_0.1.csv'
    assert os.path.isfile(csv) and epochs == [0, 1]
    assert np.array_equal(np.atleast_1d(np.loadtxt(csv, delimiter=',')), np.array(acc))
    assert all(a * 30 / 100 == round(a * 30 / 100) for a in acc)           # accuracies over the files' 30 test rows
    assert "'dataset': 'MNIST'" in open(tmp_path / 'log.txt').read()
    with pytest.raises(ValueError, match='train_size'):
        harness.main(0.0, 1.0, 'NoDefense', epochs=1, device='cpu', data_dir=root, train_size=20000, out_dir=str(out))
    root10 = write_cifar10(tmp_path / 'cifar10_data', per_batch=12, n_test=10)
    _, _, csv = harness.main(0.0, 1.0, 'NoDefense', users_count=3, epochs=1, device='cpu', data_dir=root10,
                             dataset='CIFAR10', out_dir=str(out), output=str(tmp_path / 'log.txt'), backdoor=1)
    assert os.path.basename(csv).startswith('CIFAR10_stdev_1.0_NoDefense_backdoor-1_')


def test_setup_keeps_the_initial_weights(tmp_path):
    root = write_mnist(tmp_path)
    for seed in (0, 4):
        _, _, net = harness.experiment_setup(seed, None, None, 'cpu', data_dir=root)
        _, _, want = harness.experiment_setup(seed, 20000, 4000, 'cpu')
        for p, q in zip(net.parameters(), want.parameters()):
            assert torch.equal(p, q)


def test_sweep_names_and_cli(tmp_path):
    e = sweep.Experiment('Krum', 0.1, 1.0, 51, 2)
    assert sweep.csv_name(e, 0.1, data_dir='d') == \
        'MNIST_stdev_1.0_Krum_backdoor-False_mal_prop_0.1_users_51_alpha_None_lr_0.1_seed_2.csv'
    assert sweep.csv_name(e, 0.1).startswith('SYNTH-MNIST_')
    assert sweep.csv_name(e, 0.1, dataset='CIFAR10', data_dir='d').startswith('CIFAR10_')
    with pytest.raises(FileNotFoundError):
        sweep.main(['--data-dir', str(tmp_path / 'none'), '-e', '1'])
    with pytest.raises(NotImplementedError):                              # CIFAR10 backdoor cells stay rejected
        sweep.Sweep([('NoDefense', 0.0, 1.0, 3, 0, 1)], 1, dataset='CIFAR10',
                    data_dir=write_cifar10(tmp_path))
