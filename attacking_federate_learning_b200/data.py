"""Real MNIST and CIFAR10 from the files torchvision keeps on disk, and the reference's sampler orders over them.

`load(dataset, data_dir)` reads what `datasets.MNIST(root)` / `datasets.CIFAR10(root)` read (data_sets.py:30, 60) and
returns every row through the reference's transforms (data_sets.py:27-28, 57-58), computed as torchvision computes them
in fp32: `u8.float().div(255)`, then `.sub_(mean).div_(std)`.  Nothing is downloaded; the files are checked before any
of them reaches a GPU, and a malformed one raises ValueError.

`sampler_order` and `backdoor_indices` restate the DistributedSampler partitions user.py:49-54 and backdoor.py:30-42
build: a seed-0 permutation of the training set, tiled to a multiple of the replica count, of which rank r holds every
num_replicas-th entry from r.  The reference never calls set_epoch, so every pass yields the same order.
"""
from __future__ import annotations

import gzip
import os
import pickle

import numpy as np
import torch

MNIST_DIRS = (os.path.join('MNIST', 'raw'), 'raw')        # torchvision's layout now, and in 2019
MNIST_FILES = {True: ('train-images-idx3-ubyte', 'train-labels-idx1-ubyte'),
               False: ('t10k-images-idx3-ubyte', 't10k-labels-idx1-ubyte')}
CIFAR10_DIR = 'cifar-10-batches-py'
CIFAR10_TRAIN = tuple(f'data_batch_{i}' for i in range(1, 6))
CIFAR10_TEST = ('test_batch',)
NORMALIZE = {'MNIST': ((0.1307,), (0.3081,)), 'CIFAR10': ((0.5, 0.5, 0.5), (0.5, 0.5, 0.5))}
N_CLASSES = 10


def _normalise(u8, dataset):
    """ToTensor() then Normalize(mean, std) on a uint8 [n, C, H, W] batch, with torchvision's fp32 operations."""
    mean, std = NORMALIZE[dataset]
    x = u8.to(torch.float32).div(255)
    return x.sub_(torch.as_tensor(mean, dtype=torch.float32).view(-1, 1, 1)).div_(
        torch.as_tensor(std, dtype=torch.float32).view(-1, 1, 1))


def _check_labels(y, where):
    if len(y) and (int(y.min()) < 0 or int(y.max()) >= N_CLASSES):
        raise ValueError(f"{where}: labels must lie in 0..{N_CLASSES - 1} (got {int(y.min())}..{int(y.max())})")
    return y


def _read_idx(path, ndim):
    """An IDX file of unsigned bytes with `ndim` dimensions (magic 0x08 << 8 | ndim), as a uint8 tensor."""
    try:
        with (gzip.open if path.endswith('.gz') else open)(path, 'rb') as f:
            data = f.read()
    except (EOFError, gzip.BadGzipFile) as e:
        raise ValueError(f"{path}: unreadable gzip stream ({e})") from e
    head = 4 * (ndim + 1)
    if len(data) < head:
        raise ValueError(f"{path}: {len(data)} bytes, shorter than an IDX header")
    magic = int.from_bytes(data[:4], 'big')
    if magic != 0x800 | ndim:
        raise ValueError(f"{path}: IDX magic {magic:#010x}, expected {0x800 | ndim:#010x}")
    dims = [int.from_bytes(data[4 * i:4 * i + 4], 'big') for i in range(1, ndim + 1)]
    if len(data) != head + int(np.prod(dims)):
        raise ValueError(f"{path}: {len(data) - head} data bytes, the header's dimensions {dims} need "
                         f"{int(np.prod(dims))}")
    return torch.frombuffer(bytearray(data), dtype=torch.uint8, offset=head).view(*dims)


def _find(dirs, name):
    for d in dirs:
        for p in (os.path.join(d, name), os.path.join(d, name + '.gz')):
            if os.path.isfile(p):
                return p
    return None


def _load_mnist(root, train):
    dirs = [os.path.join(root, d) for d in MNIST_DIRS]
    images, labels = MNIST_FILES[train]
    for d in dirs:                                   # the first directory that holds both files (plain or .gz)
        pi, pl = _find([d], images), _find([d], labels)
        if pi and pl:
            break
    else:
        raise FileNotFoundError(f"MNIST: no {images}[.gz] and {labels}[.gz] under {' or '.join(dirs)}")
    x, y = _read_idx(pi, 3), _read_idx(pl, 1)
    if tuple(x.shape[1:]) != (28, 28):
        raise ValueError(f"{pi}: images must be 28x28 (got {tuple(x.shape[1:])})")
    if len(x) != len(y):
        raise ValueError(f"{pi}: {len(x)} images but {pl} has {len(y)} labels")
    return _normalise(x.unsqueeze(1), 'MNIST').view(len(x), 28 * 28), _check_labels(y.to(torch.int64), pl)


class _NumpyUnpickler(pickle.Unpickler):
    """Unpickles the dicts of a CIFAR batch file: built-in containers and numpy arrays, nothing else."""
    _reconstruct = np.zeros(0).__reduce__()[0]
    ALLOWED = {('numpy.core.multiarray', '_reconstruct'): _reconstruct,
               ('numpy._core.multiarray', '_reconstruct'): _reconstruct,
               ('numpy', 'ndarray'): np.ndarray, ('numpy', 'dtype'): np.dtype}

    def find_class(self, module, name):
        try:
            return self.ALLOWED[(module, name)]
        except KeyError:
            raise ValueError(f"a CIFAR batch may only reference numpy arrays (found global {module}.{name})") from None


def _read_cifar_batch(path):
    with open(path, 'rb') as f:
        try:
            entry = _NumpyUnpickler(f, encoding='latin1').load()
        except (pickle.UnpicklingError, EOFError, TypeError, AttributeError, IndexError) as e:
            raise ValueError(f"{path}: not a CIFAR batch pickle ({type(e).__name__}: {e})") from e
    if not isinstance(entry, dict) or 'data' not in entry or 'labels' not in entry:
        raise ValueError(f"{path}: a CIFAR10 batch is a dict with 'data' and 'labels'")
    x, labels = entry['data'], entry['labels']
    if not isinstance(x, np.ndarray) or x.dtype != np.uint8 or x.ndim != 2 or x.shape[1] != 3 * 32 * 32:
        raise ValueError(f"{path}: 'data' must be a uint8 [k, 3072] array (got "
                         f"{getattr(x, 'dtype', type(x).__name__)} {getattr(x, 'shape', '')})")
    try:
        y = torch.as_tensor(np.asarray(labels, dtype=np.int64).reshape(-1))
    except (TypeError, ValueError) as e:
        raise ValueError(f"{path}: 'labels' must be a list of integers ({e})") from e
    if len(y) != len(x):
        raise ValueError(f"{path}: {len(x)} images but {len(y)} labels")
    return torch.from_numpy(np.ascontiguousarray(x)), _check_labels(y, path)


def _load_cifar10(root, train):
    d = os.path.join(root, CIFAR10_DIR)
    names = CIFAR10_TRAIN if train else CIFAR10_TEST
    missing = [n for n in names if not os.path.isfile(os.path.join(d, n))]
    if missing:
        raise FileNotFoundError(f"CIFAR10: no {', '.join(missing)} under {d}")
    parts = [_read_cifar_batch(os.path.join(d, n)) for n in names]
    x = torch.cat([p[0] for p in parts]).view(-1, 3, 32, 32)
    return _normalise(x, 'CIFAR10'), torch.cat([p[1] for p in parts])


def load(dataset, data_dir):
    """((x_train, y_train), (x_test, y_test)) on the CPU, as the reference's Dataset.__getitem__ yields them: MNIST
    x fp32 [n, 784] (ToTensor, Normalize((0.1307,), (0.3081,)), flattened as user.py:70 does), CIFAR10 x fp32
    [n, 3, 32, 32] (ToTensor, Normalize((0.5,) * 3, (0.5,) * 3)); y int64.  data_dir is the root data_sets.py passes
    (./mnist_data, ./cifar10_data): MNIST's four IDX files, plain or .gz, under <data_dir>/MNIST/raw/ or
    <data_dir>/raw/; CIFAR10's data_batch_1..5 (training order) and test_batch under <data_dir>/cifar-10-batches-py/.
    Raises FileNotFoundError naming what is missing and ValueError for a malformed file."""
    if dataset not in NORMALIZE:
        raise ValueError(f"unknown dataset {dataset!r} (expected one of {', '.join(NORMALIZE)})")
    if not os.path.isdir(data_dir):
        raise FileNotFoundError(f"{dataset}: data directory {data_dir} does not exist")
    read = _load_cifar10 if dataset == 'CIFAR10' else _load_mnist
    return read(data_dir, True), read(data_dir, False)


def sampler_order(n_rows, num_replicas):
    """The index list DistributedSampler(dataset of n_rows, num_replicas, rank) subsamples (shuffle=True, seed 0,
    epoch 0, drop_last=False): torch.randperm(n_rows) from a generator seeded 0, repeated up to
    ceil(n_rows / num_replicas) * num_replicas entries.  Rank r holds order[r::num_replicas], every pass."""
    if n_rows < 1 or num_replicas < 1:
        raise ValueError(f"sampler_order: n_rows and num_replicas must be >= 1 (got {n_rows}, {num_replicas})")
    perm = torch.randperm(n_rows, generator=torch.Generator().manual_seed(0))
    total = -(-n_rows // num_replicas) * num_replicas
    return perm.repeat(-(-total // n_rows))[:total]


def padded_length(n_rows, users_count):
    """The length of sampler_order(n_rows, users_count): every one of the users holds padded_length // users_count."""
    return -(-n_rows // users_count) * users_count


def backdoor_indices(backdoor, n_rows, seed=0, batch_size=200):
    """The training rows of BackdoorAttack's loader (backdoor.py:30-42), in its order.  'pattern': rank r of
    DistributedSampler(num_replicas=u) with u = max(n_rows // batch_size // 10, 1) and r = default_rng(seed).integers(u)
    (the reference draws r from the unseeded np.random.randint); sample 1, 2 or 3: rank backdoor - 1 of
    DistributedSampler(num_replicas=n_rows), one shuffled row."""
    if backdoor == 'pattern':
        u = max(n_rows // batch_size // 10, 1)
        return sampler_order(n_rows, u)[int(np.random.default_rng(seed).integers(u))::u]
    i = int(backdoor) - 1
    if not 0 <= i < n_rows:
        raise ValueError(f"backdoor sample {backdoor} lies past the training set ({n_rows} rows)")
    return sampler_order(n_rows, n_rows)[i:i + 1]
