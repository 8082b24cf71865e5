"""Drop-in for the reference's `defences.py` (same names, same argument meaning, same error
behaviour), backed by the sm_90a kernels in lib/libafl_b200.so.

Reference surface mirrored (file:line in /root/reference):
    DefenseTypes                          defences.py:4-11
    no_defense(users_grads, n, f)         defences.py:13-14
    _krum_create_distances(users_grads)   defences.py:16-21
    krum(users_grads, n, f, distances=None, return_index=False, debug=False)   defences.py:23-42
    trimmed_mean(users_grads, n, f)       defences.py:44-52
    bulyan(users_grads, n, f)             defences.py:55-70
    defend                                defences.py:73-75

`users_grads` may be
  * a NumPy float32 [N, D] array (what server.py:35 holds): the call goes through the host-buffer
    C entry point `afl_defend_host` (H2D staging overlapped with the kernels) and returns NumPy —
    `krum` returns a *view* of the winning row exactly like the reference.  The matrix may be larger
    than the GPU: column slabs are streamed through a bounded device budget (free memory less 1 GiB,
    capped by the environment variable AFL_HOST_DEVICE_BYTES); a budget too small for two slabs and
    the N x N tables raises NotImplementedError stating the bytes needed.  `_krum_create_distances` and
    `krum(..., return_index=True)` stream the matrix into the same slab-summed distance table
    (`afl_sqdist_host`), so `krum(G, n, f)` is `G[krum(G, n, f, return_index=True)]`;
    `bulyan(..., return_selection=True)` also returns the selection (`afl_bulyan_host`);
  * a torch.cuda float32 / bfloat16 / float16 [N, D] tensor: device-resident path, returns torch tensors
    (fp32; a 16-bit matrix gives the reference's result on its values upcast to fp32), `krum` again returns a
    view `users_grads[idx]`.
There is no CPU implementation in this package.
"""
from __future__ import annotations

import ctypes as C

import numpy as np

from . import _native as nat


class DefenseTypes:
    NoDefense = 'NoDefense'
    Krum = 'Krum'
    TrimmedMean = 'TrimmedMean'
    Bulyan = 'Bulyan'

    def __str__(self):
        return self.value


def _is_torch_cuda(x) -> bool:
    try:
        import torch
    except ImportError:  # pragma: no cover
        return False
    return isinstance(x, torch.Tensor) and x.is_cuda


def _as_host_matrix(users_grads) -> np.ndarray:
    G = np.asarray(users_grads)
    if G.ndim != 2:
        raise ValueError("users_grads must be 2-D [clients, params]")
    if G.dtype != np.float32 or not G.flags.c_contiguous:
        raise NotImplementedError("host path: users_grads must be a C-contiguous float32 array "
                                  "(as allocated by the reference, server.py:35)")
    return G


def _host_call(rule: str, G: np.ndarray, users_count: int, corrupted_count: int, want_out: bool = True):
    n, d = G.shape
    out = np.empty((d,), np.float32) if want_out else None
    idx = C.c_int(-1)
    rc = nat.lib().afl_defend_host(rule.encode(), G.ctypes.data, n, d, G.strides[0] // 4, int(users_count),
                                   int(corrupted_count), out.ctypes.data if want_out else None, C.byref(idx), 0)
    nat.check(rc)
    return out, idx.value


class DistanceTable:
    """Dense replacement for the reference's dict-of-dicts (defences.py:16-21).

    `dense` is the symmetric [n, n] fp32 table (torch.cuda tensor).  `order` is the list of users still
    present, in the reference's dict order.  The mapping protocol used by the reference (`keys()`,
    `[user].values()`, `pop`) is provided so that code written against the dict keeps working.
    """

    def __init__(self, dense, order=None):
        self.dense = dense
        n = dense.shape[0]
        self.order = list(order) if order is not None else ([1, 0] + list(range(2, n)) if n >= 2 else [])
        self._host = None

    def _rows(self):
        if self._host is None:
            self._host = self.dense.detach().cpu().numpy() if hasattr(self.dense, "detach") else np.asarray(self.dense)
        return self._host

    def keys(self):
        return list(self.order)

    def __len__(self):
        return len(self.order)

    def __iter__(self):
        return iter(list(self.order))

    def __contains__(self, user):
        return user in self.order

    def __getitem__(self, user):
        if user not in self.order:
            raise KeyError(user)
        row = self._rows()[user]
        # inner dict: ascending client index, without self (and without popped users)
        return {v: row[v] for v in sorted(self.order) if v != user}

    def pop(self, user):
        if user not in self.order:
            raise KeyError(user)
        row = self[user]
        self.order.remove(user)
        return row


def no_defense(users_grads, users_count, corrupted_count):
    if _is_torch_cuda(users_grads):
        from . import _device as dev
        return dev.mean(users_grads)
    out, _ = _host_call(DefenseTypes.NoDefense, _as_host_matrix(users_grads), users_count, corrupted_count)
    return out


def _host_sqdist(G: np.ndarray):
    """Squared-distance table (float64 [n, n] torch.cuda) of a host matrix, streamed in slabs (afl_sqdist_host):
    the table the host Krum call selects on."""
    import torch
    n, d = G.shape
    d2 = torch.empty((n, n), dtype=torch.float64, device="cuda")
    torch.cuda.current_stream().synchronize()        # the call writes d2 from its own stream
    nat.check(nat.lib().afl_sqdist_host(G.ctypes.data, n, d, G.strides[0] // 4, d2.data_ptr(), 0))
    return d2


def _krum_create_distances(users_grads):
    """Pairwise L2 distances of all clients as a DistanceTable (dense [n, n] fp32 on the GPU)."""
    from . import _device as dev
    if _is_torch_cuda(users_grads):
        d2 = dev.sqdist_partial(users_grads)
    else:
        d2 = _host_sqdist(_as_host_matrix(users_grads))
    return DistanceTable(dev.sqdist_to_dist(d2))


def _table_from_mapping(distances):
    """Accept a reference-style dict-of-dicts: returns (compact dense table, original user ids) with the
    compact index chosen so that the kernel's fixed visit order [1,0,2,...] equals the dict's key order."""
    import torch
    keys = list(distances.keys())
    m = len(keys)
    slot_of = {}
    for pos, u in enumerate(keys):
        slot_of[u] = (1 if pos == 0 else 0 if pos == 1 else pos) if m >= 2 else pos
    users = [None] * m
    for u, s in slot_of.items():
        users[s] = u
    table = np.zeros((m, m), np.float32)
    for u in keys:
        for v, val in distances[u].items():
            if v in slot_of:
                table[slot_of[u], slot_of[v]] = val
    return torch.from_numpy(table).cuda(), users


def krum(users_grads, users_count, corrupted_count, distances=None, return_index=False, debug=False):
    if not return_index:
        assert users_count >= 2 * corrupted_count + 1, ('users_count>=2*corrupted_count + 3', users_count, corrupted_count)
    if distances is None and not _is_torch_cuda(users_grads):
        G = _as_host_matrix(users_grads)
        if return_index:                                 # no assert, as in the reference: select on the same table
            from . import _device as dev
            return int(dev.krum_from_sqdist(_host_sqdist(G), users_count, corrupted_count).item())
        _, idx = _host_call(DefenseTypes.Krum, G, users_count, corrupted_count, want_out=False)
        return G[idx]
    from . import _device as dev
    users = None
    if distances is None:
        dense = dev.sqdist_to_dist(dev.sqdist_partial(users_grads))
    elif isinstance(distances, DistanceTable):
        if len(distances.order) == distances.dense.shape[0] and distances.order == DistanceTable(distances.dense).order:
            dense = distances.dense
        else:
            dense, users = _table_from_mapping(distances)
    else:
        dense, users = _table_from_mapping(distances)
    idx = int(dev.krum_select(dense, users_count, corrupted_count).item())
    if users is not None and idx >= 0:
        idx = users[idx]
    if return_index:
        return idx
    return users_grads[idx]


def trimmed_mean(users_grads, users_count, corrupted_count):
    if _is_torch_cuda(users_grads):
        from . import _device as dev
        return dev.trimmed_mean(users_grads, corrupted_count)
    out, _ = _host_call(DefenseTypes.TrimmedMean, _as_host_matrix(users_grads), users_count, corrupted_count)
    return out


def bulyan(users_grads, users_count, corrupted_count, return_selection=False):
    assert users_count >= 4 * corrupted_count + 3
    if _is_torch_cuda(users_grads):
        from . import _device as dev
        dist = dev.sqdist_to_dist(dev.sqdist_partial(users_grads))
        sel = dev.bulyan_select(dist, users_count, corrupted_count)
        out = dev.trimmed_mean(users_grads, 2 * corrupted_count, row_index=sel)
        if sel.numel() and int(sel[-1].item()) < 0:      # a failed round marks itself and all later rounds with -1
            raise KeyError(-1)                           # defences.py:66 `distances.pop(-1)`
        return (out, sel) if return_selection else out
    G = _as_host_matrix(users_grads)
    n, d = G.shape
    out = np.empty((d,), np.float32)
    sel = np.empty((users_count - 2 * corrupted_count,), np.int32)
    nat.check(nat.lib().afl_bulyan_host(G.ctypes.data, n, d, G.strides[0] // 4, int(users_count), int(corrupted_count),
                                        out.ctypes.data, sel.ctypes.data, 0))
    return (out, sel) if return_selection else out


defend = {DefenseTypes.Krum: krum,
          DefenseTypes.TrimmedMean: trimmed_mean, DefenseTypes.NoDefense: no_defense,
          DefenseTypes.Bulyan: bulyan}
