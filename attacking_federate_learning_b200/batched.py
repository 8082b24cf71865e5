"""Batched aggregation: B independent same-shape problems (a grid of runs over the attack strength, the
defence, the malicious share or the seed) through the defences of `defences.py` in one launch per kernel
stage instead of B Python-level calls.

Every problem keeps the reference's semantics exactly: problem b's result is what the single device call
(`defences.krum` / `bulyan` / `trimmed_mean` / `no_defense`, `malicious.Attack.attack_rows`) returns for
`G[b]`, bit for bit (C ABI `afl_defend_batched` / `afl_alie_batched`).

Inputs are torch.cuda float32 / bfloat16 / float16 tensors `[B, N, D]` with `stride(2) == 1` and N <= 128 clients (one
Gram tile); every problem shares N, D and `users_count`.  `corrupted_count` (and `alie_rows`' `num_std`) is
either one number for every problem or a host sequence of B values (list, tuple, NumPy array, CPU tensor), one
per problem (C ABI `afl_defend_batched_each` / `afl_alie_batched_each`), so that a grid over the malicious
share and z runs as one batch.  Nothing here synchronises the host except `bulyan`, which checks for a failed
selection round as `defences.bulyan` does.

`backdoor_rows` is the per-problem `BackdoorAttack.attack_rows`: the backdoor crafting of every problem in three
launches, with one call of the caller's malicious-network training between the second and the third.  It has no
client limit.

`attack_metrics` turns the batch's results into the sweep's attack-success table (SURVEY 8d) in one call: each
problem's distance from its honest mean, whether Krum picked a malicious client, and the malicious share of
Bulyan's selection.  It has no client limit.

The server's momentum step needs no batched form: `_device.momentum_step` on contiguous `[B, D]` weights,
velocity and gradients is already the batched step (server.py:89-90 is element-wise).
"""
from __future__ import annotations

import numpy as np
import torch

from . import _native as nat
from ._device import Workspace, _stream_ptr, dtype_code
from .defences import DefenseTypes


def _check(G: torch.Tensor):
    """(B, N, D, ld, batch_stride) of a [B, N, D] row-major CUDA tensor."""
    if not (isinstance(G, torch.Tensor) and G.is_cuda):
        raise TypeError("expected a torch.cuda tensor")
    if G.dim() != 3 or G.stride(2) != 1:
        raise ValueError("users_grads must be a [problems, clients, params] tensor with stride(2) == 1")
    B, N, D = G.shape
    ld = G.stride(1) if N > 1 else max(G.stride(1), D)
    return B, N, D, ld, G.stride(0)


def _per_problem(x, B: int, name: str, dtype):
    """None when x is one number for every problem, else its B per-problem values as a contiguous host array."""
    if isinstance(x, torch.Tensor):
        if x.dim() == 0:
            return None
        if x.is_cuda:
            raise TypeError(f"{name}: per-problem values must be on the host (reading a CUDA tensor would synchronise)")
        x = x.numpy()
    if np.ndim(x) == 0:
        return None
    a = np.asarray(x)
    if dtype == np.int32 and a.size and not np.issubdtype(a.dtype, np.integer):
        raise TypeError(f"{name}: per-problem counts must be integers (got {a.dtype})")
    if a.ndim != 1 or a.shape[0] != B:
        raise ValueError(f"{name}: expected one value per problem ({B}), got shape {a.shape}")
    return np.ascontiguousarray(a, dtype=dtype)


def _defend(rule: str, G: torch.Tensor, users_count: int, corrupted_count, out=None, idx=None, sel=None):
    B, N, D, ld, bs = _check(G)
    L = nat.lib()
    fs = _per_problem(corrupted_count, B, "corrupted_count", np.int32)
    with torch.cuda.device(G.device):
        if fs is not None:
            nbytes = L.afl_batched_each_workspace_bytes(rule.encode(), B, N, D, dtype_code(G))
            ws = Workspace.get(G.device, "batched", nbytes)
            nat.check(L.afl_defend_batched_each(rule.encode(), G.data_ptr(), B, bs, N, D, ld, dtype_code(G),
                                                int(users_count), fs.ctypes.data,
                                                None if out is None else out.data_ptr(),
                                                None if idx is None else idx.data_ptr(),
                                                None if sel is None else sel.data_ptr(), ws.data_ptr(), ws.numel(),
                                                _stream_ptr(G)))
            return
        nbytes = L.afl_batched_workspace_bytes(rule.encode(), B, N, D, dtype_code(G))
        ws = Workspace.get(G.device, "batched", nbytes) if nbytes else None
        nat.check(L.afl_defend_batched(rule.encode(), G.data_ptr(), B, bs, N, D, ld, dtype_code(G), int(users_count),
                                       int(corrupted_count), None if out is None else out.data_ptr(),
                                       None if idx is None else idx.data_ptr(), None if sel is None else sel.data_ptr(),
                                       None if ws is None else ws.data_ptr(), 0 if ws is None else ws.numel(),
                                       _stream_ptr(G)))


def krum(users_grads, users_count, corrupted_count, return_index=False):
    """Per problem defences.krum (corrupted_count: one int or B of them): the winning rows `G[arange(B), idx]`
    ([B, D], input dtype), or with return_index the device int32 [B] indices (-1 where no user is eligible).
    No host synchronisation."""
    B = users_grads.shape[0]
    idx = torch.empty(B, dtype=torch.int32, device=users_grads.device)
    _defend(DefenseTypes.Krum, users_grads, users_count, corrupted_count, idx=idx)
    if return_index:
        return idx
    return users_grads[torch.arange(B, device=users_grads.device), idx.long()]


def trimmed_mean(users_grads, users_count, corrupted_count):
    """Per problem defences.trimmed_mean: fp32 [B, D]."""
    B, _, D = users_grads.shape
    out = torch.empty((B, D), dtype=torch.float32, device=users_grads.device)
    _defend(DefenseTypes.TrimmedMean, users_grads, users_count, corrupted_count, out=out)
    return out


def no_defense(users_grads, users_count, corrupted_count):
    """Per problem defences.no_defense: fp32 [B, D]."""
    B, _, D = users_grads.shape
    out = torch.empty((B, D), dtype=torch.float32, device=users_grads.device)
    _defend(DefenseTypes.NoDefense, users_grads, users_count, corrupted_count, out=out)
    return out


def bulyan(users_grads, users_count, corrupted_count, return_selection=False):
    """Per problem defences.bulyan: fp32 [B, D] and, with return_selection, the int32 [B, theta] selections.
    With one corrupted_count per problem the selections are [B, theta_max], theta_max = users_count - 2 min(f):
    problem b's theta_b = users_count - 2 f_b rounds, then -2 ("no such round").  Raises KeyError(-1) when any
    problem's last round is -1 (a round found no eligible user), as `defences.bulyan` does for one problem."""
    B, _, D = users_grads.shape
    fs = _per_problem(corrupted_count, B, "corrupted_count", np.int32)
    if fs is None:
        assert users_count >= 4 * corrupted_count + 3
        theta = users_count - 2 * corrupted_count
    else:                                                # each problem's assert is checked by the call
        theta = max(users_count - 2 * int(fs.min()), 1) if B else 1
    out = torch.empty((B, D), dtype=torch.float32, device=users_grads.device)
    sel = torch.empty((B, theta), dtype=torch.int32, device=users_grads.device)
    _defend(DefenseTypes.Bulyan, users_grads, users_count, corrupted_count if fs is None else fs, out=out, sel=sel)
    if fs is None:
        last = sel[:, -1]
    else:
        last = sel.cpu()[torch.arange(B), torch.from_numpy(users_count - 2 * fs.astype(np.int64) - 1)]
    if bool((last < 0).any()):                           # defences.py:66 `distances.pop(-1)`
        raise KeyError(-1)
    return (out, sel) if return_selection else out


defend = {DefenseTypes.Krum: krum,
          DefenseTypes.TrimmedMean: trimmed_mean, DefenseTypes.NoDefense: no_defense,
          DefenseTypes.Bulyan: bulyan}


def alie_rows(users_grads, corrupted_count, num_std):
    """Per problem malicious.Attack.attack_rows (DriftAttack): the malicious users are rows 0..f-1 of every
    problem.  Returns (crafted, mu, sigma), each fp32 [B, D] (mu is the unperturbed mean), and writes crafted
    = mu - num_std * sigma into those rows in place (fp32 directly; bf16 and fp16 through a cast, as attack_rows does).
    With num_std == 0 the rows are left alone, as attack_rows does.  None when corrupted_count <= 0.

    corrupted_count and num_std may each be one number or B of them (host sequences).  Per problem, f_b <= N;
    f_b = 0 leaves the problem's rows alone and its crafted, mu and sigma are NaN; z_b = 0 computes the
    statistics (crafted = mu) and leaves the rows alone."""
    B = users_grads.shape[0]
    fs = _per_problem(corrupted_count, B, "corrupted_count", np.int32)
    zs = _per_problem(num_std, B, "num_std", np.float64)
    if fs is not None or zs is not None:
        return _alie_rows_each(users_grads, corrupted_count if fs is None else fs, num_std if zs is None else zs)
    f = int(corrupted_count)
    if f <= 0:
        return None
    B, _, D, ld, bs = _check(users_grads)
    dev = users_grads.device
    mu, sigma, crafted = (torch.empty((B, D), dtype=torch.float32, device=dev) for _ in range(3))
    write = num_std != 0
    bcast = users_grads if write and users_grads.dtype == torch.float32 else None
    with torch.cuda.device(dev):
        nat.check(nat.lib().afl_alie_batched(users_grads.data_ptr(), B, bs, f, D, ld, dtype_code(users_grads),
                                             float(num_std), mu.data_ptr(), sigma.data_ptr(), crafted.data_ptr(),
                                             None if bcast is None else bcast.data_ptr(), bs, ld,
                                             _stream_ptr(users_grads)))
    if write and bcast is None:
        users_grads[:, :f] = crafted[:, None, :].to(users_grads.dtype)
    return crafted, mu, sigma


def _alie_rows_each(users_grads, fs, zs):
    B, N, D, ld, bs = _check(users_grads)
    fs = np.ascontiguousarray(np.broadcast_to(np.asarray(fs, np.int32), (B,)))
    zs = np.ascontiguousarray(np.broadcast_to(np.asarray(zs, np.float64), (B,)))
    dev = users_grads.device
    mu, sigma, crafted = (torch.empty((B, D), dtype=torch.float32, device=dev) for _ in range(3))
    write = (fs > 0) & (zs != 0)
    bcast = users_grads if write.any() and users_grads.dtype == torch.float32 else None
    L = nat.lib()
    with torch.cuda.device(dev):
        nbytes = L.afl_batched_each_workspace_bytes(b"ALIE", B, N, D, dtype_code(users_grads))
        ws = Workspace.get(dev, "batched_alie", nbytes)
        nat.check(L.afl_alie_batched_each(users_grads.data_ptr(), B, bs, N, D, ld, dtype_code(users_grads),
                                          fs.ctypes.data, zs.ctypes.data, mu.data_ptr(), sigma.data_ptr(),
                                          crafted.data_ptr(), None if bcast is None else bcast.data_ptr(), bs, ld,
                                          ws.data_ptr(), ws.numel(), _stream_ptr(users_grads)))
    if write.any() and bcast is None:
        _cast_rows(users_grads, crafted, fs, write)
    return crafted, mu, sigma


def _cast_rows(users_grads, crafted, fs, write):
    """bf16 / fp16 matrices: crafted[b] over rows r < f_b of the problems that write, via a cast."""
    N = users_grads.shape[1]
    b_idx, r_idx = np.nonzero(write[:, None] & (np.arange(N)[None, :] < fs[:, None]))
    b_idx, r_idx = (torch.from_numpy(x).pin_memory().to(users_grads.device, non_blocking=True) for x in (b_idx, r_idx))
    users_grads[b_idx, r_idx] = crafted[b_idx].to(users_grads.dtype)


def backdoor_rows(users_grads, corrupted_count, num_std, original_params, learning_rate, train_malicious_network):
    """Per problem malicious.BackdoorAttack.attack_rows (backdoor.py:52-63): the malicious users are rows 0..f_b-1 of
    problem b.  Returns (crafted, mu, sigma), each fp32 [B, D] (mu is the malicious rows' mean), and writes crafted into
    those rows in place (fp32 directly; bf16 and fp16 through a cast).  Any number of clients.

    corrupted_count, num_std and learning_rate are each one number or B host values (as `alie_rows`), f_b <= N.
    original_params: fp32 CUDA [D] (shared by every problem) or [B, D].  The crafting runs on the device, with one
    call of `train_malicious_network(initial, problems)` in the middle (backdoor.py:56): `problems` is the host list of
    the k problems that attack (f_b > 0 and z_b != 0), in order, `initial` their fp32 [k, D] starting parameters
    w_b - lr_b * mu_b, and it returns their trained parameters as a fp32 CUDA [k, D] tensor.  With no such problem it
    is not called.  f_b = 0 gives NaN crafted, mu and sigma; z_b = 0 the statistics only (crafted = mu); neither
    writes a row.  Nothing here synchronises the host."""
    if not (isinstance(original_params, torch.Tensor) and original_params.is_cuda):
        raise TypeError("original_params: expected a torch.cuda float32 tensor of shape [D] or [B, D]")
    B, N, D, ld, bs = _check(users_grads)
    dev = users_grads.device
    if original_params.dtype != torch.float32 or original_params.device != dev or \
            tuple(original_params.shape) not in ((D,), (B, D)):
        raise ValueError(f"original_params: expected a float32 tensor of shape ({D},) or ({B}, {D}) on {dev}")
    w = original_params.contiguous()

    def per_problem(x, name, dtype):
        a = _per_problem(x, B, name, dtype)
        return np.full(B, int(x) if dtype == np.int32 else float(x), dtype) if a is None else a
    fs = per_problem(corrupted_count, "corrupted_count", np.int32)
    zs = per_problem(num_std, "num_std", np.float64)
    lrs = per_problem(learning_rate, "learning_rate", np.float64)
    mu, sigma, initial, crafted = (torch.empty((B, D), dtype=torch.float32, device=dev) for _ in range(4))
    L = nat.lib()
    code = dtype_code(users_grads)
    stream = _stream_ptr(users_grads)
    with torch.cuda.device(dev):
        ws = Workspace.get(dev, "backdoor", L.afl_batched_each_workspace_bytes(b"ALIE", B, 1, D, code))   # the table
        nat.check(L.afl_backdoor_start_batched(users_grads.data_ptr(), B, bs, N, D, ld, code, fs.ctypes.data,
                                               zs.ctypes.data, lrs.ctypes.data, w.data_ptr(),
                                               w.stride(0) if w.dim() == 2 else 0, mu.data_ptr(), sigma.data_ptr(),
                                               initial.data_ptr(), ws.data_ptr(), ws.numel(), stream))
    write = (fs > 0) & (zs != 0)
    problems = np.flatnonzero(write).tolist()
    mal = initial                                        # read for the problems that attack only
    if problems:
        k = len(problems)
        sel = None if k == B else torch.as_tensor(problems, device=dev)
        out = train_malicious_network(initial if sel is None else initial[sel], problems)
        if not (isinstance(out, torch.Tensor) and out.device == dev and out.dtype == torch.float32
                and tuple(out.shape) == (k, D)):
            raise ValueError(f"train_malicious_network must return a float32 tensor of shape ({k}, {D}) on {dev}")
        if sel is None:
            mal = out.contiguous()
        else:
            mal = torch.empty((B, D), dtype=torch.float32, device=dev)
            mal[sel] = out
    bcast = users_grads if problems and users_grads.dtype == torch.float32 else None
    with torch.cuda.device(dev):
        nat.check(L.afl_backdoor_finish_batched(B, D, fs.ctypes.data, zs.ctypes.data, lrs.ctypes.data, mu.data_ptr(),
                                                sigma.data_ptr(), initial.data_ptr(), mal.data_ptr(), mal.stride(0),
                                                crafted.data_ptr(), None if bcast is None else bcast.data_ptr(), bs,
                                                ld, ws.data_ptr(), ws.numel(), stream))
    if problems and bcast is None:
        _cast_rows(users_grads, crafted, fs, write)
    return crafted, mu, sigma


def attack_metrics(users_grads, corrupted_count, *, aggregated=None, krum_index=None, selection=None,
                   return_honest_mean=False):
    """Attack-success figures of every problem (C ABI `afl_attack_metrics_batched` / `_each`), as a dict of device
    tensors.  The malicious users are rows 0..f_b-1 (main.py:28); corrupted_count is one int or B host values.

    * aggregated (fp32 [B, D]: Bulyan's, the trimmed mean's or the mean's output) or krum_index (int32 [B], what
      `krum(..., return_index=True)` returns; the winning rows are read in place) gives `rel_deviation` [B] fp32 =
      ||a_b - h_b|| / ||h_b|| with h_b the mean of rows f_b..N-1 (`no_defense(G[b, f_b:])` bit for bit), and
      `deviation_sums` [B, 2] float64, the two sums of squares, which add across column shards.  At most one of the two.
    * krum_index also gives `krum_success` [B] bool (metrics.krum_attack_success per problem).
    * selection (int32 [B, theta], what `bulyan(..., return_selection=True)` returns; -1 and -2 entries are not
      counted) gives `bulyan_malicious_fraction` [B] fp32 (metrics.bulyan_attack_success per problem).
    * return_honest_mean adds `honest_mean` [B, D] fp32.

    f_b >= N (no honest row) and krum_index -1 give NaN deviations.  No host synchronisation.  One problem: pass
    `G[None]`."""
    fs = _per_problem(corrupted_count, users_grads.shape[0], "corrupted_count", np.int32)
    B, N, D, ld, bs = _check(users_grads)
    dev = users_grads.device

    def arg(t, name, dtype, shape):
        if t is None:
            return None
        if not (isinstance(t, torch.Tensor) and t.device == dev and t.dtype == dtype and t.dim() == len(shape)
                and all(s == (w or s) for s, w in zip(t.shape, shape))):
            raise ValueError(f"{name}: expected a {dtype} tensor of shape {shape} on {dev}")
        return t.contiguous()
    if aggregated is not None and krum_index is not None:
        raise ValueError("attack_metrics: give the aggregate as `aggregated` or as `krum_index`, not both")
    agg = arg(aggregated, "aggregated", torch.float32, (B, D))
    idx = arg(krum_index, "krum_index", torch.int32, (B,))
    sel = arg(selection, "selection", torch.int32, (B, None))       # any number of rounds

    def out(when, shape, dtype):
        return torch.empty(shape, dtype=dtype, device=dev) if when else None
    have_agg = agg is not None or idx is not None
    rel, sums = out(have_agg, (B,), torch.float32), out(have_agg, (B, 2), torch.float64)
    honest = out(return_honest_mean, (B, D), torch.float32)
    hit = out(idx is not None, (B,), torch.int32)
    mal, cnt = out(sel is not None, (B,), torch.int32), out(sel is not None, (B,), torch.int32)
    ptrs = [None if t is None else t.data_ptr() for t in (agg, idx, sel, rel, sums, honest, hit, mal, cnt)]
    L = nat.lib()
    code = dtype_code(users_grads)
    with torch.cuda.device(dev):
        ws = Workspace.get(dev, "metrics", L.afl_metrics_workspace_bytes(B, N, D, code))
        call, f = (L.afl_attack_metrics_batched, int(corrupted_count)) if fs is None else \
            (L.afl_attack_metrics_batched_each, fs.ctypes.data)
        nat.check(call(users_grads.data_ptr(), B, bs, N, D, ld, code, f, *ptrs[:3], 0 if sel is None else sel.shape[1],
                       *ptrs[3:], ws.data_ptr(), ws.numel(), _stream_ptr(users_grads)))
    res = {}
    if have_agg:
        res["rel_deviation"], res["deviation_sums"] = rel, sums
    if hit is not None:
        res["krum_success"] = hit.bool()
    if sel is not None:
        res["bulyan_malicious_fraction"] = mal.float() / cnt.clamp(min=1).float()
    if honest is not None:
        res["honest_mean"] = honest
    return res
