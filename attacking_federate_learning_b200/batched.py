"""Batched aggregation: B independent same-shape problems (a grid of runs over the attack strength, the
defence, the malicious share or the seed) through the defences of `defences.py` in one launch per kernel
stage instead of B Python-level calls.

Every problem keeps the reference's semantics exactly: problem b's result is what the single device call
(`defences.krum` / `bulyan` / `trimmed_mean` / `no_defense`, `malicious.Attack.attack_rows`) returns for
`G[b]`, bit for bit (C ABI `afl_defend_batched` / `afl_alie_batched`).

Inputs are torch.cuda float32 / bfloat16 / float16 tensors `[B, N, D]` with `stride(2) == 1` and N <= 1024 clients;
every problem shares N, D and `users_count`.  `corrupted_count` (and `alie_rows`' `num_std`) is
either one number for every problem or a host sequence of B values (list, tuple, NumPy array, CPU tensor), one
per problem (C ABI `afl_defend_batched_each` / `afl_alie_batched_each`), so that a grid over the malicious
share and z runs as one batch.  Nothing here synchronises the host except `bulyan`, which checks for a failed
selection round as `defences.bulyan` does.

Every defence and `attack_metrics` also take `rows=` (B host ints, 1 <= rows_b <= N): a ragged batch, where problem b
is `G[b, :rows_b]` and rows rows_b..N-1 are padding that no result depends on (C ABI `afl_defend_batched_rows` /
`afl_attack_metrics_batched_rows`).  So a grid over the number of users (main.py:118), or rounds in which a different
number of clients reports, runs as one batch; `users_count` may then be B values too and defaults to `rows`, the
`len(self.users)` that `Server.defend` passes (server.py:87).

N <= 128 (one Gram tile) runs the calls above.  128 < N <= 1024 (the N = 500 and N = 1000 runs, f = 240 at N = 1000)
runs `afl_defend_batched_large`, the ragged call with the larger limit: without `rows`, every problem has N rows and
scalar counts apply to every problem.  Results and return shapes are the same as at N <= 128; every problem's trimmed
mean runs the kernel its own row count selects.  N > 1024 raises NotImplementedError.  `alie_rows` takes any N: a
scalar f > 128, or per-problem counts with N > 128, run `afl_alie_batched_large`.

`backdoor_rows` is the per-problem `BackdoorAttack.attack_rows`: the backdoor crafting of every problem in three
launches, with one call of the caller's malicious-network training between the second and the third.  It has no
client limit.

`attack_metrics` turns the batch's results into the sweep's attack-success table (SURVEY 8d) in one call: each
problem's distance from its honest mean, whether Krum picked a malicious client, and the malicious share of
Bulyan's selection.  It has no client limit.

`DeviceRound` runs the same calls with `f`, `z`, `rows` and `users_count` held as device tensors that the caller
refills in place (C ABI `afl_*_dev`): its methods never synchronise, so after one eager warm-up a whole round can be
captured with `torch.cuda.graph` and replayed.  Per-problem checks run on the device and land in `DeviceRound.status`;
`raise_for_status` raises what the host-parameter call would.  Its defences take N <= 128, or N <= 1024 with
`large=True` (C ABI `afl_defend_batched_large_dev`, which groups the problems by trimmed-mean slot class on the
device), so the N = 500 and N = 1000 sweeps run as captured rounds too.  The functions above do not change and keep
refusing CUDA tensors for their per-problem values.

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


def _full(x, B: int, name: str):
    """B per-problem int32 host values of x (one number or B of them)."""
    a = _per_problem(x, B, name, np.int32)
    return np.full(B, int(x), np.int32) if a is None else a


def _ragged(B: int, rows, users_count, corrupted_count):
    """(rows, users_count, corrupted_count) of a ragged batch as int32 host arrays; users_count defaults to rows."""
    rs = _full(rows, B, "rows")
    return rs, (rs if users_count is None else _full(users_count, B, "users_count")), \
        _full(corrupted_count, B, "corrupted_count")


MAX_CLIENTS = 1024          # clients per problem of the batched defences (afl_defend_batched_large)
ONE_TILE = 128              # the calls for one Gram tile (afl_defend_batched, _each, _rows)


def _defend(rule: str, G: torch.Tensor, users_count: int, corrupted_count, out=None, idx=None, sel=None, rows=None):
    B, N, D, ld, bs = _check(G)
    if N > MAX_CLIENTS:
        raise NotImplementedError(f"batched defences support N <= {MAX_CLIENTS} clients per problem (got {N})")
    L = nat.lib()
    if rows is not None or N > ONE_TILE:
        rs, ucs, fs = _ragged(B, N if rows is None else rows, users_count, corrupted_count)
        ws_bytes, call = ((L.afl_batched_rows_workspace_bytes, L.afl_defend_batched_rows) if N <= ONE_TILE
                          else (L.afl_batched_large_workspace_bytes, L.afl_defend_batched_large))
        with torch.cuda.device(G.device):
            ws = Workspace.get(G.device, "batched", ws_bytes(rule.encode(), B, N, D, dtype_code(G)))
            nat.check(call(rule.encode(), G.data_ptr(), B, bs, N, D, ld, dtype_code(G),
                           rs.ctypes.data, ucs.ctypes.data, fs.ctypes.data,
                           None if out is None else out.data_ptr(),
                           None if idx is None else idx.data_ptr(),
                           None if sel is None else sel.data_ptr(), ws.data_ptr(), ws.numel(),
                           _stream_ptr(G)))
        return
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


def krum(users_grads, users_count, corrupted_count, return_index=False, *, rows=None):
    """Per problem defences.krum (corrupted_count: one int or B of them): the winning rows `G[arange(B), idx]`
    ([B, D], input dtype), or with return_index the device int32 [B] indices (-1 where no user is eligible).
    With rows, problem b is G[b, :rows_b] and index -1 returns its row rows_b - 1 (the reference's users_grads[-1]).
    No host synchronisation."""
    B = users_grads.shape[0]
    dev = users_grads.device
    idx = torch.empty(B, dtype=torch.int32, device=dev)
    _defend(DefenseTypes.Krum, users_grads, users_count, corrupted_count, idx=idx, rows=rows)
    if return_index:
        return idx
    row = idx.long()
    if rows is not None:
        last = torch.from_numpy(_full(rows, B, "rows").astype(np.int64) - 1).pin_memory().to(dev, non_blocking=True)
        row = torch.where(row < 0, last, row)
    return users_grads[torch.arange(B, device=dev), row]


def trimmed_mean(users_grads, users_count, corrupted_count, *, rows=None):
    """Per problem defences.trimmed_mean: fp32 [B, D].  With rows, over G[b, :rows_b]."""
    B, _, D = users_grads.shape
    out = torch.empty((B, D), dtype=torch.float32, device=users_grads.device)
    _defend(DefenseTypes.TrimmedMean, users_grads, users_count, corrupted_count, out=out, rows=rows)
    return out


def no_defense(users_grads, users_count, corrupted_count, *, rows=None):
    """Per problem defences.no_defense: fp32 [B, D].  With rows, the mean of G[b, :rows_b]."""
    B, _, D = users_grads.shape
    out = torch.empty((B, D), dtype=torch.float32, device=users_grads.device)
    _defend(DefenseTypes.NoDefense, users_grads, users_count, corrupted_count, out=out, rows=rows)
    return out


def bulyan(users_grads, users_count, corrupted_count, return_selection=False, *, rows=None):
    """Per problem defences.bulyan: fp32 [B, D] and, with return_selection, the int32 [B, theta] selections.
    With one corrupted_count per problem the selections are [B, theta_max], theta_max = users_count - 2 min(f):
    problem b's theta_b = users_count - 2 f_b rounds, then -2 ("no such round").  Raises KeyError(-1) when any
    problem's last round is -1 (a round found no eligible user), as `defences.bulyan` does for one problem.
    With rows, problem b is G[b, :rows_b] with users_count_b == rows_b, and theta_max = max_b(users_count_b - 2 f_b)."""
    B, _, D = users_grads.shape
    if rows is not None:
        rs, ucs, fs = _ragged(B, rows, users_count, corrupted_count)
        theta = ucs.astype(np.int64) - 2 * fs
        out = torch.empty((B, D), dtype=torch.float32, device=users_grads.device)
        sel = torch.empty((B, max(int(theta.max()), 1) if B else 1), dtype=torch.int32, device=users_grads.device)
        _defend(DefenseTypes.Bulyan, users_grads, ucs, fs, out=out, sel=sel, rows=rs)
        if bool((sel.cpu()[torch.arange(B), torch.from_numpy(theta - 1)] < 0).any()):   # defences.py:66
            raise KeyError(-1)
        return (out, sel) if return_selection else out
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
    problem.  A ragged batch (rows_b clients in problem b, as the defences' `rows=`) needs no extra argument: the
    attack reads and writes rows 0..f_b-1 only, so f_b <= rows_b is all it asks.  Returns (crafted, mu, sigma), each fp32 [B, D] (mu is the unperturbed mean), and writes crafted
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
    if f > ONE_TILE:                                     # afl_alie_batched takes f-row problems of one tile
        return _alie_rows_each(users_grads, f, num_std)
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
    call = L.afl_alie_batched_each if N <= ONE_TILE else L.afl_alie_batched_large
    with torch.cuda.device(dev):
        nbytes = L.afl_batched_each_workspace_bytes(b"ALIE", B, min(N, ONE_TILE), D, dtype_code(users_grads))
        ws = Workspace.get(dev, "batched_alie", nbytes)
        nat.check(call(users_grads.data_ptr(), B, bs, N, D, ld, dtype_code(users_grads),
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
    problem b (which is all a ragged batch needs: no `rows` argument, f_b <= rows_b).  Returns (crafted, mu, sigma), each fp32 [B, D] (mu is the malicious rows' mean), and writes crafted into
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
                   return_honest_mean=False, rows=None):
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
    `G[None]`.  rows (B host ints, C ABI `afl_attack_metrics_batched_rows`): a ragged batch, problem b being
    G[b, :rows_b], so its honest rows are f_b..rows_b-1."""
    fs = _per_problem(corrupted_count, users_grads.shape[0], "corrupted_count", np.int32)
    if rows is not None:
        rs, _, fs = _ragged(users_grads.shape[0], rows, None, corrupted_count)
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
        if rows is not None:
            call, f = (lambda *a: L.afl_attack_metrics_batched_rows(*a[:7], rs.ctypes.data, *a[7:])), fs.ctypes.data
        elif fs is None:
            call, f = L.afl_attack_metrics_batched, int(corrupted_count)
        else:
            call, f = L.afl_attack_metrics_batched_each, fs.ctypes.data
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


_STATUS_ERRORS = {nat.AFL_ERR_BAD_ARG: (ValueError, "a corrupted count or row count is out of range"),
                  nat.AFL_ERR_PRECONDITION: (AssertionError, "the reference's assert users_count >= 2*corrupted_count"
                                             " + 1 (Krum) or >= 4*corrupted_count + 3 (Bulyan) is violated"),
                  nat.AFL_ERR_UNSUPPORTED: (NotImplementedError, "Bulyan's users_count must equal its number of rows")}


def krum_gather_rows(idx, rows, N):
    """The row DeviceRound.krum gathers per problem (int64, same device as idx): idx_b for an index >= 0, and for
    -1 (no eligible user) the last row the problem ran with, rows_b - 1 when rows_b lies in [1, N] and N - 1 otherwise
    (the safe row of a problem flagged for its row count).  rows: int32 [B] or None (N rows in every problem).  For
    kernel indices in [-1, N) the result is in [0, N) whatever int32 rows holds."""
    idx = idx.long()
    if rows is None:
        last = N - 1
    else:
        rows = rows.long()
        last = torch.where((rows >= 1) & (rows <= N), rows - 1, N - 1)
    return torch.where(idx < 0, last, idx)


class DeviceRound:
    """One lock-step round of a batch whose per-problem parameters live on the device (C ABI `afl_*_dev`).

    The module-level functions take corrupted counts, strengths, row counts and users counts as host values and refuse
    CUDA tensors, since reading one would synchronise.  A DeviceRound holds them as device tensors instead, which the
    caller refills in place between rounds: `f` (int32 [B]), `z` (float64 [B]), `rows` (int32 [B], with rows=True) and
    `users_count` (int32 [B], with rows=True and per_problem_users_count=True; otherwise it follows `rows`).  `G` is the
    caller's [B, N, D] client tensor, also refilled in place.  Every method only enqueues work on the current stream
    into outputs and a workspace sized once here (attack_metrics' small outputs are allocated per call, which a
    captured graph serves from its own pool), so after one eager warm-up a whole round (your own training, then
    `alie`, a defence, `attack_metrics` and `_device.momentum_step`) can be captured with `torch.cuda.graph` and
    replayed.  Each method's result is the host-parameter call's on the same values, bit for bit.

    `lr` (float64 [B]) is the backdoor crafting's per-problem client learning rate: `backdoor_start` and
    `backdoor_finish` are `backdoor_rows` around the caller's training of the malicious networks (in a sweep,
    `afl_mnist_backdoor_train`), with f, z and lr read on the device.

    Per-problem checks run on the device.  A problem that fails one gets its first error code in `status` (int32 [B],
    sticky until `clear_status`) and runs on a safe row (rows_b = N, users_count_b = N, f_b = 0), so its outputs are
    not the reference's; `raise_for_status` (the one call that synchronises) raises what the host-parameter call would:
    ValueError, AssertionError, NotImplementedError, or KeyError(-1) for a Bulyan round with no eligible user.

    users_count: one int for every problem without rows (default N).  rules: the defences this round runs (their
    workspace is sized here); any of them needs N <= 128, or N <= 1024 with large=True.  large=True runs the defences
    through `afl_defend_batched_large_dev` (at N <= 128 the same call as without it); each result is then the
    host-parameter call's (`afl_defend_batched_large` above 128 clients) bit for bit."""

    def __init__(self, users_grads, users_count=None, *, rows=False, per_problem_users_count=False,
                 rules=(DefenseTypes.Krum, DefenseTypes.Bulyan, DefenseTypes.TrimmedMean, DefenseTypes.NoDefense),
                 large=False):
        if not isinstance(users_grads, torch.Tensor):
            raise TypeError("users_grads: expected a torch.cuda tensor")
        if users_grads.dim() != 3 or users_grads.stride(2) != 1:
            raise ValueError("users_grads must be a [problems, clients, params] tensor with stride(2) == 1")
        B, N, D = users_grads.shape
        rules = tuple(rules)
        for r in rules:
            if r not in defend:
                raise ValueError(f"DeviceRound: unknown rule {r!r}")
        limit = MAX_CLIENTS if large else ONE_TILE
        if rules and N > limit:
            hint = "" if large else f"; large=True takes up to {MAX_CLIENTS}"
            raise NotImplementedError(f"DeviceRound defences support N <= {limit} clients per problem (got {N}){hint}")
        if per_problem_users_count and not rows:
            raise ValueError("DeviceRound: per-problem users counts need rows=True")
        if rows and users_count is not None:
            raise ValueError("DeviceRound: with rows, users_count follows rows or is per problem")
        if B < 1 or N < 1 or D < 1:
            raise ValueError(f"DeviceRound: empty batch {tuple(users_grads.shape)}")
        code = dtype_code(users_grads)
        if not users_grads.is_cuda:
            raise TypeError("users_grads: expected a torch.cuda tensor")
        _, _, _, self._ld, self._bs = _check(users_grads)
        self.G, self.B, self.N, self.D, self._code, self.rules, self.large = users_grads, B, N, D, code, rules, large
        self.users_count_scalar = N if users_count is None else int(users_count)
        dev = self.device = users_grads.device
        self.f = torch.zeros(B, dtype=torch.int32, device=dev)
        self.z = torch.zeros(B, dtype=torch.float64, device=dev)
        self.rows = torch.full((B,), N, dtype=torch.int32, device=dev) if rows else None
        self.users_count = torch.full((B,), N, dtype=torch.int32, device=dev) if per_problem_users_count else None
        self.lr = torch.zeros(B, dtype=torch.float64, device=dev)
        self.status = torch.zeros(B, dtype=torch.int32, device=dev)
        L = nat.lib()
        rule_bytes = L.afl_batched_large_dev_workspace_bytes if large else L.afl_batched_rows_workspace_bytes
        nbytes = max([rule_bytes(r.encode(), B, N, D, code) for r in rules] +
                     [L.afl_batched_each_workspace_bytes(b"ALIE", B, 1, D, code),
                      L.afl_metrics_workspace_bytes(B, N, D, code)])
        self._ws = torch.empty(nbytes, dtype=torch.uint8, device=dev)     # one round's calls run in stream order
        f32 = dict(dtype=torch.float32, device=dev)
        self.mu, self.sigma, self.crafted = (torch.empty((B, D), **f32) for _ in range(3))
        self.out = {r: torch.empty((B, D), **f32) for r in rules if r != DefenseTypes.Krum}
        self.krum_index = torch.empty(B, dtype=torch.int32, device=dev)
        self.krum_rows = torch.empty((B, D), dtype=users_grads.dtype, device=dev)
        self.selection = torch.empty((B, N), dtype=torch.int32, device=dev)
        self._problems = torch.arange(B, dtype=torch.int64, device=dev)
        self.initial = None                              # backdoor_start's [B, D], allocated by its first call
        self._initial_used = None                        # the initial the last backdoor_start wrote
        self._trace_ws = None                            # attack_trace's workspace, allocated by its first call

    @staticmethod
    def _ptr(t):
        return None if t is None else t.data_ptr()

    def _call(self, fn, *args):
        with torch.cuda.device(self.device):
            nat.check(fn(*args))

    def _defend(self, rule, out=None, idx=None, sel=None):
        if rule not in self.rules:
            raise ValueError(f"DeviceRound: {rule} was not among the rules given at construction")
        L = nat.lib()
        call = L.afl_defend_batched_large_dev if self.large else L.afl_defend_batched_dev
        self._call(call, rule.encode(), self.G.data_ptr(), self.B, self._bs, self.N, self.D,
                   self._ld, self._code, self._ptr(self.rows), self.users_count_scalar, self._ptr(self.users_count),
                   self.f.data_ptr(), self._ptr(out), self._ptr(idx), self._ptr(sel), self.N, self._ws.data_ptr(),
                   self._ws.numel(), self.status.data_ptr(), _stream_ptr(self.G))

    def alie(self):
        """alie_rows with the device f and z: returns (crafted, mu, sigma), fp32 [B, D], and writes crafted over rows
        0..f_b-1 of the problems with f_b > 0 and z_b != 0, in G's dtype (bf16 and fp16 rounded to nearest even)."""
        self._call(nat.lib().afl_alie_batched_dev, self.G.data_ptr(), self.B, self._bs, self.N, self.D, self._ld,
                   self._code, self.f.data_ptr(), self.z.data_ptr(), self.mu.data_ptr(), self.sigma.data_ptr(),
                   self.crafted.data_ptr(), self.G.data_ptr(), self._bs, self._ld, self._ws.data_ptr(), self._ws.numel(),
                   self.status.data_ptr(), _stream_ptr(self.G))
        return self.crafted, self.mu, self.sigma

    def backdoor_start(self, original_params, initial=None):
        """`backdoor_rows` up to the training, with the device f, z and lr (float64 [B]): returns (mu, sigma, initial),
        fp32 [B, D], initial_b = w_b - lr_b * mu_b (w: original_params, fp32 CUDA [D] or [B, D]).  `initial` (fp32 [B, D],
        contiguous) receives it when given; otherwise `self.initial` does.  A problem with f_b < 0 or f_b > N is flagged
        (ValueError) and runs with f_b = 0.  The problems that attack, f_b > 0 and z_b != 0 with a clear status, are
        the ones `afl_mnist_backdoor_train` trains."""
        w = original_params
        if not (isinstance(w, torch.Tensor) and w.device == self.device and w.dtype == torch.float32
                and tuple(w.shape) in ((self.D,), (self.B, self.D)) and w.stride(-1) == 1
                and (w.dim() == 1 or w.stride(0) >= self.D)):
            raise ValueError(f"original_params: expected a float32 tensor of shape ({self.D},) or ({self.B}, {self.D}) "
                             f"with unit column stride on {self.device}")
        if initial is None:
            if self.initial is None:
                self.initial = torch.empty((self.B, self.D), dtype=torch.float32, device=self.device)
            initial = self.initial
        elif not (initial.device == self.device and initial.dtype == torch.float32 and initial.is_contiguous()
                  and tuple(initial.shape) == (self.B, self.D)):
            raise ValueError(f"initial: expected a contiguous float32 tensor of shape ({self.B}, {self.D})")
        self._call(nat.lib().afl_backdoor_start_batched_dev, self.G.data_ptr(), self.B, self._bs, self.N, self.D,
                   self._ld, self._code, self.f.data_ptr(), self.z.data_ptr(), self.lr.data_ptr(), w.data_ptr(),
                   w.stride(0) if w.dim() == 2 else 0, self.mu.data_ptr(), self.sigma.data_ptr(), initial.data_ptr(),
                   self._ws.data_ptr(), self._ws.numel(), self.status.data_ptr(), _stream_ptr(self.G))
        self._initial_used = initial
        return self.mu, self.sigma, initial

    def backdoor_finish(self, mal):
        """`backdoor_rows` after the training: returns crafted (fp32 [B, D]) from the last backdoor_start's mu, sigma
        and initial and the trained parameters `mal` (fp32 [B, D], rows read only for the problems that attack), and
        writes it over rows 0..f_b-1 of those problems.  Takes the f, z and lr backdoor_start took.  fp32 client
        matrices only (a 16-bit one needs the host-parameter `backdoor_rows`)."""
        if self._initial_used is None:
            raise RuntimeError("DeviceRound.backdoor_finish: call backdoor_start first")
        if self.G.dtype != torch.float32:
            raise TypeError("DeviceRound.backdoor_finish writes fp32 client matrices only")
        if not (isinstance(mal, torch.Tensor) and mal.device == self.device and mal.dtype == torch.float32
                and tuple(mal.shape) == (self.B, self.D) and mal.stride(1) == 1
                and (self.B == 1 or mal.stride(0) >= self.D)):
            raise ValueError(f"mal: expected a float32 tensor of shape ({self.B}, {self.D}) on {self.device}")
        self._call(nat.lib().afl_backdoor_finish_batched_dev, self.B, self.N, self.D, self.f.data_ptr(),
                   self.z.data_ptr(), self.lr.data_ptr(), self.mu.data_ptr(), self.sigma.data_ptr(),
                   self._initial_used.data_ptr(), mal.data_ptr(), mal.stride(0), self.crafted.data_ptr(),
                   self.G.data_ptr(), self._bs, self._ld, self._ws.data_ptr(), self._ws.numel(), self.status.data_ptr(),
                   _stream_ptr(self.G))
        return self.crafted

    def krum(self, return_index=False):
        """`krum`: the device int32 [B] indices, or the winning rows [B, D] in G's dtype.  Index -1 (no eligible user)
        selects the last row the problem ran with, the reference's users_grads[-1]: row rows_b - 1 (N - 1 without
        rows), and N - 1 for a problem whose rows_b lies outside [1, N], which ran on the safe row (see
        `krum_gather_rows`)."""
        self._defend(DefenseTypes.Krum, idx=self.krum_index)
        if return_index:
            return self.krum_index
        self.krum_rows.copy_(self.G[self._problems, krum_gather_rows(self.krum_index, self.rows, self.N)])
        return self.krum_rows

    def bulyan(self, return_selection=False):
        """`bulyan`: fp32 [B, D] and, with return_selection, the int32 [B, N] selections (theta_b rounds, then -2; -1
        from a failed round on).  A failed round flags its problem with KeyError(-1) in `status`."""
        out = self.out[DefenseTypes.Bulyan] if DefenseTypes.Bulyan in self.out else None
        self._defend(DefenseTypes.Bulyan, out=out, sel=self.selection)
        return (out, self.selection) if return_selection else out

    def trimmed_mean(self):
        """`trimmed_mean`: fp32 [B, D]."""
        out = self.out.get(DefenseTypes.TrimmedMean)
        self._defend(DefenseTypes.TrimmedMean, out=out)
        return out

    def no_defense(self):
        """`no_defense`: fp32 [B, D]."""
        out = self.out.get(DefenseTypes.NoDefense)
        self._defend(DefenseTypes.NoDefense, out=out)
        return out

    def attack_metrics(self, *, aggregated=None, krum_index=None, selection=None, return_honest_mean=False):
        """`attack_metrics` with the device f (and rows): the same dict of device tensors."""
        if aggregated is not None and krum_index is not None:
            raise ValueError("attack_metrics: give the aggregate as `aggregated` or as `krum_index`, not both")
        for t, name, dtype, shape in ((aggregated, "aggregated", torch.float32, (self.B, self.D)),
                                      (krum_index, "krum_index", torch.int32, (self.B,)),
                                      (selection, "selection", torch.int32, None)):
            if t is not None and not (isinstance(t, torch.Tensor) and t.device == self.device and t.dtype == dtype
                                      and t.is_contiguous() and (t.shape == shape if shape else
                                                                 (t.dim() == 2 and t.shape[0] == self.B))):
                raise ValueError(f"{name}: expected a contiguous {dtype} tensor for {self.B} problems on {self.device}")
        def out(when, shape, dtype):                     # fresh outputs: two calls in one round keep both results
            return torch.empty(shape, dtype=dtype, device=self.device) if when else None
        have_agg = aggregated is not None or krum_index is not None
        rel, sums = out(have_agg, (self.B,), torch.float32), out(have_agg, (self.B, 2), torch.float64)
        honest = out(return_honest_mean, (self.B, self.D), torch.float32)
        hit = out(krum_index is not None, (self.B,), torch.int32)
        mal, cnt = (out(selection is not None, (self.B,), torch.int32) for _ in range(2))
        self._call(nat.lib().afl_attack_metrics_batched_dev, self.G.data_ptr(), self.B, self._bs, self.N, self.D,
                   self._ld, self._code, self._ptr(self.rows), self.f.data_ptr(), self._ptr(aggregated),
                   self._ptr(krum_index), self._ptr(selection), 0 if selection is None else selection.shape[1],
                   *(self._ptr(t) for t in (rel, sums, honest, hit, mal, cnt)), self._ws.data_ptr(), self._ws.numel(),
                   self.status.data_ptr(), _stream_ptr(self.G))
        res = {}
        if have_agg:
            res["rel_deviation"], res["deviation_sums"] = rel, sums
        if hit is not None:
            res["krum_success"] = hit.bool()
        if mal is not None:
            res["bulyan_malicious_fraction"] = mal.float() / cnt.clamp(min=1).float()
        if honest is not None:
            res["honest_mean"] = honest
        return res

    TRACE_TABLES = {"agg_deviation": torch.float32, "malicious_deviation": torch.float32, "krum_index": torch.int32,
                    "bulyan_malicious": torch.int32, "bulyan_selected": torch.int32}

    def attack_trace(self, aggregated, slot, tables, *, krum_index=None, selection=None):
        """This round's attack figures into row `slot` (a device int32 [1], e.g. a sweep's epoch counter) of the
        caller's tables (C ABI `afl_attack_trace_dev`, fp32 client matrices): per problem b, `agg_deviation`
        ||a_b - h_b|| / ||h_b|| of `aggregated` (fp32 [B, D]; for Krum the gathered rows `krum` returns),
        `malicious_deviation` the same for row 0 (NaN when f_b = 0), `krum_index` (needs krum_index) and Bulyan's
        `bulyan_malicious` / `bulyan_selected` counts (need selection) -- attack_metrics' figures bit for bit.
        tables: {name: tensor} of any of those names (TRACE_TABLES gives the dtypes), each an [n_slots, B] view with
        unit column stride and one row pitch >= B, e.g. a column slice of an [n_slots, B_total] tensor allocated once,
        so that a captured round keeps its pointers.  A slot outside [0, n_slots) writes nothing.  Allocates nothing
        per call: the workspace comes with the first call and is kept."""
        if self.G.dtype != torch.float32:
            raise TypeError("DeviceRound.attack_trace takes fp32 client matrices only")
        for t, name, dtype, shape in ((aggregated, "aggregated", torch.float32, (self.B, self.D)),
                                      (slot, "slot", torch.int32, (1,)),
                                      (krum_index, "krum_index", torch.int32, (self.B,)),
                                      (selection, "selection", torch.int32, None)):
            if t is not None and not (isinstance(t, torch.Tensor) and t.device == self.device and t.dtype == dtype
                                      and t.is_contiguous() and (t.shape == shape if shape else
                                                                 (t.dim() == 2 and t.shape[0] == self.B))):
                raise ValueError(f"{name}: expected a contiguous {dtype} tensor for {self.B} problems on {self.device}")
        if aggregated is None or slot is None:
            raise ValueError("attack_trace: aggregated and slot are required")
        unknown = set(tables) - set(self.TRACE_TABLES)
        if unknown or not tables:
            raise ValueError(f"attack_trace: tables names one or more of {', '.join(self.TRACE_TABLES)} "
                             f"(got {sorted(tables)})")
        first = next(iter(tables.values()))
        n_slots, table_ld = first.shape[0], first.stride(0)
        for name, t in tables.items():
            if not (isinstance(t, torch.Tensor) and t.device == self.device and t.dtype == self.TRACE_TABLES[name]
                    and t.dim() == 2 and tuple(t.shape) == (n_slots, self.B) and t.stride(1) == 1
                    and t.stride(0) == table_ld and table_ld >= self.B):
                raise ValueError(f"tables[{name!r}]: expected a {self.TRACE_TABLES[name]} [{n_slots}, {self.B}] view "
                                 f"with unit column stride and row pitch {table_ld} >= {self.B} on {self.device}")
        L = nat.lib()
        if self._trace_ws is None:
            self._trace_ws = torch.empty(L.afl_attack_trace_workspace_bytes(self.B, self.D), dtype=torch.uint8,
                                         device=self.device)
        self._call(L.afl_attack_trace_dev, self.G.data_ptr(), self.B, self._bs, self.N, self.D, self._ld,
                   self._ptr(self.rows), self.f.data_ptr(), aggregated.data_ptr(), self._ptr(krum_index),
                   self._ptr(selection), 0 if selection is None else selection.shape[1], slot.data_ptr(), n_slots,
                   table_ld, *(self._ptr(tables.get(k)) for k in self.TRACE_TABLES), self._trace_ws.data_ptr(),
                   self._trace_ws.numel(), self.status.data_ptr(), _stream_ptr(self.G))

    def clear_status(self):
        """Zero `status` (enqueued)."""
        self.status.zero_()

    def raise_for_status(self):
        """Synchronise and raise for the first flagged problem, as the host-parameter call raises for it."""
        st = self.status.cpu().numpy()
        bad = np.flatnonzero(st)
        if not bad.size:
            return
        b, code = int(bad[0]), int(st[bad[0]])
        if code == nat.AFL_ERR_NO_WINNER:
            e = KeyError(-1)
            e.add_note(f"problem {b}: a Bulyan selection round found no eligible user (defences.py:66)")
            raise e
        exc, what = _STATUS_ERRORS.get(code, (nat.NativeError, None))
        if what is None:
            raise nat.NativeError(code, f"problem {b}")
        raise exc(f"problem {b}: {what}")
