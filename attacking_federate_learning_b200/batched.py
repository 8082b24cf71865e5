"""Batched aggregation: B independent same-shape problems (a grid of runs over the attack strength, the
defence, the malicious share or the seed) through the defences of `defences.py` in one launch per kernel
stage instead of B Python-level calls.

Every problem keeps the reference's semantics exactly: problem b's result is what the single device call
(`defences.krum` / `bulyan` / `trimmed_mean` / `no_defense`, `malicious.Attack.attack_rows`) returns for
`G[b]`, bit for bit (C ABI `afl_defend_batched` / `afl_alie_batched`).

Inputs are torch.cuda float32 / bfloat16 tensors `[B, N, D]` with `stride(2) == 1` and N <= 128 clients (one
Gram tile); every problem shares N, D, `users_count` and `corrupted_count`.  Nothing here synchronises the
host except `bulyan`, which checks for a failed selection round as `defences.bulyan` does.

The server's momentum step needs no batched form: `_device.momentum_step` on contiguous `[B, D]` weights,
velocity and gradients is already the batched step (server.py:89-90 is element-wise).
"""
from __future__ import annotations

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


def _defend(rule: str, G: torch.Tensor, users_count: int, corrupted_count: int, out=None, idx=None, sel=None):
    B, N, D, ld, bs = _check(G)
    L = nat.lib()
    with torch.cuda.device(G.device):
        nbytes = L.afl_batched_workspace_bytes(rule.encode(), B, N, D, dtype_code(G))
        ws = Workspace.get(G.device, "batched", nbytes) if nbytes else None
        nat.check(L.afl_defend_batched(rule.encode(), G.data_ptr(), B, bs, N, D, ld, dtype_code(G), int(users_count),
                                       int(corrupted_count), None if out is None else out.data_ptr(),
                                       None if idx is None else idx.data_ptr(), None if sel is None else sel.data_ptr(),
                                       None if ws is None else ws.data_ptr(), 0 if ws is None else ws.numel(),
                                       _stream_ptr(G)))


def krum(users_grads, users_count, corrupted_count, return_index=False):
    """Per problem defences.krum: the winning rows `G[arange(B), idx]` ([B, D], input dtype), or with
    return_index the device int32 [B] indices (-1 where no user is eligible).  No host synchronisation."""
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
    Raises KeyError(-1) when any problem's last selection is -1 (a round found no eligible user), as
    `defences.bulyan` does for one problem."""
    assert users_count >= 4 * corrupted_count + 3
    B, _, D = users_grads.shape
    theta = users_count - 2 * corrupted_count
    out = torch.empty((B, D), dtype=torch.float32, device=users_grads.device)
    sel = torch.empty((B, theta), dtype=torch.int32, device=users_grads.device)
    _defend(DefenseTypes.Bulyan, users_grads, users_count, corrupted_count, out=out, sel=sel)
    if bool((sel[:, -1] < 0).any()):                     # defences.py:66 `distances.pop(-1)`
        raise KeyError(-1)
    return (out, sel) if return_selection else out


defend = {DefenseTypes.Krum: krum,
          DefenseTypes.TrimmedMean: trimmed_mean, DefenseTypes.NoDefense: no_defense,
          DefenseTypes.Bulyan: bulyan}


def alie_rows(users_grads, corrupted_count, num_std):
    """Per problem malicious.Attack.attack_rows (DriftAttack): the malicious users are rows 0..f-1 of every
    problem.  Returns (crafted, mu, sigma), each fp32 [B, D] (mu is the unperturbed mean), and writes crafted
    = mu - num_std * sigma into those rows in place (fp32 directly; bf16 through a cast, as attack_rows does).
    With num_std == 0 the rows are left alone, as attack_rows does.  None when corrupted_count <= 0."""
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
