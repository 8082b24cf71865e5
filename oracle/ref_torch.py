"""Float64 restatement of Bulyan's selection loop (defences.py:57-68) in torch.  TEST INFRASTRUCTURE ONLY.

`oracle/oracle.c` re-sorts every alive row in every round on the CPU: O(theta * n^2 log n), about an hour at
n = 4096.  This module does the same arithmetic as one batched sort per round, so it runs on a CUDA tensor in
seconds at that size (and on a CPU tensor for the small tables that pin it to the C oracle in the CPU suite).

Per round r (users_count = n - r, the same table with the already selected users removed):
  * dead users and self are masked to +inf;
  * every alive user's score is the float64 sum of its `users_count - f` smallest entries (Python slice semantics
    over the n - r - 1 alive neighbours), taken from a sort plus a sequential float64 cumsum, so identical rows
    tie exactly;
  * the winner is the reference's strict-< scan from (1e20, -1) in visit order [1, 0, 2, ...], which skips scores
    >= 1e20 and NaN;
  * the margin is the C oracle's: (runner-up - best) / |best|, inf without a runner-up or with best == 0.
"""
from __future__ import annotations

import torch


def _slice_take(m: int, length: int) -> int:
    """len(errors[:m]) for a list of `length` entries."""
    if m >= 0:
        return min(m, length)
    return max(length + m, 0)


def bulyan_select(dist, n: int, f: int, with_margins: bool = False):
    """Selection sequence of Bulyan's first stage on the dense [n, n] table `dist` (any float dtype, CPU or
    CUDA).  A round with no eligible user ends the sequence there, like oracle.c's orc_bulyan_select_m."""
    t = torch.as_tensor(dist).to(torch.float64)
    assert t.shape == (n, n)
    dev = t.device
    inf = torch.tensor(float("inf"), dtype=torch.float64, device=dev)
    pos = torch.arange(n, device=dev)                          # visit position of user u
    if n >= 2:
        pos[0], pos[1] = 1, 0
    alive = torch.ones(n, dtype=torch.bool, device=dev)
    eye = torch.eye(n, dtype=torch.bool, device=dev)
    chosen, margins = [], []
    for r in range(n - 2 * f):
        users = torch.nonzero(alive).flatten()
        take = _slice_take((n - r) - f, (n - r) - 1)
        rows = torch.where(eye[users] | ~alive[None, :], inf, t[users])
        if take > 0:
            srt = torch.sort(rows, dim=1).values[:, :take]
            score = torch.cumsum(srt, dim=1)[:, -1]
        else:
            score = torch.zeros(len(users), dtype=torch.float64, device=dev)
        ok = score < 1e20                                      # False for NaN
        if not bool(ok.any()):
            break
        best = torch.min(torch.where(ok, score, inf))
        tied = ok & (score == best)
        k = int(torch.argmin(torch.where(tied, pos[users], n)))
        idx = int(users[k])
        best = float(best)
        rest = torch.cat([score[:k], score[k + 1:]])
        rest = rest[~torch.isnan(rest)]
        second = float(rest.min()) if rest.numel() else float("inf")
        margins.append(float("inf") if second == float("inf") or best == 0.0 else (second - best) / abs(best))
        chosen.append(idx)
        alive[idx] = False
    return (chosen, margins) if with_margins else chosen
