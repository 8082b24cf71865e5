"""The row DeviceRound.krum gathers (batched.krum_gather_rows), on CPU tensors: torch raises IndexError there for an
index outside the slot, where a CUDA gather would stop the process with a device-side assert.

A Krum index of -1 (no eligible user) selects the last row the problem ran with.  A problem flagged for its row count
ran on the safe row (N rows), and its safe run gives -1 whenever no user is eligible: always at N = 1, or on a slot of
infinite rows.  Whatever int32 the caller wrote into `rows`, the gathered row must lie in [0, N); a valid rows_b gives
rows_b - 1 for -1 and the index itself otherwise.
"""
import numpy as np
import pytest
import torch

from attacking_federate_learning_b200.batched import krum_gather_rows

INT32_MIN, INT32_MAX = -2 ** 31, 2 ** 31 - 1


@pytest.mark.parametrize("N", [1, 2, 40, 128])
def test_gather_row_stays_in_the_slot(N):
    rows = list(range(-N - 3, N + 4)) + [INT32_MIN, INT32_MAX]
    idxs = sorted({-1, 0, N - 1})
    pairs = [(i, r) for i in idxs for r in rows]
    idx = torch.tensor([i for i, _ in pairs], dtype=torch.int32)
    rs = torch.tensor([r for _, r in pairs], dtype=torch.int32)
    got = krum_gather_rows(idx, rs, N)
    assert got.dtype == torch.int64 and got.shape == idx.shape
    for (i, r), g in zip(pairs, got.tolist()):
        assert 0 <= g < N, (N, i, r, g)
        if i >= 0:
            assert g == i, (N, i, r, g)
        elif 1 <= r <= N:
            assert g == r - 1, (N, i, r, g)
        else:
            assert g == N - 1, (N, i, r, g)                  # the safe row's last row
    # the gather itself: one [N, 2] slot per pair, each row holding its own number
    G = torch.arange(N, dtype=torch.float32)[None, :, None].expand(len(pairs), N, 2)
    picked = G[torch.arange(len(pairs)), got]
    assert torch.equal(picked[:, 0].long(), got)


@pytest.mark.parametrize("N", [1, 2, 40, 128])
def test_gather_row_without_rows(N):
    idx = torch.tensor(sorted({-1, 0, N - 1}), dtype=torch.int32)
    got = krum_gather_rows(idx, None, N).tolist()
    assert got == [N - 1 if i < 0 else i for i in idx.tolist()]


def test_gather_row_keeps_the_valid_problems_result():
    """The expression DeviceRound.krum used before: rows_b - 1 for -1.  Every valid rows_b gives the same row."""
    N = 40
    rng = np.random.default_rng(0)
    rows = torch.from_numpy(rng.integers(1, N + 1, 500).astype(np.int32))
    idx = torch.from_numpy(np.where(rng.random(500) < 0.5, -1, rng.integers(0, N, 500)).astype(np.int32))
    old = torch.where(idx.long() < 0, rows.long() - 1, idx.long())
    assert torch.equal(krum_gather_rows(idx, rows, N), old)
