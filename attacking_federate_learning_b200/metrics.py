"""Attack-success figures for the ALIE experiments (SURVEY.md section 8d, "Attack-success (C5)").

The reference itself only logs test accuracy (main.py:73-82); these follow from its conventions: the
malicious users are ids 0..f-1 (main.py:28), Krum returns one user's gradient (defences.py:42), Bulyan
averages around the median of theta = n - 2f selected users (defences.py:57-70).  Pure bookkeeping on
indices and on one [D] vector norm; the aggregation itself is done by `defences`.

These three take one problem at a time and `relative_deviation` synchronises the host.  For a batch of problems (a
z x malicious-share x seed grid run through `batched`), `batched.attack_metrics` gives the same three figures for
every problem in one call on the device, with one corrupted_count per problem and no synchronisation; D-sharded:
`sharded.ShardedAggregator.relative_deviation`.
"""
from __future__ import annotations


def krum_attack_success(selected_index: int, corrupted_count: int) -> bool:
    """True when Krum picked one of the malicious users (ids < f, main.py:28)."""
    return 0 <= int(selected_index) < int(corrupted_count)


def bulyan_attack_success(selected_indices, corrupted_count: int) -> float:
    """Fraction of Bulyan's theta selected users that are malicious."""
    sel = [int(i) for i in selected_indices]
    return sum(1 for i in sel if i < corrupted_count) / max(1, len(sel))


def relative_deviation(aggregated, honest_mean) -> float:
    """||agg - honest_mean|| / ||honest_mean|| for torch.cuda tensors (computed on the device)."""
    import torch
    a, h = aggregated.float(), honest_mean.float()
    return float(torch.linalg.vector_norm(a - h) / torch.linalg.vector_norm(h))
