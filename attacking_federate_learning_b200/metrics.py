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


# An experiment's per-epoch attack trace (sweep.run(trace=True), harness.main(trace=True)): a dict of numpy arrays over
# epochs.  Every rule has agg_deviation (||aggregate - honest mean|| / ||honest mean||) and malicious_deviation (the
# same for the first malicious row, NaN without one); Krum adds krum_index and krum_malicious, Bulyan
# bulyan_malicious_fraction.
TRACE_HEADER = ['epoch', 'agg_deviation', 'malicious_deviation', 'krum_index', 'krum_malicious',
                'bulyan_malicious_fraction']
TRACE_SUMMARY = ['krum_malicious_epochs', 'bulyan_malicious_fraction_mean', 'agg_deviation_mean',
                 'agg_deviation_final']


def trace_record(defense, corrupted_count, agg_deviation, malicious_deviation, krum_index=None, bulyan_malicious=None,
                 bulyan_selected=None):
    """The trace dict from one experiment's per-epoch figures: krum_malicious is krum_attack_success per epoch (Krum,
    krum_index given) and bulyan_malicious_fraction bulyan_attack_success's mal / max(1, selected) (Bulyan, counts
    given).  The arrays are copies."""
    import numpy as np
    tr = dict(agg_deviation=np.array(agg_deviation, dtype=np.float32),
              malicious_deviation=np.array(malicious_deviation, dtype=np.float32))
    if defense == 'Krum':
        idx = np.array(krum_index, dtype=np.int32)
        tr['krum_index'] = idx
        tr['krum_malicious'] = (idx >= 0) & (idx < int(corrupted_count))
    elif defense == 'Bulyan':
        mal = np.asarray(bulyan_malicious, dtype=np.int64)
        tr['bulyan_malicious_fraction'] = mal / np.maximum(1, np.asarray(bulyan_selected, dtype=np.int64))
    return tr


def write_trace_csv(path, trace):
    """One row per epoch under TRACE_HEADER; the cells of figures the experiment's rule has none of stay empty."""
    import csv
    cols = [trace.get(k) for k in TRACE_HEADER[1:]]
    with open(path, 'w', newline='') as fh:
        w = csv.writer(fh)
        w.writerow(TRACE_HEADER)
        for e in range(len(trace['agg_deviation'])):
            w.writerow([e] + ['' if c is None else (int(c[e]) if c.dtype.kind in 'biu' else float(c[e]))
                              for c in cols])


def trace_summary(trace):
    """TRACE_SUMMARY's cells for one experiment: the epochs Krum picked a malicious client, Bulyan's mean malicious
    fraction (each empty for the other rules), and the mean and final agg_deviation."""
    import numpy as np
    krum = trace.get('krum_malicious')
    bul = trace.get('bulyan_malicious_fraction')
    agg = trace['agg_deviation'].astype(np.float64)
    return ['' if krum is None else int(krum.sum()), '' if bul is None else float(bul.mean()), float(agg.mean()),
            float(agg[-1])]
