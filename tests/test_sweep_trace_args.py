"""CPU checks of the attack trace: afl_attack_trace_dev's host checks and workspace size (rejected before any CUDA
call, so no GPU is needed), --trace on the sweep and harness command lines, and the trace files `sweep.write_logs`
and metrics.write_trace_csv write from synthetic results."""
import csv
import ctypes
import os

import numpy as np
import pytest

P = ctypes.c_void_p(256)         # a non-NULL, 256-byte aligned pointer that is never dereferenced
NULL = ctypes.c_void_p()
BIG = 1 << 30


@pytest.fixture(scope="module")
def nat():
    import __graft_entry__ as g
    g.build()
    from attacking_federate_learning_b200 import _native
    _native.lib()
    return _native


def trace(nat, G=P, batch=3, n=12, d=64, ld=64, stride=None, rows=None, fs=P, agg=P, idx=None, sel=None, sel_ld=0,
          slot=P, n_slots=4, table_ld=None, agg_dev=P, mal_dev=P, idx_out=None, mal_count=None, sel_count=None, ws=P,
          ws_bytes=BIG, status=P):
    stride = n * ld if stride is None else stride
    table_ld = batch if table_ld is None else table_ld
    return nat.lib().afl_attack_trace_dev(G, batch, stride, n, d, ld, rows, fs, agg, idx, sel, sel_ld, slot, n_slots,
                                          table_ld, agg_dev, mal_dev, idx_out, mal_count, sel_count, ws, ws_bytes,
                                          status, None)


@pytest.mark.parametrize("kw, text", [
    (dict(G=NULL), b"bad argument"),
    (dict(agg=NULL), b"agg"),
    (dict(slot=NULL), b"slot"),
    (dict(fs=NULL), b"NULL"),
    (dict(status=NULL), b"NULL"),
    (dict(n_slots=0), b"n_slots must be >= 1"),
    (dict(batch=3, table_ld=2), b"table_ld 2 is less than batch 3"),
    (dict(sel=P, sel_ld=0), b"sel_ld must be >= 1"),
    (dict(mal_count=P), b"mal_count and sel_count need sel"),
    (dict(sel_count=P), b"mal_count and sel_count need sel"),
    (dict(idx_out=P), b"idx_out needs idx"),
    (dict(stride=12 * 64 - 1), b"batch_stride"),
    (dict(batch=0), b"batch must be >= 1"),
    (dict(d=0), b"bad argument"),
])
def test_trace_bad_arguments(nat, kw, text):
    assert trace(nat, **kw) == nat.AFL_ERR_BAD_ARG
    assert text in nat.lib().afl_last_error()
    assert b"afl_attack_trace_dev" in nat.lib().afl_last_error()


def test_trace_workspace(nat):
    L = nat.lib()
    batch, d = 5, 79_510
    tiles = -(-d // (256 * 4))                                  # fp32 column tiles of 256 threads x 4 columns
    align = lambda x: -(-x // 256) * 256                        # noqa: E731
    want = align(batch * 40) + align(batch * tiles * 3 * 8)    # the ProblemParams table, then 3 doubles a tile
    assert L.afl_attack_trace_workspace_bytes(batch, d) == want
    assert L.afl_attack_trace_workspace_bytes(0, d) == 0
    assert L.afl_attack_trace_workspace_bytes(65536, d) == 0
    assert L.afl_attack_trace_workspace_bytes(batch, 0) == 0
    need = L.afl_attack_trace_workspace_bytes(3, 64)
    for ws, nbytes in ((P, need - 1), (ctypes.c_void_p(260), BIG), (NULL, BIG)):
        assert trace(nat, ws=ws, ws_bytes=nbytes) == nat.AFL_ERR_WORKSPACE
        assert b"workspace" in L.afl_last_error()


def test_trace_flag_parses():
    from attacking_federate_learning_b200 import harness, sweep
    assert sweep.parser().parse_args(['--trace']).trace is True
    assert sweep.parser().parse_args([]).trace is False
    assert harness.parser().parse_args(['--trace', '-d', 'Krum']).trace is True
    assert harness.parser().parse_args([]).trace is False


def test_trace_record_derives_metrics_figures():
    from attacking_federate_learning_b200 import metrics
    idx, f = np.array([0, 1, 2, -1, 3], np.int32), 2
    tr = metrics.trace_record('Krum', f, np.ones(5), np.ones(5), krum_index=idx)
    assert tr['krum_malicious'].tolist() == [metrics.krum_attack_success(i, f) for i in idx]
    assert tr['krum_index'].tolist() == idx.tolist() and 'bulyan_malicious_fraction' not in tr
    sels = [[0, 3, 4, 5], [-1, -1, -2, -2], [1, -1, -2, -2], [2, 3, 0, 1]]
    mal = [sum(0 <= i < f for i in s) for s in sels]
    cnt = [sum(i >= 0 for i in s) for s in sels]
    tr = metrics.trace_record('Bulyan', f, np.ones(4), np.ones(4), bulyan_malicious=mal, bulyan_selected=cnt)
    want = [metrics.bulyan_attack_success([i for i in s if i >= 0], f) for s in sels]
    assert tr['bulyan_malicious_fraction'].tolist() == want and 'krum_index' not in tr
    tr = metrics.trace_record('TrimmedMean', 0, [0.5, 0.25], [np.nan, np.nan])
    assert sorted(tr) == ['agg_deviation', 'malicious_deviation']


def _results():
    from attacking_federate_learning_b200 import metrics, sweep
    exps = [sweep.Experiment('Krum', 0.24, 1.5, 10, 0), sweep.Experiment('Bulyan', 0.1, 0.5, 10, 0),
            sweep.Experiment('NoDefense', 0.0, 1.0, 10, 1), sweep.Experiment('Bulyan', 0.24, 1.5, 10, 1)]
    E = 3
    res = []
    for k, e in enumerate(exps):
        f = e.corrupted_count
        tr = metrics.trace_record(e.defense, f, np.full(E, 0.5 + k, np.float32),
                                  np.full(E, np.nan if f == 0 else 2.0, np.float32),
                                  krum_index=[0, 5, -1], bulyan_malicious=[1, 0, 1], bulyan_selected=[6, 6, 0])
        err = KeyError(-1) if k == 3 else None
        res.append(dict(experiment=e, accuracies=[10.0, 20.0], accuracies_epochs=[0, 2], error=err,
                        trace=None if err else tr))
    names = [sweep.csv_name(e, 0.1) for e in exps]
    return res, names


def _read(path):
    with open(path, newline='') as fh:
        return list(csv.reader(fh))


def test_trace_files(tmp_path):
    from attacking_federate_learning_b200 import metrics, sweep
    res, names = _results()
    sweep.write_logs(res, str(tmp_path), names, trace=True)
    assert metrics.TRACE_HEADER == ['epoch', 'agg_deviation', 'malicious_deviation', 'krum_index', 'krum_malicious',
                                    'bulyan_malicious_fraction']
    for r, name in zip(res, names):
        if r['error'] is not None:                               # a failed experiment writes no trace
            assert r['trace_csv'] is None and r['csv'] is None
            assert not os.path.exists(tmp_path / sweep.trace_csv_name(name))
            continue
        assert r['trace_csv'] == os.path.join(str(tmp_path), name[:-4] + '_trace.csv')
        assert r['trace_csv'].endswith(f"_seed_{r['experiment'].seed}_trace.csv")
        rows = _read(r['trace_csv'])
        assert rows[0] == metrics.TRACE_HEADER and [x[0] for x in rows[1:]] == ['0', '1', '2']
        rule = r['experiment'].defense
        for x in rows[1:]:
            assert (x[3] != '') == (x[4] != '') == (rule == 'Krum')
            assert (x[5] != '') == (rule == 'Bulyan')
            assert x[1] != '' and x[2] != ''
        if rule == 'Krum':
            assert [x[3] for x in rows[1:]] == ['0', '5', '-1'] and [x[4] for x in rows[1:]] == ['1', '0', '0']
        if rule == 'Bulyan':
            assert [float(x[5]) for x in rows[1:]] == [1 / 6, 0.0, 1.0]
        if rule == 'NoDefense':
            assert all(x[2] == 'nan' for x in rows[1:])
    summary = _read(tmp_path / sweep.SUMMARY)
    assert summary[0] == sweep.summary_header(False, False, True)
    assert summary[0][-5:] == metrics.TRACE_SUMMARY + ['status']
    krum, bulyan, nodef, failed = summary[1:]
    assert krum[-5:-1] == ['1', '', '0.5', '0.5'] and bulyan[-5:-1] == ['', repr((1 / 6 + 1.0) / 3), '1.5', '1.5']
    assert nodef[-5:-1] == ['', '', '2.5', '2.5']
    assert failed[-5:-1] == ['', '', '', ''] and failed[-1].startswith('failed: KeyError')


def test_no_trace_columns_or_files_without_trace(tmp_path):
    from attacking_federate_learning_b200 import sweep
    res, names = _results()
    for r in res:
        del r['trace']
    sweep.write_logs(res, str(tmp_path), names)
    summary = _read(tmp_path / sweep.SUMMARY)
    assert summary[0] == sweep.summary_header(False) and 'agg_deviation_mean' not in summary[0]
    assert all(len(row) == len(summary[0]) for row in summary)
    assert not [p for p in os.listdir(tmp_path) if p.endswith('_trace.csv')]
    assert all('trace_csv' not in r for r in res)
