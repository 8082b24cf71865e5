"""CPU checks of the ragged batched entry points afl_defend_batched_rows, afl_attack_metrics_batched_rows and
afl_batched_rows_workspace_bytes, and of batched.py's `rows=` arguments: NULL arrays, row counts outside [1, N],
negative counts, the reference's asserts per problem (naming the problem), Bulyan's users_count == rows_b and short or
misaligned workspaces are rejected before any CUDA call, so these run without a GPU."""
import ctypes

import numpy as np
import pytest

P = ctypes.c_void_p(256)         # a non-NULL pointer that is never dereferenced: validation fails first
BIG = 1 << 30
RULES = (b"Krum", b"Bulyan", b"TrimmedMean", b"NoDefense")


@pytest.fixture(scope="module")
def nat():
    import __graft_entry__ as g
    g.build()
    from attacking_federate_learning_b200 import _native
    _native.lib()
    return _native


def ints(*v):
    return (ctypes.c_int * len(v))(*v)


def defend(nat, rows, users=None, fs=None, rule=b"TrimmedMean", G=P, n=12, d=64, ld=64, stride=None, out=P, idx=P,
           sel=P, ws=P, ws_bytes=BIG, batch=None):
    batch = len(rows) if batch is None else batch
    users = rows if users is None else users
    fs = ints(*([0] * batch)) if fs is None else fs
    stride = n * ld if stride is None else stride
    return nat.lib().afl_defend_batched_rows(rule, G, batch, stride, n, d, ld, nat.AFL_F32, rows, users, fs, out, idx,
                                             sel, ws, ws_bytes, None)


def metrics(nat, rows, fs, n=12, ws=P, ws_bytes=BIG, batch=None):
    batch = len(fs) if batch is None else batch
    return nat.lib().afl_attack_metrics_batched_rows(P, batch, n * 64, n, 64, 64, nat.AFL_F32, rows, fs, P, None, None, 0,
                                                     P, None, None, None, None, None, ws, ws_bytes, None)


def test_rows_rejects_null_arrays(nat):
    L = nat.lib()
    for rule in RULES:
        assert defend(nat, None, users=ints(10, 10), fs=ints(1, 1), rule=rule, batch=2) == nat.AFL_ERR_BAD_ARG
        assert b"NULL" in L.afl_last_error()
        assert defend(nat, ints(10, 10), users=ctypes.c_void_p(), rule=rule) == nat.AFL_ERR_BAD_ARG
        assert b"NULL" in L.afl_last_error()
        assert defend(nat, ints(10, 10), fs=ctypes.c_void_p(), rule=rule) == nat.AFL_ERR_BAD_ARG
        assert b"NULL" in L.afl_last_error()


def test_rows_rejects_row_counts_outside_the_slot(nat):
    L = nat.lib()
    for rule in RULES:
        for bad in (0, -1, 13):
            assert defend(nat, ints(10, 12, bad, 3), rule=rule) == nat.AFL_ERR_BAD_ARG
            msg = L.afl_last_error()
            assert b"problem 2" in msg and b"[1, 12]" in msg
    assert defend(nat, ints(10, 12), rule=b"Nope") == nat.AFL_ERR_BAD_ARG
    assert b"unknown rule" in L.afl_last_error()


def test_rows_rejects_negative_counts(nat):
    L = nat.lib()
    for rule in RULES:
        assert defend(nat, ints(10, 12, 11), fs=ints(1, -2, 0), rule=rule) == nat.AFL_ERR_BAD_ARG
        assert b"problem 1" in L.afl_last_error()


def test_rows_keeps_the_batch_limits(nat):
    L = nat.lib()
    assert defend(nat, ints(10, 12), G=None) == nat.AFL_ERR_BAD_ARG
    assert b"afl_defend_batched_rows" in L.afl_last_error()
    assert defend(nat, ints(10, 12), n=129) == nat.AFL_ERR_UNSUPPORTED
    assert b"n <= 128" in L.afl_last_error()
    assert defend(nat, ints(10), batch=0) == nat.AFL_ERR_BAD_ARG
    assert defend(nat, (ctypes.c_int * 65536)(), batch=65536) == nat.AFL_ERR_UNSUPPORTED
    assert defend(nat, ints(10, 12), stride=11 * 64 + 63) == nat.AFL_ERR_BAD_ARG
    assert b"overlap" in L.afl_last_error()
    assert defend(nat, ints(10, 12), rule=b"Krum", idx=None) == nat.AFL_ERR_BAD_ARG
    assert defend(nat, ints(11, 12), rule=b"Bulyan", sel=None) == nat.AFL_ERR_BAD_ARG
    assert defend(nat, ints(10, 12), rule=b"TrimmedMean", out=None) == nat.AFL_ERR_BAD_ARG


def test_rows_preconditions_name_the_problem(nat):
    L = nat.lib()
    # Krum: users_count_b >= 2 f_b + 1 (defences.py:24-25), with each problem's own users_count
    assert defend(nat, ints(12, 5, 9), users=ints(12, 5, 9), fs=ints(5, 2, 5), rule=b"Krum") == nat.AFL_ERR_PRECONDITION
    msg = L.afl_last_error()
    assert b"2*corrupted_count + 1" in msg and b"problem 2" in msg
    with pytest.raises(AssertionError, match="problem 2"):
        nat.check(defend(nat, ints(12, 5, 9), users=ints(12, 5, 9), fs=ints(5, 2, 5), rule=b"Krum"))
    # Bulyan: users_count_b >= 4 f_b + 3 (defences.py:56); f = 2 holds at 11 users, f = 1 does not at 6
    assert defend(nat, ints(11, 6), fs=ints(2, 1), rule=b"Bulyan") == nat.AFL_ERR_PRECONDITION
    msg = L.afl_last_error()
    assert b"4*corrupted_count + 3" in msg and b"problem 1" in msg


def test_rows_bulyan_users_count_is_the_row_count(nat):
    L = nat.lib()
    assert defend(nat, ints(11, 9), users=ints(11, 10), fs=ints(2, 1), rule=b"Bulyan") == nat.AFL_ERR_UNSUPPORTED
    msg = L.afl_last_error()
    assert b"problem 1" in msg and b"users_count" in msg


def test_rows_workspace(nat):
    L = nat.lib()
    for rule in RULES:
        need = L.afl_batched_rows_workspace_bytes(rule, 2, 12, 64, nat.AFL_F32)
        assert need > 0
        assert defend(nat, ints(11, 12), rule=rule, ws=None) == nat.AFL_ERR_WORKSPACE
        assert defend(nat, ints(11, 12), rule=rule, ws_bytes=need - 1) == nat.AFL_ERR_WORKSPACE
        assert defend(nat, ints(11, 12), rule=rule, ws=ctypes.c_void_p(128)) == nat.AFL_ERR_WORKSPACE
        assert b"workspace" in L.afl_last_error()


def test_rows_workspace_bytes_match_each(nat):
    L = nat.lib()
    rows, each = L.afl_batched_rows_workspace_bytes, L.afl_batched_each_workspace_bytes
    for rule in RULES:
        for B, n, d in ((1, 1, 1), (4, 10, 64), (252, 100, 79_510), (65535, 10, 79_510), (16, 128, 4096)):
            for dt in (nat.AFL_F32, nat.AFL_BF16, nat.AFL_F16):
                assert rows(rule, B, n, d, dt) == each(rule, B, n, d, dt) > 0
        assert rows(rule, 0, 10, 64, nat.AFL_F32) == 0
        assert rows(rule, 65536, 10, 64, nat.AFL_F32) == 0
        assert rows(rule, 4, 129, 64, nat.AFL_F32) == 0
        assert rows(rule, 4, 10, 0, nat.AFL_F32) == 0
    assert rows(b"ALIE", 4, 10, 64, nat.AFL_F32) == 0
    assert rows(b"Nope", 4, 10, 64, nat.AFL_F32) == 0
    assert rows(None, 4, 10, 64, nat.AFL_F32) == 0


def test_metrics_rows_rejects_bad_arguments(nat):
    L = nat.lib()
    assert metrics(nat, None, ints(1, 2)) == nat.AFL_ERR_BAD_ARG
    assert b"NULL" in L.afl_last_error()
    assert metrics(nat, ints(10, 12), None, batch=2) == nat.AFL_ERR_BAD_ARG
    assert metrics(nat, ints(10, 0), ints(1, 2)) == nat.AFL_ERR_BAD_ARG
    assert b"problem 1" in L.afl_last_error()
    assert metrics(nat, ints(10, 13), ints(1, 2)) == nat.AFL_ERR_BAD_ARG
    assert metrics(nat, ints(10, 12), ints(1, -2)) == nat.AFL_ERR_BAD_ARG
    assert b"problem 1" in L.afl_last_error()
    need = L.afl_metrics_workspace_bytes(2, 12, 64, nat.AFL_F32)
    assert metrics(nat, ints(10, 12), ints(1, 2), ws=None) == nat.AFL_ERR_WORKSPACE
    assert metrics(nat, ints(10, 12), ints(1, 2), ws_bytes=need - 1) == nat.AFL_ERR_WORKSPACE


def test_python_rows_arguments(nat):
    torch = pytest.importorskip("torch")
    from attacking_federate_learning_b200 import batched as bt
    rs, ucs, fs = bt._ragged(3, [10, 25, 51], None, 2)
    assert rs.dtype == ucs.dtype == fs.dtype == np.int32
    assert rs.tolist() == ucs.tolist() == [10, 25, 51] and fs.tolist() == [2, 2, 2]
    _, ucs, fs = bt._ragged(3, np.array([10, 25, 51]), 30, torch.tensor([1, 2, 3]))
    assert ucs.tolist() == [30, 30, 30] and fs.tolist() == [1, 2, 3]
    with pytest.raises(ValueError):
        bt._ragged(3, [10, 25], None, 2)
    with pytest.raises(TypeError):
        bt._ragged(3, [10.0, 25.5, 3.0], None, 2)
