"""CPU checks of the large batched entry points afl_defend_batched_large, afl_alie_batched_large and
afl_batched_large_workspace_bytes (up to 1024 clients per problem), and of batched.py's limit: the client limit, the
per-problem rejections (naming the problem) and short or misaligned workspaces are rejected before any CUDA call, so
these run without a GPU."""
import ctypes

import numpy as np
import pytest

P = ctypes.c_void_p(256)         # a non-NULL pointer that is never dereferenced: validation fails first
BIG = 1 << 30
RULES = (b"Krum", b"Bulyan", b"TrimmedMean", b"NoDefense")
DTYPES = (0, 1, 2)               # AFL_F32, AFL_BF16, AFL_F16


@pytest.fixture(scope="module")
def nat():
    import __graft_entry__ as g
    g.build()
    from attacking_federate_learning_b200 import _native
    _native.lib()
    assert (_native.AFL_F32, _native.AFL_BF16, _native.AFL_F16) == DTYPES
    return _native


def ints(*v):
    return (ctypes.c_int * len(v))(*v)


def defend(nat, rows, users=None, fs=None, rule=b"TrimmedMean", G=P, n=1000, d=64, ld=64, stride=None, out=P, idx=P,
           sel=P, ws=P, ws_bytes=BIG, batch=None):
    batch = (len(rows) if rows else 2) if batch is None else batch
    users = (rows if rows else ints(*([n] * batch))) if users is None else users
    fs = ints(*([0] * batch)) if fs is None else fs
    stride = n * ld if stride is None else stride
    return nat.lib().afl_defend_batched_large(rule, G, batch, stride, n, d, ld, nat.AFL_F32, rows, users, fs, out, idx,
                                              sel, ws, ws_bytes, None)


def test_large_client_limit(nat):
    L = nat.lib()
    for rule in RULES:
        assert defend(nat, None, rule=rule, n=1025) == nat.AFL_ERR_UNSUPPORTED
        msg = L.afl_last_error()
        assert b"n <= 1024" in msg and b"afl_defend_batched_large" in msg
        # 129 .. 1024 rows pass the size check and every per-problem check: the call stops at the missing workspace
        for n in (129, 500, 1000, 1024):
            assert defend(nat, None, rule=rule, n=n, ws=None) == nat.AFL_ERR_WORKSPACE
            assert b"workspace" in L.afl_last_error()
            assert defend(nat, ints(n, 3), users=ints(n, 3), rule=rule, n=n, ws=None) == nat.AFL_ERR_WORKSPACE


def test_large_rejects_row_counts_outside_the_slot(nat):
    L = nat.lib()
    for rule in RULES:
        for bad in (0, -1, 1001):
            assert defend(nat, ints(1000, 129, bad, 3), rule=rule) == nat.AFL_ERR_BAD_ARG
            msg = L.afl_last_error()
            assert b"problem 2" in msg and b"[1, 1000]" in msg


def test_large_rejects_negative_counts(nat):
    L = nat.lib()
    for rule in RULES:
        assert defend(nat, ints(1000, 500, 300), fs=ints(1, -2, 0), rule=rule) == nat.AFL_ERR_BAD_ARG
        assert b"problem 1" in L.afl_last_error()
        assert defend(nat, None, fs=ctypes.c_void_p(), rule=rule) == nat.AFL_ERR_BAD_ARG
        assert b"NULL" in L.afl_last_error()


def test_large_preconditions_name_the_problem(nat):
    L = nat.lib()
    # Krum: users_count_b >= 2 f_b + 1 (defences.py:24-25)
    assert defend(nat, ints(1000, 500, 300), fs=ints(240, 100, 150), rule=b"Krum") == nat.AFL_ERR_PRECONDITION
    msg = L.afl_last_error()
    assert b"2*corrupted_count + 1" in msg and b"problem 2" in msg
    # Bulyan: users_count_b >= 4 f_b + 3 (defences.py:56); f = 240 holds at 1000 users, f = 125 does not at 500
    assert defend(nat, ints(1000, 500), fs=ints(240, 125), rule=b"Bulyan") == nat.AFL_ERR_PRECONDITION
    msg = L.afl_last_error()
    assert b"4*corrupted_count + 3" in msg and b"problem 1" in msg
    # the asserts hold: the call reaches the workspace check
    assert defend(nat, ints(1000, 500), fs=ints(240, 124), rule=b"Bulyan", ws=None) == nat.AFL_ERR_WORKSPACE


def test_large_bulyan_users_count_is_the_row_count(nat):
    L = nat.lib()
    assert defend(nat, ints(1000, 300), users=ints(1000, 301), fs=ints(2, 1), rule=b"Bulyan") == nat.AFL_ERR_UNSUPPORTED
    msg = L.afl_last_error()
    assert b"problem 1" in msg and b"users_count" in msg


def test_large_workspace(nat):
    L = nat.lib()
    for rule in RULES:
        need = L.afl_batched_large_workspace_bytes(rule, 2, 1000, 64, nat.AFL_F32)
        assert need > 0
        assert defend(nat, ints(999, 1000), rule=rule, ws=None) == nat.AFL_ERR_WORKSPACE
        assert defend(nat, ints(999, 1000), rule=rule, ws_bytes=need - 1) == nat.AFL_ERR_WORKSPACE
        assert defend(nat, ints(999, 1000), rule=rule, ws=ctypes.c_void_p(128)) == nat.AFL_ERR_WORKSPACE
        assert b"workspace" in L.afl_last_error()


def test_large_workspace_bytes(nat):
    L = nat.lib()
    large, rows = L.afl_batched_large_workspace_bytes, L.afl_batched_rows_workspace_bytes
    for rule in RULES:
        for dt in DTYPES:
            for B, n, d in ((1, 1, 1), (4, 10, 64), (252, 100, 79_510), (65535, 10, 79_510), (16, 128, 4096)):
                assert large(rule, B, n, d, dt) == rows(rule, B, n, d, dt) > 0
            for B, n, d in ((1, 129, 64), (48, 1000, 79_510), (4, 1024, 4096), (65535, 200, 64)):
                assert large(rule, B, n, d, dt) > 0
                # at least the table, the class permutation and (Krum, Bulyan) the n x n float64 tables
                assert large(rule, B, n, d, dt) >= B * 44 + (B * n * n * 8 if rule in (b"Krum", b"Bulyan") else 0)
            assert large(rule, 4, 1025, 64, dt) == 0
        assert large(rule, 0, 200, 64, nat.AFL_F32) == 0
        assert large(rule, 65536, 200, 64, nat.AFL_F32) == 0
        assert large(rule, 4, 200, 0, nat.AFL_F32) == 0
        assert large(rule, 4, 0, 64, nat.AFL_F32) == 0
        assert large(rule, 4, 200, 64, 7) == 0
    assert large(b"ALIE", 4, 200, 64, nat.AFL_F32) == 0
    assert large(b"Nope", 4, 200, 64, nat.AFL_F32) == 0
    assert large(None, 4, 200, 64, nat.AFL_F32) == 0


def test_alie_large_counts(nat):
    L = nat.lib()
    zs = (ctypes.c_double * 2)(1.0, 1.5)

    def alie(fs, n=1000, ws=None):
        return L.afl_alie_batched_large(P, 2, n * 64, n, 64, 64, nat.AFL_F32, fs, zs, P, P, P, None, 0, 0, ws, 0, None)
    # f_b <= n passes every count check and stops at the missing workspace (the table)
    assert alie(ints(240, 1000)) == nat.AFL_ERR_WORKSPACE
    assert alie(ints(1, 0)) == nat.AFL_ERR_WORKSPACE
    assert alie(ints(240, 1001)) == nat.AFL_ERR_BAD_ARG
    assert b"problem 1" in L.afl_last_error() and b"[0, 1000]" in L.afl_last_error()
    assert alie(ints(-1, 3)) == nat.AFL_ERR_BAD_ARG
    assert alie(None) == nat.AFL_ERR_BAD_ARG
    assert b"afl_alie_batched_large" in L.afl_last_error()
    # no client limit: 5000-row problems are accepted too
    assert alie(ints(4000, 2), n=5000) == nat.AFL_ERR_WORKSPACE
    # the one-tile entry keeps its limit
    assert L.afl_alie_batched_each(P, 2, 1000 * 64, 1000, 64, 64, nat.AFL_F32, ints(240, 10), zs, P, P, P, None, 0, 0,
                                   None, 0, None) == nat.AFL_ERR_UNSUPPORTED


def test_python_limit(nat):
    torch = pytest.importorskip("torch")
    from attacking_federate_learning_b200 import batched as bt
    assert bt.MAX_CLIENTS == 1024
    with pytest.raises(TypeError):               # a CPU tensor is refused before anything else
        bt.krum(torch.empty((2, 1025, 8)), 1025, 10)
    rs, ucs, fs = bt._ragged(3, 1000, 1000, [240, 100, 0])
    assert rs.tolist() == [1000] * 3 and ucs.tolist() == [1000] * 3 and fs.tolist() == [240, 100, 0]
    assert np.asarray(rs).dtype == np.int32
