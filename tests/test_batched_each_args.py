"""CPU checks of the per-problem batched entry points afl_defend_batched_each, afl_alie_batched_each and
afl_batched_each_workspace_bytes, and of batched.py's per-problem arguments: NULL arrays, negative or too large
counts, short workspaces, the batch limits and the reference's asserts (per problem, naming the problem) are
rejected before any CUDA call, so these run without a GPU."""
import ctypes

import numpy as np
import pytest

P = ctypes.c_void_p(256)         # a non-NULL pointer that is never dereferenced: validation fails first
BIG = 1 << 30


@pytest.fixture(scope="module")
def nat():
    import __graft_entry__ as g
    g.build()
    from attacking_federate_learning_b200 import _native
    _native.lib()
    return _native


def counts(*f):
    return (ctypes.c_int * len(f))(*f)


def defend(nat, fs, rule=b"TrimmedMean", G=P, stride=10 * 64, n=10, d=64, ld=64, users=10, out=P, idx=P, sel=P,
           ws=P, ws_bytes=BIG, batch=None):
    batch = len(fs) if batch is None else batch
    return nat.lib().afl_defend_batched_each(rule, G, batch, stride, n, d, ld, nat.AFL_F32, users, fs, out, idx, sel,
                                             ws, ws_bytes, None)


def alie(nat, fs, zs=None, G=P, stride=10 * 64, n=10, d=64, ld=64, bcast=None, bstride=0, bld=64, ws=P, ws_bytes=BIG,
         batch=None):
    batch = len(fs) if batch is None else batch
    zs = (ctypes.c_double * batch)(*([1.5] * batch)) if zs is None else zs
    return nat.lib().afl_alie_batched_each(G, batch, stride, n, d, ld, nat.AFL_F32, fs, zs, P, P, P, bcast, bstride, bld,
                                           ws, ws_bytes, None)


def test_defend_each_rejects_bad_counts(nat):
    L = nat.lib()
    assert defend(nat, None, batch=4) == nat.AFL_ERR_BAD_ARG
    assert b"NULL" in L.afl_last_error()
    assert defend(nat, counts(1, 2, -1, 1)) == nat.AFL_ERR_BAD_ARG
    assert b"problem 2" in L.afl_last_error()
    for rule in (b"Krum", b"Bulyan", b"TrimmedMean", b"NoDefense"):
        assert defend(nat, counts(0, -3), rule=rule, n=11, users=11, stride=11 * 64) == nat.AFL_ERR_BAD_ARG
    assert defend(nat, counts(1, 2), rule=b"Nope") == nat.AFL_ERR_BAD_ARG
    assert b"unknown rule" in L.afl_last_error()


def test_defend_each_keeps_the_batch_limits(nat):
    L = nat.lib()
    assert defend(nat, counts(1, 2), G=None) == nat.AFL_ERR_BAD_ARG
    assert b"afl_defend_batched_each" in L.afl_last_error()
    assert defend(nat, counts(1, 2), n=129, users=129, stride=129 * 64) == nat.AFL_ERR_UNSUPPORTED
    assert b"n <= 128" in L.afl_last_error()
    assert defend(nat, counts(1), batch=0) == nat.AFL_ERR_BAD_ARG
    assert defend(nat, (ctypes.c_int * 65536)(), batch=65536) == nat.AFL_ERR_UNSUPPORTED
    assert defend(nat, counts(1, 2), stride=9 * 64 + 63) == nat.AFL_ERR_BAD_ARG
    assert b"overlap" in L.afl_last_error()
    assert defend(nat, counts(1, 2), rule=b"Krum", idx=None) == nat.AFL_ERR_BAD_ARG
    assert defend(nat, counts(1, 2), rule=b"Bulyan", n=11, users=11, stride=11 * 64, sel=None) == nat.AFL_ERR_BAD_ARG


def test_defend_each_preconditions_name_the_problem(nat):
    L = nat.lib()
    # Krum: users_count >= 2 f_b + 1 for every b (defences.py:24-25)
    assert defend(nat, counts(1, 2, 5, 1), rule=b"Krum") == nat.AFL_ERR_PRECONDITION
    msg = L.afl_last_error()
    assert b"2*corrupted_count + 1" in msg and b"problem 2" in msg
    with pytest.raises(AssertionError, match="problem 2"):
        nat.check(defend(nat, counts(1, 2, 5, 1), rule=b"Krum"))
    # every problem fails: the first failing one is named, not the first with the largest count
    assert defend(nat, counts(5, 9), rule=b"Krum") == nat.AFL_ERR_PRECONDITION
    msg = L.afl_last_error()
    assert b"(10, 5) in problem 0" in msg
    # Bulyan: users_count >= 4 f_b + 3 for every b (defences.py:56); f = 2 holds at 11 users, f = 3 does not
    assert defend(nat, counts(2, 3, 0), rule=b"Bulyan", n=11, users=11, stride=11 * 64) == nat.AFL_ERR_PRECONDITION
    msg = L.afl_last_error()
    assert b"4*corrupted_count + 3" in msg and b"problem 1" in msg
    with pytest.raises(AssertionError):
        nat.check(defend(nat, counts(2, 3, 0), rule=b"Bulyan", n=11, users=11, stride=11 * 64))


def test_defend_each_workspace(nat):
    L = nat.lib()
    for rule in (b"Krum", b"TrimmedMean"):
        need = L.afl_batched_each_workspace_bytes(rule, 2, 10, 64, nat.AFL_F32)
        assert defend(nat, counts(1, 2), rule=rule, ws=None) == nat.AFL_ERR_WORKSPACE
        assert defend(nat, counts(1, 2), rule=rule, ws_bytes=need - 1) == nat.AFL_ERR_WORKSPACE
        assert defend(nat, counts(1, 2), rule=rule, ws=ctypes.c_void_p(128)) == nat.AFL_ERR_WORKSPACE
        assert b"workspace" in L.afl_last_error()
    need = L.afl_batched_each_workspace_bytes(b"Bulyan", 2, 11, 64, nat.AFL_F32)
    assert defend(nat, counts(1, 2), rule=b"Bulyan", n=11, users=11, stride=11 * 64,
                  ws_bytes=need - 1) == nat.AFL_ERR_WORKSPACE


def test_alie_each_rejects_bad_arguments(nat):
    L = nat.lib()
    assert alie(nat, None, batch=3) == nat.AFL_ERR_BAD_ARG
    assert alie(nat, counts(1, 2, 3), zs=ctypes.c_void_p()) == nat.AFL_ERR_BAD_ARG
    assert b"NULL" in L.afl_last_error()
    assert alie(nat, counts(1, -1, 3)) == nat.AFL_ERR_BAD_ARG
    assert b"problem 1" in L.afl_last_error()
    assert alie(nat, counts(1, 2, 11)) == nat.AFL_ERR_BAD_ARG                   # f_b <= n
    assert b"problem 2" in L.afl_last_error()
    assert alie(nat, counts(1, 2), G=None) == nat.AFL_ERR_BAD_ARG
    assert alie(nat, counts(1), batch=0) == nat.AFL_ERR_BAD_ARG
    assert alie(nat, counts(1, 2), n=129, stride=129 * 64) == nat.AFL_ERR_UNSUPPORTED
    assert alie(nat, counts(1, 2), stride=64) == nat.AFL_ERR_BAD_ARG
    # the written rows of two problems may not overlap: the largest f_b counts
    assert alie(nat, counts(1, 3), bcast=P, bstride=2 * 64) == nat.AFL_ERR_BAD_ARG
    assert alie(nat, counts(1, 2), bcast=P, bstride=640, bld=32) == nat.AFL_ERR_BAD_ARG
    need = L.afl_batched_each_workspace_bytes(b"ALIE", 2, 10, 64, nat.AFL_F32)
    assert alie(nat, counts(1, 2), ws=None) == nat.AFL_ERR_WORKSPACE
    assert alie(nat, counts(1, 2), ws_bytes=need - 1) == nat.AFL_ERR_WORKSPACE


def test_each_workspace_bytes(nat):
    L = nat.lib()
    each = L.afl_batched_each_workspace_bytes
    assert each(b"Nope", 4, 10, 64, nat.AFL_F32) == 0
    assert each(None, 4, 10, 64, nat.AFL_F32) == 0
    for rule in (b"Krum", b"Bulyan", b"TrimmedMean", b"NoDefense", b"ALIE"):
        assert each(rule, 0, 10, 64, nat.AFL_F32) == 0
        assert each(rule, 65536, 10, 64, nat.AFL_F32) == 0
        assert each(rule, 4, 129, 64, nat.AFL_F32) == 0
        assert each(rule, 4, 10, 0, nat.AFL_F32) == 0
    for rule in (b"Krum", b"Bulyan", b"TrimmedMean", b"NoDefense"):
        for B in (1, 252, 65535):
            scalar = L.afl_batched_workspace_bytes(rule, B, 10, 79_510, nat.AFL_F32)
            assert each(rule, B, 10, 79_510, nat.AFL_F32) >= scalar
            if rule in (b"Krum", b"Bulyan"):                      # the table, then the scalar call's layout
                table = each(rule, B, 10, 79_510, nat.AFL_F32) - scalar
                assert table >= B * 4 * 4 and table % 256 == 0
    assert each(b"ALIE", 252, 10, 79_510, nat.AFL_F32) == each(b"Krum", 252, 10, 79_510, nat.AFL_F32) - \
        L.afl_batched_workspace_bytes(b"Krum", 252, 10, 79_510, nat.AFL_F32)


def test_python_per_problem_arguments():
    torch = pytest.importorskip("torch")
    from attacking_federate_learning_b200 import batched as bt
    assert bt._per_problem(2, 3, "f", np.int32) is None
    assert bt._per_problem(np.int64(2), 3, "f", np.int32) is None
    assert bt._per_problem(torch.tensor(2), 3, "f", np.int32) is None
    assert bt._per_problem(1.5, 3, "z", np.float64) is None
    for seq in ([1, 2, 0], (1, 2, 0), np.array([1, 2, 0]), torch.tensor([1, 2, 0])):
        a = bt._per_problem(seq, 3, "f", np.int32)
        assert a.dtype == np.int32 and a.flags.c_contiguous and a.tolist() == [1, 2, 0]
    z = bt._per_problem(torch.tensor([0.5, 0.0]), 2, "z", np.float64)
    assert z.dtype == np.float64 and z.tolist() == [0.5, 0.0]
    with pytest.raises(ValueError):
        bt._per_problem([1, 2], 3, "f", np.int32)
    with pytest.raises(ValueError):
        bt._per_problem(np.zeros((3, 1), np.int32), 3, "f", np.int32)
    with pytest.raises(TypeError):
        bt._per_problem([1.0, 2.5, 0.0], 3, "f", np.int32)
