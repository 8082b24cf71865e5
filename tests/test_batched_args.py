"""CPU checks of the batched entry points afl_defend_batched, afl_alie_batched and afl_batched_workspace_bytes:
null pointers, sizes past the batch limits, overlapping batch strides and the reference's asserts are rejected
before any CUDA call, so these run without a GPU."""
import ctypes

import pytest

P = ctypes.c_void_p(256)         # a non-NULL pointer that is never dereferenced: validation fails first


@pytest.fixture(scope="module")
def nat():
    import __graft_entry__ as g
    g.build()
    from attacking_federate_learning_b200 import _native
    _native.lib()
    return _native


def defend(nat, rule=b"TrimmedMean", G=P, batch=4, stride=10 * 64, n=10, d=64, ld=64, users=10, f=2, out=P, idx=P,
           sel=P):
    return nat.lib().afl_defend_batched(rule, G, batch, stride, n, d, ld, nat.AFL_F32, users, f, out, idx, sel, P,
                                        1 << 30, None)


def alie(nat, G=P, batch=4, stride=10 * 64, f=2, d=64, ld=64, bcast=None, bstride=0, bld=64):
    return nat.lib().afl_alie_batched(G, batch, stride, f, d, ld, nat.AFL_F32, 1.5, P, P, P, bcast, bstride, bld, None)


def test_defend_batched_null_pointers(nat):
    L = nat.lib()
    assert defend(nat, rule=None) == nat.AFL_ERR_BAD_ARG
    assert defend(nat, rule=b"Nope") == nat.AFL_ERR_BAD_ARG
    assert b"unknown rule" in L.afl_last_error()
    assert defend(nat, G=None) == nat.AFL_ERR_BAD_ARG
    assert b"afl_defend_batched" in L.afl_last_error()
    assert defend(nat, rule=b"TrimmedMean", out=None) == nat.AFL_ERR_BAD_ARG
    assert defend(nat, rule=b"NoDefense", out=None) == nat.AFL_ERR_BAD_ARG
    assert defend(nat, rule=b"Krum", idx=None) == nat.AFL_ERR_BAD_ARG
    assert defend(nat, rule=b"Bulyan", n=11, users=11, sel=None) == nat.AFL_ERR_BAD_ARG
    assert defend(nat, rule=b"Bulyan", n=11, users=11, out=None) == nat.AFL_ERR_BAD_ARG


def test_defend_batched_sizes(nat):
    L = nat.lib()
    assert defend(nat, n=0) == nat.AFL_ERR_BAD_ARG
    assert defend(nat, d=0) == nat.AFL_ERR_BAD_ARG
    assert defend(nat, ld=63) == nat.AFL_ERR_BAD_ARG
    assert defend(nat, n=129, users=129, stride=129 * 64) == nat.AFL_ERR_UNSUPPORTED
    assert b"n <= 128" in L.afl_last_error()
    assert defend(nat, batch=0) == nat.AFL_ERR_BAD_ARG
    assert defend(nat, batch=-1) == nat.AFL_ERR_BAD_ARG
    assert defend(nat, batch=65536) == nat.AFL_ERR_UNSUPPORTED
    assert b"65535" in L.afl_last_error()


def test_defend_batched_strides(nat):
    L = nat.lib()
    assert defend(nat, stride=-640) == nat.AFL_ERR_BAD_ARG
    assert b"overlap" in L.afl_last_error()
    assert defend(nat, stride=0) == nat.AFL_ERR_BAD_ARG
    assert defend(nat, stride=9 * 64 + 63) == nat.AFL_ERR_BAD_ARG       # one element short of a problem's span
    # the span is (n - 1) * ld + d, so the stride may be shorter than n * ld when ld > d
    assert defend(nat, rule=b"Krum", stride=9 * 80 + 64, ld=80, idx=None) == nat.AFL_ERR_BAD_ARG   # stride accepted
    assert b"needs idx_out" in L.afl_last_error()


def test_defend_batched_preconditions(nat):
    L = nat.lib()
    # Krum: users_count >= 2f + 1 (defences.py:24-25)
    assert defend(nat, rule=b"Krum", f=5) == nat.AFL_ERR_PRECONDITION
    assert b"2*corrupted_count + 1" in L.afl_last_error()
    # Bulyan: users_count >= 4f + 3 (defences.py:56)
    assert defend(nat, rule=b"Bulyan", f=2) == nat.AFL_ERR_PRECONDITION
    assert b"4*corrupted_count + 3" in L.afl_last_error()
    assert defend(nat, rule=b"Bulyan", n=12, users=11, stride=12 * 64, f=2) == nat.AFL_ERR_UNSUPPORTED
    with pytest.raises(AssertionError):
        nat.check(defend(nat, rule=b"Bulyan", f=2))


def test_alie_batched_rejects_bad_arguments(nat):
    L = nat.lib()
    assert alie(nat, G=None) == nat.AFL_ERR_BAD_ARG
    assert b"afl_alie_batched" in L.afl_last_error()
    assert alie(nat, f=0) == nat.AFL_ERR_BAD_ARG
    assert alie(nat, batch=0) == nat.AFL_ERR_BAD_ARG
    assert alie(nat, batch=65536) == nat.AFL_ERR_UNSUPPORTED
    assert alie(nat, f=129, stride=129 * 64) == nat.AFL_ERR_UNSUPPORTED
    assert alie(nat, stride=64) == nat.AFL_ERR_BAD_ARG
    assert alie(nat, bcast=P, bstride=64) == nat.AFL_ERR_BAD_ARG
    assert alie(nat, bcast=P, bstride=640, bld=32) == nat.AFL_ERR_BAD_ARG


def test_batched_workspace_bytes(nat):
    L = nat.lib()
    assert L.afl_batched_workspace_bytes(b"Nope", 4, 10, 64, nat.AFL_F32) == 0
    assert L.afl_batched_workspace_bytes(b"Krum", 0, 10, 64, nat.AFL_F32) == 0
    assert L.afl_batched_workspace_bytes(b"Krum", 4, 129, 64, nat.AFL_F32) == 0
    krum = L.afl_batched_workspace_bytes(b"Krum", 256, 10, 79_510, nat.AFL_F32)
    assert krum >= 256 * 10 * 10 * 8
    assert L.afl_batched_workspace_bytes(b"Bulyan", 256, 10, 79_510, nat.AFL_F32) > krum
    # the split count is chosen for the whole batch: the partials do not grow with it (C1 size, 132 splits alone)
    assert krum < 64 << 20
    assert L.afl_batched_workspace_bytes(b"TrimmedMean", 256, 10, 79_510, nat.AFL_F32) == 256
