"""CPU checks of the backdoor entry points afl_backdoor_start_batched and afl_backdoor_finish_batched, and of the Python
arguments of batched.backdoor_rows and BackdoorAttack.attack_rows that are checked before anything needs a GPU: NULL
pointers and arrays, the batch limits, counts outside [0, n], overlapping strides and short workspaces are rejected
before any CUDA call, with the status codes of the other per-problem calls."""
import ctypes

import numpy as np
import pytest

P = ctypes.c_void_p(256)         # a non-NULL pointer that is never dereferenced: validation fails first
BIG = 1 << 30
NULL = ctypes.c_void_p()


@pytest.fixture(scope="module")
def nat():
    import __graft_entry__ as g
    g.build()
    from attacking_federate_learning_b200 import _native
    _native.lib()
    return _native


def counts(*f):
    return (ctypes.c_int * len(f))(*f)


def doubles(batch, v):
    return (ctypes.c_double * batch)(*([v] * batch))


def start(nat, fs, zs=None, lrs=None, G=P, batch=None, stride=10 * 64, n=10, d=64, ld=64, dtype=None, w=P, w_stride=0,
          mu=P, sigma=P, initial=P, ws=P, ws_bytes=BIG):
    batch = len(fs) if batch is None else batch
    zs = doubles(max(batch, 1), 1.5) if zs is None else zs
    lrs = doubles(max(batch, 1), 0.1) if lrs is None else lrs
    dtype = nat.AFL_F32 if dtype is None else dtype
    return nat.lib().afl_backdoor_start_batched(G, batch, stride, n, d, ld, dtype, fs, zs, lrs, w, w_stride, mu, sigma,
                                                initial, ws, ws_bytes, None)


def finish(nat, fs, zs=None, lrs=None, batch=None, d=64, mu=P, sigma=P, initial=P, mal=P, mal_stride=64, crafted=P,
           bcast=None, bstride=0, bld=64, ws=P, ws_bytes=BIG):
    batch = len(fs) if batch is None else batch
    zs = doubles(max(batch, 1), 1.5) if zs is None else zs
    lrs = doubles(max(batch, 1), 0.1) if lrs is None else lrs
    return nat.lib().afl_backdoor_finish_batched(batch, d, fs, zs, lrs, mu, sigma, initial, mal, mal_stride, crafted,
                                                 bcast, bstride, bld, ws, ws_bytes, None)


def test_start_rejects_bad_arguments(nat):
    L = nat.lib()
    for kw in ({"G": None}, {"w": None}, {"mu": None}, {"sigma": None}, {"initial": None}, {"d": 0}, {"ld": 63}):
        assert start(nat, counts(1, 2), **kw) == nat.AFL_ERR_BAD_ARG, kw
        assert b"afl_backdoor_start_batched" in L.afl_last_error()
    assert start(nat, None, batch=2) == nat.AFL_ERR_BAD_ARG
    assert b"NULL" in L.afl_last_error()
    assert start(nat, counts(1, 2), lrs=NULL) == nat.AFL_ERR_BAD_ARG
    assert b"NULL" in L.afl_last_error()
    assert start(nat, counts(1, 2), zs=NULL) == nat.AFL_ERR_BAD_ARG
    assert start(nat, counts(1), batch=0) == nat.AFL_ERR_BAD_ARG
    assert b"batch" in L.afl_last_error()
    assert start(nat, counts(1), batch=65536) == nat.AFL_ERR_UNSUPPORTED
    assert start(nat, counts(1, 2), dtype=3) == nat.AFL_ERR_UNSUPPORTED
    assert b"dtype" in L.afl_last_error()
    # f_b outside [0, n], naming the problem
    assert start(nat, counts(1, -1)) == nat.AFL_ERR_BAD_ARG
    assert b"problem 1" in L.afl_last_error()
    assert start(nat, counts(10, 11)) == nat.AFL_ERR_BAD_ARG
    assert b"problem 1" in L.afl_last_error()
    # overlapping problems, a w pitch that is neither shared (0) nor a full row
    assert start(nat, counts(1, 2), stride=9 * 64 + 63) == nat.AFL_ERR_BAD_ARG
    assert b"overlap" in L.afl_last_error()
    for w_stride in (-64, 1, 63):
        assert start(nat, counts(1, 2), w_stride=w_stride) == nat.AFL_ERR_BAD_ARG
        assert b"w_batch_stride" in L.afl_last_error()


def test_start_has_no_client_limit(nat):
    # n = 300 > 128 (the Gram tile of the defences) gets as far as the workspace
    assert start(nat, counts(300, 0), n=300, stride=300 * 64, ws=None) == nat.AFL_ERR_WORKSPACE


def test_finish_rejects_bad_arguments(nat):
    L = nat.lib()
    for kw in ({"mu": None}, {"sigma": None}, {"initial": None}, {"mal": None}, {"crafted": None}, {"d": 0}):
        assert finish(nat, counts(1, 2), **kw) == nat.AFL_ERR_BAD_ARG, kw
        assert b"afl_backdoor_finish_batched" in L.afl_last_error()
    assert finish(nat, None, batch=2) == nat.AFL_ERR_BAD_ARG
    assert finish(nat, counts(1, 2), lrs=NULL) == nat.AFL_ERR_BAD_ARG
    assert finish(nat, counts(1, 2), zs=NULL) == nat.AFL_ERR_BAD_ARG
    assert finish(nat, counts(1), batch=0) == nat.AFL_ERR_BAD_ARG
    assert finish(nat, counts(1), batch=65536) == nat.AFL_ERR_UNSUPPORTED
    assert finish(nat, counts(1, -2)) == nat.AFL_ERR_BAD_ARG
    assert b"problem 1" in L.afl_last_error()
    assert finish(nat, counts(1, 2), mal_stride=63) == nat.AFL_ERR_BAD_ARG
    assert b"mal_batch_stride" in L.afl_last_error()
    # written rows that overlap: within a problem (bcast_ld < d) or across problems (f_max rows per problem)
    assert finish(nat, counts(1, 2), bcast=P, bstride=10 * 64, bld=63) == nat.AFL_ERR_BAD_ARG
    assert b"overlap" in L.afl_last_error()
    assert finish(nat, counts(1, 2), bcast=P, bstride=64 + 63, bld=64) == nat.AFL_ERR_BAD_ARG
    # one batch of one, or no problem that writes, needs no batch pitch
    assert finish(nat, counts(3), mal_stride=0, bcast=P, bstride=0, ws=None) == nat.AFL_ERR_WORKSPACE
    assert finish(nat, counts(0, 0), bcast=P, bstride=0, ws=None) == nat.AFL_ERR_WORKSPACE


def test_workspace_is_checked(nat):
    L = nat.lib()
    need = L.afl_batched_each_workspace_bytes(b"ALIE", 2, 1, 64, nat.AFL_F32)
    assert need >= 2 * 40 and need % 256 == 0
    assert need == L.afl_batched_each_workspace_bytes(b"ALIE", 2, 128, 79_510, nat.AFL_BF16)   # the table: batch only
    for kw in ({"ws": None}, {"ws_bytes": need - 1}, {"ws": ctypes.c_void_p(128)}):
        assert start(nat, counts(1, 2), **kw) == nat.AFL_ERR_WORKSPACE
        assert b"workspace" in L.afl_last_error()
        assert finish(nat, counts(1, 2), **kw) == nat.AFL_ERR_WORKSPACE
    with pytest.raises(ValueError, match="problem 1"):
        nat.check(start(nat, counts(1, -1)))


def test_python_arguments():
    torch = pytest.importorskip("torch")
    from attacking_federate_learning_b200 import batched as bt, malicious as M
    G = torch.zeros((3, 10, 64))
    train = lambda x, problems: x                                                 # noqa: E731
    with pytest.raises(TypeError, match="original_params"):
        bt.backdoor_rows(G, 2, 1.5, None, 0.1, train)
    with pytest.raises(TypeError, match="original_params"):                    # a host vector is not accepted
        bt.backdoor_rows(G, 2, 1.5, torch.zeros(64), 0.1, train)
    # attack_rows without the parameters and the learning rate would silently be some other attack: refused
    att = M.BackdoorAttack(1.5, lambda p: p)
    with pytest.raises(TypeError, match="original_params and learning_rate"):
        att.attack_rows(G[0], 2)
    with pytest.raises(TypeError, match="original_params and learning_rate"):
        att.attack_rows(G[0], 2, original_params=torch.zeros(64))
    assert att.attack_rows(G[0], 0) is None                                   # malicious.py:11-12: nothing to craft
    assert att.grads_mean is None and att.grads_stdev is None
    assert np.array_equal(G.numpy(), np.zeros((3, 10, 64), np.float32))
