"""CPU checks of the attack-success entry points afl_attack_metrics_batched, afl_attack_metrics_batched_each and
afl_metrics_workspace_bytes, and of batched.attack_metrics' arguments: everything below is rejected before any CUDA
call, so these run without a GPU."""
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


def scalar(nat, f=2, G=P, batch=2, stride=10 * 64, n=10, d=64, ld=64, dtype=None, agg=P, idx=None, sel=None, sel_ld=6,
           dev=P, sums=None, honest=None, hit=None, mal=None, cnt=None, ws=P, ws_bytes=BIG):
    dtype = nat.AFL_F32 if dtype is None else dtype
    return nat.lib().afl_attack_metrics_batched(G, batch, stride, n, d, ld, dtype, f, agg, idx, sel, sel_ld, dev, sums,
                                                honest, hit, mal, cnt, ws, ws_bytes, None)


def each(nat, fs, G=P, batch=None, stride=10 * 64, n=10, d=64, ld=64, agg=P, idx=None, dev=P, ws=P, ws_bytes=BIG):
    batch = len(fs) if batch is None else batch
    return nat.lib().afl_attack_metrics_batched_each(G, batch, stride, n, d, ld, nat.AFL_F32, fs, agg, idx, None, 0, dev,
                                                     None, None, None, None, None, ws, ws_bytes, None)


def test_workspace_bytes(nat):
    need = nat.lib().afl_metrics_workspace_bytes
    for bad in ((0, 10, 64, nat.AFL_F32), (65536, 10, 64, nat.AFL_F32), (4, 0, 64, nat.AFL_F32), (4, 10, 0, nat.AFL_F32),
                (4, 10, 64, 7)):
        assert need(*bad) == 0
    assert need(4, 300, 64, nat.AFL_F32) > 0                                    # no client limit
    assert need(4, 10, 79_510, nat.AFL_BF16) == need(4, 10, 79_510, nat.AFL_F16)
    assert need(4, 10, 79_510, nat.AFL_F32) > need(4, 10, 79_510, nat.AFL_F16)  # 1024- against 2048-column tiles
    assert need(252, 10, 79_510, nat.AFL_F32) > need(4, 10, 79_510, nat.AFL_F32)
    assert need(4, 10, 11_200_000, nat.AFL_F32) > need(4, 10, 79_510, nat.AFL_F32)
    tiles = -(-79_510 // 1024)
    assert need(252, 10, 79_510, nat.AFL_F32) >= 252 * tiles * 16
    assert need(252, 10, 79_510, nat.AFL_F32) % 256 == 0


def test_scalar_call_rejects_bad_arguments(nat):
    L = nat.lib()
    assert scalar(nat, G=None) == nat.AFL_ERR_BAD_ARG
    assert b"afl_attack_metrics_batched" in L.afl_last_error()
    assert scalar(nat, batch=0) == nat.AFL_ERR_BAD_ARG
    assert b"batch" in L.afl_last_error()
    assert scalar(nat, batch=65536) == nat.AFL_ERR_UNSUPPORTED
    assert scalar(nat, stride=9 * 64 + 63) == nat.AFL_ERR_BAD_ARG
    assert b"overlap" in L.afl_last_error()
    assert scalar(nat, agg=P, idx=P) == nat.AFL_ERR_BAD_ARG
    assert b"not both" in L.afl_last_error()
    assert scalar(nat, f=-1) == nat.AFL_ERR_BAD_ARG
    assert b"negative" in L.afl_last_error()
    assert scalar(nat, dtype=7) == nat.AFL_ERR_UNSUPPORTED
    assert b"dtype" in L.afl_last_error()
    # an output without the input it is computed from
    assert scalar(nat, agg=None) == nat.AFL_ERR_BAD_ARG
    assert scalar(nat, hit=P) == nat.AFL_ERR_BAD_ARG
    assert scalar(nat, mal=P) == nat.AFL_ERR_BAD_ARG
    assert scalar(nat, sel=P, sel_ld=0, cnt=P) == nat.AFL_ERR_BAD_ARG
    assert b"sel_ld" in L.afl_last_error()


def test_workspace_is_checked(nat):
    L = nat.lib()
    need = L.afl_metrics_workspace_bytes(2, 10, 64, nat.AFL_F32)
    for kw in ({"ws": None}, {"ws_bytes": need - 1}, {"ws": ctypes.c_void_p(128)}):
        assert scalar(nat, **kw) == nat.AFL_ERR_WORKSPACE
        assert b"workspace" in L.afl_last_error()
        assert each(nat, counts(1, 2), **kw) == nat.AFL_ERR_WORKSPACE
    # the honest mean alone also runs the column pass
    assert scalar(nat, agg=None, dev=None, honest=P, ws=None) == nat.AFL_ERR_WORKSPACE


def test_each_call_rejects_bad_counts(nat):
    L = nat.lib()
    assert each(nat, None, batch=3) == nat.AFL_ERR_BAD_ARG
    assert b"NULL" in L.afl_last_error()
    assert each(nat, counts(1, -1, 3)) == nat.AFL_ERR_BAD_ARG
    assert b"problem 1" in L.afl_last_error()
    assert each(nat, counts(1, 2), G=None) == nat.AFL_ERR_BAD_ARG
    assert b"afl_attack_metrics_batched_each" in L.afl_last_error()
    assert each(nat, counts(1), batch=0) == nat.AFL_ERR_BAD_ARG
    assert each(nat, counts(1, 2), stride=64) == nat.AFL_ERR_BAD_ARG
    assert each(nat, counts(1, 2), agg=P, idx=P) == nat.AFL_ERR_BAD_ARG
    # f_b >= n is a problem without honest rows (NaN), not an error: the call gets as far as its workspace
    assert each(nat, counts(10, 11), ws=None) == nat.AFL_ERR_WORKSPACE
    with pytest.raises(ValueError, match="problem 1"):
        nat.check(each(nat, counts(1, -1, 3)))


def test_python_arguments():
    torch = pytest.importorskip("torch")
    from attacking_federate_learning_b200 import batched as bt
    G = torch.zeros((3, 10, 64))
    with pytest.raises(ValueError, match="one value per problem"):
        bt.attack_metrics(G, [1, 2])
    with pytest.raises(ValueError):
        bt.attack_metrics(G, np.zeros((3, 1), np.int32))
    with pytest.raises(TypeError, match="integers"):
        bt.attack_metrics(G, [1.0, 2.5, 0.0])
    with pytest.raises(TypeError, match="torch.cuda"):                        # no host-matrix form
        bt.attack_metrics(G, [1, 2, 0])
