"""CPU checks of the device-parameter batched entry points (afl_batched_table_dev, afl_defend_batched_dev,
afl_alie_batched_dev, afl_attack_metrics_batched_dev) and of batched.DeviceRound's construction: NULL pointers, batch
limits, N > 128 for the defences, dtype, Bulyan's selection width and short or misaligned workspaces are rejected on
the host before any CUDA call, so these run without a GPU."""
import ctypes
import os
import re

import pytest
import torch

P = ctypes.c_void_p(256)         # a non-NULL pointer that is never dereferenced: validation fails first
NULL = ctypes.c_void_p()
BIG = 1 << 30
RULES = (b"Krum", b"Bulyan", b"TrimmedMean", b"NoDefense")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DEV_CALLS = ("afl_batched_table_dev", "afl_defend_batched_dev", "afl_alie_batched_dev", "afl_attack_metrics_batched_dev")


@pytest.fixture(scope="module")
def nat():
    import __graft_entry__ as g
    g.build()
    from attacking_federate_learning_b200 import _native
    _native.lib()
    return _native


def defend(nat, rule=b"TrimmedMean", G=P, batch=3, n=12, d=64, ld=64, stride=None, dtype=0, fs=P, out=P, idx=P, sel=P,
           sel_ld=None, ws=P, ws_bytes=BIG, status=P, rows=None):
    stride = n * ld if stride is None else stride
    sel_ld = n if sel_ld is None else sel_ld
    return nat.lib().afl_defend_batched_dev(rule, G, batch, stride, n, d, ld, dtype, rows, n, None, fs, out, idx, sel,
                                            sel_ld, ws, ws_bytes, status, None)


def alie(nat, G=P, batch=3, n=12, d=64, dtype=0, fs=P, zs=P, bcast=None, bcast_stride=None, ws=P, ws_bytes=BIG,
         status=P):
    bcast_stride = n * 64 if bcast_stride is None else bcast_stride
    return nat.lib().afl_alie_batched_dev(G, batch, n * 64, n, d, 64, dtype, fs, zs, P, P, P, bcast, bcast_stride, 64,
                                          ws, ws_bytes, status, None)


def metrics(nat, G=P, batch=3, n=12, dtype=0, fs=P, agg=P, idx=None, ws=P, ws_bytes=BIG, status=P):
    return nat.lib().afl_attack_metrics_batched_dev(G, batch, n * 64, n, 64, 64, dtype, None, fs, agg, idx, None, 0, P,
                                                    None, None, None, None, None, ws, ws_bytes, status, None)


def table(nat, rule=b"Krum", batch=3, n=12, fs=P, zs=None, ws=P, ws_bytes=BIG, status=P):
    return nat.lib().afl_batched_table_dev(rule, batch, n, None, n, None, fs, zs, ws, ws_bytes, status, None)


def test_null_pointers_are_rejected(nat):
    for rule in RULES:
        assert defend(nat, rule, G=NULL) == nat.AFL_ERR_BAD_ARG
        assert defend(nat, rule, fs=NULL) == nat.AFL_ERR_BAD_ARG
        assert defend(nat, rule, status=NULL) == nat.AFL_ERR_BAD_ARG
        assert b"NULL" in nat.lib().afl_last_error()
    assert defend(nat, b"Krum", idx=NULL) == nat.AFL_ERR_BAD_ARG
    assert defend(nat, b"Bulyan", sel=NULL) == nat.AFL_ERR_BAD_ARG
    assert defend(nat, b"TrimmedMean", out=NULL) == nat.AFL_ERR_BAD_ARG
    assert defend(nat, b"Nope") == nat.AFL_ERR_BAD_ARG
    for kw in ("G", "fs", "zs", "status"):
        assert alie(nat, **{kw: NULL}) == nat.AFL_ERR_BAD_ARG
    for kw in ("G", "fs", "status"):
        assert metrics(nat, **{kw: NULL}) == nat.AFL_ERR_BAD_ARG
    assert metrics(nat, agg=P, idx=P) == nat.AFL_ERR_BAD_ARG           # both aggregates
    assert table(nat, fs=NULL) == nat.AFL_ERR_BAD_ARG
    assert table(nat, status=NULL) == nat.AFL_ERR_BAD_ARG
    assert table(nat, rule=b"ALIE", zs=None) == nat.AFL_ERR_BAD_ARG
    assert table(nat, rule=b"Nope") == nat.AFL_ERR_BAD_ARG


def test_batch_limits(nat):
    for rule in RULES:
        assert defend(nat, rule, batch=0) == nat.AFL_ERR_BAD_ARG
        assert defend(nat, rule, batch=65536) == nat.AFL_ERR_UNSUPPORTED
        assert defend(nat, rule, stride=12 * 64 - 1) == nat.AFL_ERR_BAD_ARG        # problems overlap
    assert alie(nat, batch=0) == nat.AFL_ERR_BAD_ARG
    assert alie(nat, batch=65536) == nat.AFL_ERR_UNSUPPORTED
    assert metrics(nat, batch=0) == nat.AFL_ERR_BAD_ARG
    assert metrics(nat, batch=65536) == nat.AFL_ERR_UNSUPPORTED
    assert table(nat, batch=0) == nat.AFL_ERR_BAD_ARG
    assert table(nat, batch=65536) == nat.AFL_ERR_UNSUPPORTED
    assert table(nat, n=0) == nat.AFL_ERR_BAD_ARG


def test_defences_need_one_gram_tile(nat):
    for rule in RULES:
        assert defend(nat, rule, n=129) == nat.AFL_ERR_UNSUPPORTED
        assert b"128" in nat.lib().afl_last_error()
        assert defend(nat, rule, n=128, ws_bytes=0) == nat.AFL_ERR_WORKSPACE      # 128 passes the limit
    # ALIE and the metrics take any N: they fail on the workspace, not the client count
    assert alie(nat, n=1000, ws_bytes=0) == nat.AFL_ERR_WORKSPACE
    assert metrics(nat, n=1000, ws_bytes=0) == nat.AFL_ERR_WORKSPACE


def test_dtype_is_checked(nat):
    for rule in RULES:
        assert defend(nat, rule, dtype=7) == nat.AFL_ERR_UNSUPPORTED
    assert alie(nat, dtype=7) == nat.AFL_ERR_UNSUPPORTED
    assert metrics(nat, dtype=7) == nat.AFL_ERR_UNSUPPORTED


def test_bulyan_selection_width(nat):
    assert defend(nat, b"Bulyan", sel_ld=11) == nat.AFL_ERR_BAD_ARG
    assert b"sel_ld" in nat.lib().afl_last_error()
    assert defend(nat, b"Bulyan", sel_ld=12, ws_bytes=0) == nat.AFL_ERR_WORKSPACE


def test_workspace_size_and_alignment(nat):
    L = nat.lib()
    for rule in RULES:
        need = L.afl_batched_rows_workspace_bytes(rule, 3, 12, 64, 0)
        assert defend(nat, rule, ws_bytes=need - 1) == nat.AFL_ERR_WORKSPACE
        assert defend(nat, rule, ws=ctypes.c_void_p(264)) == nat.AFL_ERR_WORKSPACE
        assert defend(nat, rule, ws=NULL) == nat.AFL_ERR_WORKSPACE
    need = L.afl_batched_each_workspace_bytes(b"ALIE", 3, 1, 64, 0)
    assert alie(nat, ws_bytes=need - 1) == nat.AFL_ERR_WORKSPACE
    need = L.afl_metrics_workspace_bytes(3, 12, 64, 0)
    assert metrics(nat, ws_bytes=need - 1) == nat.AFL_ERR_WORKSPACE
    assert table(nat, ws_bytes=3 * 40 - 1) == nat.AFL_ERR_WORKSPACE
    assert table(nat, ws=ctypes.c_void_p(264)) == nat.AFL_ERR_WORKSPACE


def test_alie_written_rows_must_not_overlap(nat):
    assert alie(nat, bcast=P, bcast_stride=11 * 64 + 63) == nat.AFL_ERR_BAD_ARG


def test_ctypes_table_matches_header_for_device_calls(nat):
    text = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "afl_b200.h")).read(), flags=re.S)
    for name in DEV_CALLS:
        m = re.search(rf"\b{name}\s*\(([^)]*)\)", text)
        assert m, name
        assert len(nat.SIGNATURES[name][1]) == len(m.group(1).split(",")), name
        assert hasattr(ctypes.CDLL(nat.LIB_PATH), name)


def test_device_round_rejects_bad_arguments():
    from attacking_federate_learning_b200.batched import DeviceRound
    G = torch.zeros(2, 10, 32)
    with pytest.raises(TypeError):
        DeviceRound(G.numpy())
    with pytest.raises(ValueError):
        DeviceRound(G[0])                                          # not [B, N, D]
    with pytest.raises(ValueError):
        DeviceRound(G.transpose(1, 2))                             # stride(2) != 1
    with pytest.raises(ValueError):
        DeviceRound(G, rules=("Median",))
    with pytest.raises(NotImplementedError):
        DeviceRound(torch.zeros(2, 129, 32))                       # defences need one Gram tile
    with pytest.raises(ValueError):
        DeviceRound(G, per_problem_users_count=True)               # needs rows
    with pytest.raises(ValueError):
        DeviceRound(G, 10, rows=True)                              # with rows, users_count is rows or per problem
    with pytest.raises(ValueError):
        DeviceRound(torch.zeros(0, 10, 32))
    with pytest.raises(NotImplementedError):
        DeviceRound(G.double())
    with pytest.raises(TypeError):
        DeviceRound(G)                                             # valid, but not on a GPU
    with pytest.raises(TypeError):
        DeviceRound(torch.zeros(2, 129, 32), rules=())             # ALIE and metrics alone take any N
