"""CPU checks of the device-parameter large batched call (afl_defend_batched_large_dev, afl_batched_large_dev_workspace_bytes)
and of batched.DeviceRound(large=True)'s construction: the client limit of 1024, NULL pointers, batch limits, dtype,
overlapping strides, Bulyan's selection width and short or misaligned workspaces are rejected on the host before any
CUDA call, so these run without a GPU."""
import ctypes
import os
import re

import pytest
import torch

P = ctypes.c_void_p(256)         # a non-NULL pointer that is never dereferenced: validation fails first
NULL = ctypes.c_void_p()
BIG = 1 << 40
RULES = (b"Krum", b"Bulyan", b"TrimmedMean", b"NoDefense")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NEW_CALLS = ("afl_batched_large_dev_workspace_bytes", "afl_defend_batched_large_dev")


@pytest.fixture(scope="module")
def nat():
    import __graft_entry__ as g
    g.build()
    from attacking_federate_learning_b200 import _native
    _native.lib()
    return _native


def defend(nat, rule=b"TrimmedMean", G=P, batch=3, n=500, d=64, ld=64, stride=None, dtype=0, fs=P, out=P, idx=P, sel=P,
           sel_ld=None, ws=P, ws_bytes=BIG, status=P, rows=None):
    stride = n * ld if stride is None else stride
    sel_ld = n if sel_ld is None else sel_ld
    return nat.lib().afl_defend_batched_large_dev(rule, G, batch, stride, n, d, ld, dtype, rows, n, None, fs, out, idx,
                                                  sel, sel_ld, ws, ws_bytes, status, None)


def test_new_symbols_match_the_header(nat):
    text = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "afl_b200.h")).read(), flags=re.S)
    for name in NEW_CALLS:
        m = re.search(rf"\b{name}\s*\(([^)]*)\)", text)
        assert m, name
        assert len(nat.SIGNATURES[name][1]) == len(m.group(1).split(",")), name
        assert hasattr(ctypes.CDLL(nat.LIB_PATH), name)
    # the large call takes afl_defend_batched_dev's argument list
    assert nat.SIGNATURES["afl_defend_batched_large_dev"] == nat.SIGNATURES["afl_defend_batched_dev"]


def test_client_limit_is_1024(nat):
    for rule in RULES:
        assert defend(nat, rule, n=1025) == nat.AFL_ERR_UNSUPPORTED
        assert b"1024" in nat.lib().afl_last_error()
        for n in (129, 1024):                                        # past the one-tile limit: fails on the workspace
            assert defend(nat, rule, n=n, ws_bytes=0) == nat.AFL_ERR_WORKSPACE
        assert defend(nat, rule, n=128, ws_bytes=0) == nat.AFL_ERR_WORKSPACE


def test_null_pointers_are_rejected(nat):
    for n in (100, 500):
        for rule in RULES:
            assert defend(nat, rule, n=n, G=NULL) == nat.AFL_ERR_BAD_ARG
            assert defend(nat, rule, n=n, fs=NULL) == nat.AFL_ERR_BAD_ARG
            assert defend(nat, rule, n=n, status=NULL) == nat.AFL_ERR_BAD_ARG
            assert b"NULL" in nat.lib().afl_last_error()
        assert defend(nat, b"Krum", n=n, idx=NULL) == nat.AFL_ERR_BAD_ARG
        assert defend(nat, b"Bulyan", n=n, sel=NULL) == nat.AFL_ERR_BAD_ARG
        assert defend(nat, b"TrimmedMean", n=n, out=NULL) == nat.AFL_ERR_BAD_ARG
        assert defend(nat, b"NoDefense", n=n, out=NULL) == nat.AFL_ERR_BAD_ARG
        assert defend(nat, b"Nope", n=n) == nat.AFL_ERR_BAD_ARG


def test_bulyan_selection_width(nat):
    assert defend(nat, b"Bulyan", sel_ld=499) == nat.AFL_ERR_BAD_ARG
    assert b"sel_ld" in nat.lib().afl_last_error()
    assert defend(nat, b"Bulyan", sel_ld=500, ws_bytes=0) == nat.AFL_ERR_WORKSPACE


def test_shape_limits(nat):
    for rule in RULES:
        assert defend(nat, rule, dtype=7) == nat.AFL_ERR_UNSUPPORTED
        assert defend(nat, rule, batch=0) == nat.AFL_ERR_BAD_ARG
        assert defend(nat, rule, batch=65536) == nat.AFL_ERR_UNSUPPORTED
        assert defend(nat, rule, stride=499 * 64 + 63) == nat.AFL_ERR_BAD_ARG      # problems overlap
        assert defend(nat, rule, batch=1, stride=0, ws_bytes=0) == nat.AFL_ERR_WORKSPACE   # one problem: no stride


def test_workspace_query(nat):
    L = nat.lib()
    for rule in RULES:
        for d, dtype in ((64, 0), (79520, 0), (1000, 1), (1000, 2)):
            assert L.afl_batched_large_dev_workspace_bytes(rule, 4, 1025, d, dtype) == 0
            for n in (1, 100, 128):
                assert L.afl_batched_large_dev_workspace_bytes(rule, 4, n, d, dtype) == \
                    L.afl_batched_rows_workspace_bytes(rule, 4, n, d, dtype)
            for n in (129, 500, 1000, 1024):
                large = L.afl_batched_large_workspace_bytes(rule, 4, n, d, dtype)
                assert large > 0
                assert L.afl_batched_large_dev_workspace_bytes(rule, 4, n, d, dtype) == large + 256
        assert L.afl_batched_large_dev_workspace_bytes(rule, 0, 500, 64, 0) == 0
        assert L.afl_batched_large_dev_workspace_bytes(rule, 65536, 500, 64, 0) == 0
        assert L.afl_batched_large_dev_workspace_bytes(rule, 4, 500, 64, 7) == 0
    assert L.afl_batched_large_dev_workspace_bytes(b"Nope", 4, 500, 64, 0) == 0


def test_workspace_size_and_alignment(nat):
    L = nat.lib()
    for n in (100, 500, 1000):
        for rule in RULES:
            need = L.afl_batched_large_dev_workspace_bytes(rule, 3, n, 64, 0)
            assert defend(nat, rule, n=n, ws_bytes=need - 1) == nat.AFL_ERR_WORKSPACE
            assert defend(nat, rule, n=n, ws=ctypes.c_void_p(264)) == nat.AFL_ERR_WORKSPACE
            assert defend(nat, rule, n=n, ws=NULL) == nat.AFL_ERR_WORKSPACE


def test_device_round_large_limits():
    from attacking_federate_learning_b200.batched import DeviceRound
    with pytest.raises(TypeError):
        DeviceRound(torch.zeros(2, 129, 32), large=True)               # passes the limit, then: not on a GPU
    with pytest.raises(TypeError):
        DeviceRound(torch.zeros(2, 1024, 32), large=True)
    with pytest.raises(NotImplementedError):
        DeviceRound(torch.zeros(2, 1025, 32), large=True)
    with pytest.raises(NotImplementedError):
        DeviceRound(torch.zeros(2, 129, 32))                           # without large=True the defences stop at 128
    with pytest.raises(TypeError):
        DeviceRound(torch.zeros(2, 1025, 32), large=True, rules=())    # ALIE and metrics alone take any N
