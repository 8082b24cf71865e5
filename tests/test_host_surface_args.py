"""CPU checks of the host-buffer entry points afl_sqdist_host, afl_bulyan_host and afl_alie_host: null pointers and
bad sizes are rejected with AFL_ERR_BAD_ARG, and the reference's Bulyan assert with AFL_ERR_PRECONDITION, before any
CUDA call (so these run without a GPU).  The NumPy ALIE route rejects mismatched gradients before it touches the
library."""
import ctypes

import numpy as np
import pytest

P = ctypes.c_void_p(16)          # a non-NULL pointer that is never dereferenced: validation fails first


@pytest.fixture(scope="module")
def nat():
    import __graft_entry__ as g
    g.build()
    from attacking_federate_learning_b200 import _native
    _native.lib()
    return _native


def test_sqdist_host_rejects_bad_arguments(nat):
    L = nat.lib()
    assert L.afl_sqdist_host(None, 4, 8, 8, P, 0) == nat.AFL_ERR_BAD_ARG
    assert b"afl_sqdist_host" in L.afl_last_error()
    assert L.afl_sqdist_host(P, 4, 8, 8, None, 0) == nat.AFL_ERR_BAD_ARG
    assert L.afl_sqdist_host(P, 0, 8, 8, P, 0) == nat.AFL_ERR_BAD_ARG
    assert L.afl_sqdist_host(P, 4, 0, 8, P, 0) == nat.AFL_ERR_BAD_ARG
    assert L.afl_sqdist_host(P, 4, 8, 7, P, 0) == nat.AFL_ERR_BAD_ARG


def test_bulyan_host_rejects_bad_arguments(nat):
    L = nat.lib()
    assert L.afl_bulyan_host(None, 11, 8, 8, 11, 2, P, P, 0) == nat.AFL_ERR_BAD_ARG
    assert b"afl_bulyan_host" in L.afl_last_error()
    assert L.afl_bulyan_host(P, 11, 8, 8, 11, 2, None, P, 0) == nat.AFL_ERR_BAD_ARG
    assert L.afl_bulyan_host(P, 0, 8, 8, 11, 2, P, P, 0) == nat.AFL_ERR_BAD_ARG
    assert L.afl_bulyan_host(P, 11, -1, 8, 11, 2, P, P, 0) == nat.AFL_ERR_BAD_ARG
    assert L.afl_bulyan_host(P, 11, 8, 4, 11, 2, P, P, 0) == nat.AFL_ERR_BAD_ARG


def test_bulyan_host_precondition_and_client_limit(nat):
    L = nat.lib()
    # n < 4f + 3: the reference's assert (defences.py:56)
    assert L.afl_bulyan_host(P, 10, 8, 8, 10, 2, P, P, 0) == nat.AFL_ERR_PRECONDITION
    assert b"4*corrupted_count + 3" in L.afl_last_error()
    assert L.afl_bulyan_host(P, 10, 8, 8, 10, 2, P, None, 0) == nat.AFL_ERR_PRECONDITION
    # selection supports n <= 4096 clients; refused before any copy or launch
    assert L.afl_bulyan_host(P, 4097, 8, 8, 4097, 2, P, P, 0) == nat.AFL_ERR_UNSUPPORTED
    assert b"n <= 4096" in L.afl_last_error()


def test_alie_host_rejects_bad_arguments(nat):
    L = nat.lib()
    a = np.zeros(8, np.float32)
    rows = (ctypes.c_void_p * 2)(a.ctypes.data, a.ctypes.data)
    assert L.afl_alie_host(None, 2, 8, 1.5, P, P, P, 0) == nat.AFL_ERR_BAD_ARG
    assert b"afl_alie_host" in L.afl_last_error()
    assert L.afl_alie_host(rows, 0, 8, 1.5, P, P, P, 0) == nat.AFL_ERR_BAD_ARG
    assert L.afl_alie_host(rows, 2, 0, 1.5, P, P, P, 0) == nat.AFL_ERR_BAD_ARG
    holes = (ctypes.c_void_p * 2)(a.ctypes.data, None)
    assert L.afl_alie_host(holes, 2, 8, 1.5, P, P, P, 0) == nat.AFL_ERR_BAD_ARG
    assert b"rows[1]" in L.afl_last_error()


class _User:
    def __init__(self, grads):
        self.grads = grads
        self.original_params = None
        self.learning_rate = 0.1


def test_numpy_attack_rejects_mismatched_gradients(nat):
    from attacking_federate_learning_b200 import malicious as M
    users = [_User(np.zeros(8, np.float32)), _User(np.zeros(9, np.float32))]
    with pytest.raises(ValueError, match="same shape"):            # what np.stack raised
        M.DriftAttack(1.5).attack(users)
    users = [_User(np.zeros((2, 4), np.float32)), _User(np.zeros((2, 4), np.float32))]
    with pytest.raises(ValueError):
        M.DriftAttack(1.5).attack(users)
    assert all(isinstance(u.grads, np.ndarray) for u in users)     # nothing was assigned
