"""CPU checks of fp16 client matrices (AFL_F16) at the C ABI and in the Python plumbing: the workspace sizes equal the
bf16 ones, the dtype checks accept AFL_F16 and still reject any other code, and the NumPy host path stays fp32-only.
Every call here fails its argument checks before any CUDA call, so these run without a GPU."""
import ctypes

import numpy as np
import pytest

P = ctypes.c_void_p(256)         # a non-NULL pointer that is never dereferenced: validation fails first
BAD_DTYPE = 3


@pytest.fixture(scope="module")
def nat():
    import __graft_entry__ as g
    g.build()
    from attacking_federate_learning_b200 import _native
    _native.lib()
    return _native


def test_f16_code(nat):
    assert nat.AFL_F16 == 2 and len({nat.AFL_F32, nat.AFL_BF16, nat.AFL_F16}) == 3


@pytest.mark.parametrize("n,d", [(1, 1), (10, 79_510), (100, 11_200_000), (129, 4_096), (1000, 10_000), (4096, 64),
                                 (4097, 64)])
def test_sqdist_workspace_equals_bf16(nat, n, d):
    L = nat.lib()
    for flags in (0, nat.GRAM_FORCE_SIMT, nat.GRAM_TF32X2, nat.GRAM_NO_CENTER):
        assert L.afl_sqdist_workspace_bytes(n, d, nat.AFL_F16, flags) == L.afl_sqdist_workspace_bytes(n, d, nat.AFL_BF16, flags)


@pytest.mark.parametrize("rule", [b"Krum", b"Bulyan", b"TrimmedMean", b"NoDefense"])
@pytest.mark.parametrize("batch,n,d", [(1, 10, 79_510), (256, 10, 79_510), (4, 51, 8_192), (3, 128, 8_192)])
def test_batched_workspace_equals_bf16(nat, rule, batch, n, d):
    L = nat.lib()
    assert L.afl_batched_workspace_bytes(rule, batch, n, d, nat.AFL_F16) == \
        L.afl_batched_workspace_bytes(rule, batch, n, d, nat.AFL_BF16) > 0
    assert L.afl_batched_each_workspace_bytes(rule, batch, n, d, nat.AFL_F16) == \
        L.afl_batched_each_workspace_bytes(rule, batch, n, d, nat.AFL_BF16) > 0
    assert L.afl_batched_each_workspace_bytes(b"ALIE", batch, n, d, nat.AFL_F16) == \
        L.afl_batched_each_workspace_bytes(b"ALIE", batch, n, d, nat.AFL_BF16)


def last_error(nat):
    return nat.lib().afl_last_error()


def test_f16_passes_the_dtype_checks(nat):
    """AFL_F16 gets past each dtype check to the next argument check; code 3 stops at the dtype check."""
    L = nat.lib()
    F16 = nat.AFL_F16
    # batched: the dtype check comes before the output checks
    for dt, rc, msg in ((F16, nat.AFL_ERR_BAD_ARG, b"needs idx_out"), (BAD_DTYPE, nat.AFL_ERR_UNSUPPORTED, b"dtype")):
        assert L.afl_defend_batched(b"Krum", P, 4, 640, 10, 64, 64, dt, 10, 2, P, None, P, P, 1 << 30, None) == rc
        assert msg in last_error(nat)
        fs = (ctypes.c_int * 4)(2, 2, 2, 2)
        assert L.afl_defend_batched_each(b"Krum", P, 4, 640, 10, 64, 64, dt, 10, fs, P, None, P, P, 1 << 30, None) == rc
        assert msg in last_error(nat)
    # trimmed mean: the row limit is checked after the dtype
    for dt, msg in ((F16, b"at most 12288"), (BAD_DTYPE, b"dtype")):
        assert L.afl_trimmed_mean(P, 12289, 64, 64, dt, None, 12289, 0, P, None) == nat.AFL_ERR_UNSUPPORTED
        assert msg in last_error(nat)
    # distance table: the workspace is checked after the dtype
    assert L.afl_sqdist_partial(P, 10, 64, 64, F16, P, None, 0, 0, None) == nat.AFL_ERR_WORKSPACE
    assert L.afl_sqdist_partial(P, 10, 64, 64, BAD_DTYPE, P, None, 0, 0, None) == nat.AFL_ERR_UNSUPPORTED
    assert b"dtype" in last_error(nat)
    # forcing the tensor path on an unaligned fp16 pitch is refused like bf16 (7 elements: not a 16-byte pitch)
    for dt in (nat.AFL_BF16, F16):
        assert L.afl_sqdist_partial(P, 10, 7, 7, dt, P, P, 1 << 30, nat.GRAM_FORCE_TCGEN05, None) == nat.AFL_ERR_UNSUPPORTED
        assert b"tensor-core path" in last_error(nat)


def test_code_3_is_rejected_everywhere(nat):
    L = nat.lib()
    U = nat.AFL_ERR_UNSUPPORTED
    assert L.afl_mean(P, 10, 64, 64, BAD_DTYPE, P, None) == U
    assert L.afl_gather_row(P, 10, 64, 64, BAD_DTYPE, P, P, None) == U
    assert L.afl_alie(P, 4, 64, 64, BAD_DTYPE, 1.5, P, P, P, None, 0, None) == U
    assert L.afl_alie_batched(P, 4, 640, 2, 64, 64, BAD_DTYPE, 1.5, P, P, P, None, 0, 64, None) == U
    fs = (ctypes.c_int * 4)(2, 2, 2, 2)
    zs = (ctypes.c_double * 4)(1.5, 1.5, 1.5, 1.5)
    assert L.afl_alie_batched_each(P, 4, 640, 10, 64, 64, BAD_DTYPE, fs, zs, P, P, P, None, 0, 64, P, 1 << 30, None) == U
    for rule in (b"Krum", b"Bulyan", b"TrimmedMean", b"NoDefense"):
        assert L.afl_defend_batched(rule, P, 4, 640, 10, 64, 64, BAD_DTYPE, 10, 1, P, P, P, P, 1 << 30, None) == U
        assert b"dtype" in last_error(nat)


def test_dtype_code_maps_float16(nat):
    torch = pytest.importorskip("torch")
    from attacking_federate_learning_b200 import _device as dev
    assert dev.dtype_code(torch.zeros(2, 2, dtype=torch.float16)) == nat.AFL_F16
    assert dev.dtype_code(torch.zeros(2, 2, dtype=torch.bfloat16)) == nat.AFL_BF16
    assert dev.dtype_code(torch.zeros(2, 2, dtype=torch.float32)) == nat.AFL_F32
    for dt in (torch.float64, torch.int16, torch.uint8):
        with pytest.raises(NotImplementedError):
            dev.dtype_code(torch.zeros(2, 2, dtype=dt))


def test_numpy_float16_stays_unsupported_on_the_host_path(nat):
    from attacking_federate_learning_b200 import defences as D
    G = np.ones((11, 64), np.float16)
    for call in (lambda: D.no_defense(G, 11, 2), lambda: D.trimmed_mean(G, 11, 2), lambda: D.krum(G, 11, 2),
                 lambda: D.krum(G, 11, 2, return_index=True), lambda: D.bulyan(G, 11, 2),
                 lambda: D._krum_create_distances(G)):
        with pytest.raises(NotImplementedError):
            call()
