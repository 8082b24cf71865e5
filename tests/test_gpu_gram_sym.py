"""GPU tests of the one-tile symmetric bf16x2 Gram form (49 <= N <= 112, D >= 32768), which issues wgmma.m64nNk16 with
N = the client count rounded up to 8, one kernel instance per N.

Every instantiated width is checked against the float64 reference (oracle/c_oracle.py, or the same arithmetic in torch
at D = 2^20) with the caps of test_gpu_edges.py's symmetric-form test; the partial last float4 of each row is checked
on storage that ends at the matrix's last element.
"""
import numpy as np
import pytest

from oracle import c_oracle as co
from test_gpu_edges import gram_centre, hetero, table_checks

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("no GPU")
    from attacking_federate_learning_b200 import _device, _native
    _native.lib()
    return _device


def sqdist_ref_gpu(Gd):
    """float64 sums of squared fl32(g_i - g_j), one row at a time on the GPU."""
    n = Gd.shape[0]
    out = torch.empty((n, n), dtype=torch.float64, device="cuda")
    for i in range(n):
        diff = (Gd[i][None, :] - Gd).double()
        out[i] = (diff * diff).sum(1)
    return out.cpu().numpy()


def check_sym_table(d2, ref2, G):
    n = len(d2)
    k = n // 2                                                             # row k is a copy of row 0
    assert d2[0, k] == 0.0 and d2[k, 0] == 0.0
    others = np.r_[1:k, k + 1:n]
    assert np.array_equal(d2[0, others], d2[k, others])                   # identical rows: identical table rows
    x = (G - gram_centre(G)).astype(np.float64)
    table_checks(d2, ref2, 4e-5, norms=(x ** 2).sum(1))                   # symmetric, zero diagonal, operand-norm cap
    table_checks(d2, ref2, 1e-5, spread_cap=5e-6)                          # centred: error relative to the distance


@pytest.mark.parametrize("n,d", [(n, 32768 + 36) for n in (49, 56, 57, 64, 72, 80, 88, 96, 100, 104, 112)]
                         + [(100, (1 << 20) + 4)])
def test_gram_sym_widths(dev, n, d):
    rng = np.random.default_rng(16000 + n + d)
    buf = np.zeros((n, d + 4), np.float32)
    buf[:, :d] = hetero(rng, n, d)
    buf[n // 2] = buf[0]
    Gd = torch.from_numpy(buf).cuda()[:, :d]
    d2 = dev.sqdist_partial(Gd).cpu().numpy()
    G = buf[:, :d]
    ref2 = co.pairwise_sqdist(np.ascontiguousarray(G)) if d < (1 << 20) else sqdist_ref_gpu(Gd)
    check_sym_table(d2, ref2, G)


@pytest.mark.parametrize("r", [1, 2, 3])
def test_gram_sym_storage_ends_at_last_element(dev, r):
    """d % 4 = r: the last row's partial float4 is the last thing in the allocation, and the table must equal, bit for
    bit, the one of the same matrix in padded storage."""
    n, d = 100, 32768 + 64 + r
    ld = (d + 3) // 4 * 4
    rng = np.random.default_rng(17000 + r)
    G = hetero(rng, n, d)
    G[n // 2] = G[0]
    flat = torch.zeros(((n - 1) * ld + d,), dtype=torch.float32, device="cuda")
    tight = torch.as_strided(flat, (n, d), (ld, 1))
    tight.copy_(torch.from_numpy(G).cuda())
    padded = torch.zeros((n, ld + 8), dtype=torch.float32, device="cuda")
    padded[:, :d] = torch.from_numpy(G).cuda()
    got = dev.sqdist_partial(tight).cpu().numpy()
    want = dev.sqdist_partial(padded[:, :d]).cpu().numpy()
    assert np.array_equal(got, want)
    check_sym_table(got, co.pairwise_sqdist(G), G)
