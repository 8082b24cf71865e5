"""GPU tests at the edges of the aggregation kernels: infinite client gradients on every route, the documented size
limits (n <= 4096 for Krum, Bulyan and the wgmma Gram, 12,288 trimmed-mean rows), and the one-tile / tiny-D shapes of
the Gram kernel.

References: oracle/ref_numpy.py (small shapes), oracle/c_oracle.py (float64; inf in, inf out) and, for Bulyan at
n >= 2048, oracle/ref_torch.py on the GPU.  Index rules as elsewhere: an index must match when the float64 top-1/top-2
margin is > 1e-5 or an exact tie.  Vectors: rtol 1e-5 plus 1e-6 x the column's mean |finite value|; non-finite
entries must match exactly (position, sign of inf, NaN).  NaN inputs are not pinned, so no input here makes a
distance, a score or a median NaN in the reference.
"""
import numpy as np
import pytest

from oracle import c_oracle as co
from oracle import ref_numpy as orc

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

MARGIN = 1e-5
INF = np.float32(np.inf)


def hetero(rng, n, d):
    return (0.1 * rng.standard_normal(d) + np.exp(0.25 * rng.standard_normal((n, 1))) * rng.standard_normal((n, d))).astype(np.float32)


@pytest.fixture(scope="module")
def api():
    if not torch.cuda.is_available():
        pytest.skip("no GPU")
    from attacking_federate_learning_b200 import defences, _device, _native
    from attacking_federate_learning_b200.sharded import ShardedAggregator
    _native.lib()
    return defences, _device, _native, ShardedAggregator


def close_cols(got, ref, G):
    """rtol 1e-5 + 1e-6 x each column's mean |finite value|; non-finite entries must be the same."""
    got = np.asarray(got, np.float64); ref = np.asarray(ref, np.float64)
    assert np.array_equal(np.isnan(got), np.isnan(ref)), np.flatnonzero(np.isnan(got) != np.isnan(ref))[:10]
    assert np.array_equal(np.isposinf(got), np.isposinf(ref)), np.flatnonzero(np.isposinf(got) != np.isposinf(ref))[:10]
    assert np.array_equal(np.isneginf(got), np.isneginf(ref)), np.flatnonzero(np.isneginf(got) != np.isneginf(ref))[:10]
    fin = np.isfinite(ref)
    A = np.where(np.isfinite(G), np.abs(G.astype(np.float64)), 0.0)
    scale = A.sum(0) / np.maximum(np.isfinite(G).sum(0), 1) + 1e-30
    err = np.abs(got[fin] - ref[fin])
    bound = 1e-5 * np.abs(ref[fin]) + 1e-6 * scale[fin]
    assert (err <= bound).all(), (np.flatnonzero(fin)[err > bound][:10], (err / bound).max())


def sqdist_ref(G):
    """float64 sums of squared fl32(g_i - g_j), as co.pairwise_sqdist; past 1024 rows the same arithmetic runs on
    the GPU in torch (8 rows at a time), which keeps the n = 4096 tables to seconds."""
    if len(G) <= 1024:
        return co.pairwise_sqdist(G)
    X = torch.from_numpy(np.ascontiguousarray(G)).cuda()
    out = torch.empty((len(X), len(X)), dtype=torch.float64, device="cuda")
    for i0 in range(0, len(X), 8):
        diff = (X[i0:i0 + 8, None, :] - X[None, :, :]).double()
        out[i0:i0 + 8] = (diff * diff).sum(-1)
    return out.cpu().numpy()


def pinned(idx, want, margin):
    if margin > MARGIN or margin == 0.0:
        assert idx == want, (idx, want, margin)


def table_checks(d2, ref2, cap, spread_cap=3e-6, norms=None):
    """Bias and pair-to-pair spread of the relative error on the off-diagonal pairs, exact symmetry, zero diagonal.
    With `norms` (squared norms of the rows the kernel multiplied) the error is measured against ref2 + q_i + q_j:
    the Gram form's cancellation error scales with the norms, and at tiny D two rows can be much closer than that."""
    n = len(d2)
    assert np.array_equal(d2, d2.T) and not d2.diagonal().any()
    if n < 2:
        return
    den = ref2 if norms is None else ref2 + norms[:, None] + norms[None, :]
    off = ~np.eye(n, dtype=bool) & (den > 0)                          # duplicate rows: checked for exact zeros
    if not off.any():
        return
    rel = (d2[off] - ref2[off]) / den[off]
    assert np.abs(rel).max() < cap, np.abs(rel).max()
    if norms is None:
        assert rel.max() - rel.min() < spread_cap, (rel.min(), rel.max())


def ref_krum_index(scores):
    """defences.py:35-37: strict < from (1e20, -1) in the visit order [1, 0, 2, ...]."""
    best, best_u = 1e20, -1
    for u in orc.visit_order(len(scores)):
        if scores[u] < best:
            best, best_u = scores[u], u
    return best_u


def ref_krum_scores(table, take):
    """Sorted row (self excluded), sequential fp32 sum of the `take` smallest: np.cumsum runs in order."""
    t = table.astype(np.float32).copy()
    np.fill_diagonal(t, np.inf)
    srt = np.sort(t, axis=1)[:, :take]
    if take == 0:
        return np.zeros(len(t), np.float32)
    return np.cumsum(srt, axis=1, dtype=np.float32)[:, -1]


# ================================================================== A1: infinite client gradients, every route
def with_infinities(rng, n, d, f, variant):
    """Rows with +inf / -inf / both in a few columns.  Attackers never share a column, so no pair difference is
    inf - inf.  Rows a and a+1 are identical honest rows (their distance must stay exactly 0)."""
    G = hetero(rng, n, d)
    if variant == "centre":
        bad = [n - 3]                                            # one of the last 8 rows: the bf16x2 centre rows
    elif variant == "one":
        bad = [0]
    else:
        bad = list(range(max(f - 1, 1)))
    for k, u in enumerate(bad):
        cols = (3 * k + np.arange(3)) % d
        sign = [(1, 1, 1), (-1, -1, -1), (1, -1, 1)][k % 3]
        G[u, cols] = np.array(sign, np.float32) * INF
    a = len(bad) if variant != "centre" else 0
    G[a + 1] = G[a]
    return G, bad, (a, a + 1)


A1_SHAPES = [(12, 1000, 2), (100, 32768, 24), (300, 4096, 70), (1000, 2048, 240)]


@pytest.mark.parametrize("bf16", [False, True])
@pytest.mark.parametrize("variant", ["one", "many", "centre"])
@pytest.mark.parametrize("n,d,f", A1_SHAPES)
def test_krum_with_infinite_rows(api, n, d, f, variant, bf16):
    D, dev, nat, Sharded = api
    rng = np.random.default_rng(1000 + n + 7 * ["one", "many", "centre"].index(variant) + 100 * bf16)
    G, bad, dup = with_infinities(rng, n, d, f, variant)
    Gd = torch.from_numpy(G).cuda()
    if bf16:
        Gd = Gd.bfloat16(); G = Gd.float().cpu().numpy()
    ref2 = co.pairwise_sqdist(G)
    want, margin = co.krum_select(np.sqrt(ref2), n, f, with_margin=True)
    assert want not in bad
    if n <= 12:
        assert orc.krum(G, n, f, return_index=True) == want
    routes = {"device": D.krum(Gd, n, f, return_index=True),
              "sharded": Sharded().krum(Gd, n, f, return_index=True)}
    row = D.krum(G, n, f)                                                    # host-buffer C entry point
    assert np.shares_memory(row, G)
    routes["host"] = (row.ctypes.data - G.ctypes.data) // G.strides[0]
    formats = {"simt": nat.GRAM_FORCE_SIMT, "tensor": nat.GRAM_FORCE_TCGEN05}
    if not bf16:
        formats.update(tf32x2=nat.GRAM_FORCE_TCGEN05 | nat.GRAM_TF32X2,
                       no_center=nat.GRAM_FORCE_TCGEN05 | nat.GRAM_NO_CENTER)
    badmask = np.zeros(n, bool); badmask[bad] = True
    one_bad = badmask[:, None] ^ badmask[None, :]
    fin = ~(badmask[:, None] | badmask[None, :])
    np.fill_diagonal(fin, False)
    fin[dup] = fin[dup[::-1]] = False
    for name, flags in formats.items():
        d2t = dev.sqdist_partial(Gd, flags)
        d2 = d2t.cpu().numpy()
        assert np.array_equal(d2, d2.T) and not d2.diagonal().any(), name
        assert np.isposinf(d2[one_bad]).all(), (name, d2[one_bad][~np.isposinf(d2[one_bad])][:5])
        assert d2[dup] == 0.0, name
        rel = np.abs(d2[fin] - ref2[fin]) / ref2[fin]
        assert rel.max() < (1e-6 if name == "simt" else 1e-5), (name, rel.max())
        routes[name + "/from_sqdist"] = int(dev.krum_from_sqdist(d2t, n, f).item())
        routes[name + "/select"] = int(dev.krum_select(dev.sqdist_to_dist(d2t), n, f).item())
    for route, idx in routes.items():
        assert idx not in bad, route
        pinned(idx, want, margin)
    dist = D._krum_create_distances(Gd).dense.cpu().numpy()
    assert np.isposinf(dist[one_bad]).all() and not np.isnan(dist).any()
    assert dist[dup] == 0.0


@pytest.mark.parametrize("bf16", [False, True])
@pytest.mark.parametrize("variant", ["many", "centre"])
@pytest.mark.parametrize("n,d,f", [(12, 1000, 2), (100, 32768, 24), (300, 4096, 70), (1000, 2048, 240)])
def test_bulyan_with_infinite_rows(api, n, d, f, variant, bf16):
    D, dev, nat, _ = api
    rng = np.random.default_rng(2000 + n + 7 * (variant == "many") + 100 * bf16)
    G, bad, _ = with_infinities(rng, n, d, f, variant)
    Gd = torch.from_numpy(G).cuda()
    if bf16:
        Gd = Gd.bfloat16(); G = Gd.float().cpu().numpy()
    out, sel = D.bulyan(Gd, n, f, return_selection=True)
    sel = sel.cpu().tolist()
    gpu_table = D._krum_create_distances(Gd).dense.cpu().numpy().astype(np.float64)
    assert sel == co.bulyan_select(gpu_table, n, f)
    want, margins = co.bulyan_select(np.sqrt(co.pairwise_sqdist(G)), n, f, with_margins=True)
    first_close = next((i for i, m in enumerate(margins) if 0.0 < m <= MARGIN), len(margins))
    assert sel[:first_close] == want[:first_close]
    assert not set(sel) & set(bad)
    close_cols(out.cpu().numpy(), co.trimmed_mean(G, 2 * f, rows=sel), G)
    # Host-buffer route.  It does not return its selection, so it is pinned through its output: bit for bit the
    # slab-wise device route (one slab staged at the padded pitch: the same Gram, selection and second-stage calls),
    # whose selection is checked against the C oracle on its own table.
    ld = (d + 31) // 32 * 32
    Gp = torch.zeros((n, ld), device="cuda")[:, :d]; Gp.copy_(torch.from_numpy(G))
    dist_h = dev.sqdist_to_dist(dev.sqdist_partial(Gp))
    sel_h = dev.bulyan_select(dist_h, n, f)
    assert sel_h.cpu().tolist() == co.bulyan_select(dist_h.cpu().numpy().astype(np.float64), n, f)
    assert not set(sel_h.cpu().tolist()) & set(bad)
    route = dev.trimmed_mean(Gp, 2 * f, row_index=sel_h).cpu().numpy()
    host = D.bulyan(G, n, f)
    assert np.array_equal(host.view(np.uint32), route.view(np.uint32))
    close_cols(host, co.trimmed_mean(G, 2 * f, rows=sel_h.cpu().tolist()), G)


@pytest.mark.parametrize("n,d,f", [(12, 1000, 3), (100, 32768, 24), (300, 4096, 70)])
def test_krum_never_selects_huge_finite_row(api, n, d, f):
    """|x| ~ 1e20: the squares overflow fp32, the reference's fp32 dot gives inf; float64 gives a finite score far
    above 1e20.  Either way the row is never selected.  Index only."""
    D, dev, nat, Sharded = api
    rng = np.random.default_rng(3000 + n)
    G = hetero(rng, n, d)
    huge = (0, 1)                                                      # user 1 is the first one visited
    G[0] = 1e20 * np.sign(G[0]); G[1] = -1e20
    Gd = torch.from_numpy(G).cuda()
    want, margin = co.krum_select(np.sqrt(co.pairwise_sqdist(G)), n, f, with_margin=True)
    assert want not in huge
    got = {"device": D.krum(Gd, n, f, return_index=True), "sharded": Sharded().krum(Gd, n, f, return_index=True),
           "bf16": D.krum(Gd.bfloat16(), n, f, return_index=True)}
    row = D.krum(G, n, f)
    got["host"] = (row.ctypes.data - G.ctypes.data) // G.strides[0]
    for flags in (nat.GRAM_FORCE_SIMT, nat.GRAM_FORCE_TCGEN05 | nat.GRAM_TF32X2, nat.GRAM_FORCE_TCGEN05,
                  nat.GRAM_FORCE_TCGEN05 | nat.GRAM_NO_CENTER):
        got[flags] = int(dev.krum_from_sqdist(dev.sqdist_partial(Gd, flags), n, f).item())
    for route, idx in got.items():
        assert idx not in huge, route
        pinned(idx, want, margin)


# ================================================================== A2: trimmed mean with infinite deviations
def tm_matrix(rng, n, d, f, bf16):
    """Columns with k_c infinite entries (k_c cycling over 0 .. f + 4; all +inf, all -inf or mixed), then columns of
    finite values near -1e38 with k_c entries at +3e38, whose deviation from the median overflows to +inf.  The
    median stays finite: fewer than n/2 - 1 infinities, and the middle values are never infinite."""
    G = hetero(rng, n, d)
    half = d // 2
    for c in range(d):
        k = c % (f + 5)
        rows = rng.choice(n, size=k, replace=False)
        if c < half:
            kind = (c // (f + 5)) % 3
            signs = np.ones(k) if kind == 0 else -np.ones(k) if kind == 1 else np.where(np.arange(k) % 2, -1.0, 1.0)
            G[rows, c] = (signs * np.inf).astype(np.float32)
        else:
            G[:, c] = (-1e38 * (1.0 + 1e-4 * rng.standard_normal(n))).astype(np.float32)
            G[rows, c] = np.float32(3e38)
    Gd = torch.from_numpy(G).cuda()
    if bf16:
        Gd = Gd.bfloat16(); G = Gd.float().cpu().numpy()
    return G, Gd


@pytest.mark.parametrize("with_rows", [False, True])
@pytest.mark.parametrize("bf16", [False, True])
@pytest.mark.parametrize("n,f", [(100, 20), (1000, 240), (1024, 240), (1500, 300)])
def test_trimmed_mean_infinite_deviations(api, n, f, bf16, with_rows):
    D, dev, _, _ = api
    rng = np.random.default_rng(4000 + n + 10 * bf16 + 20 * with_rows)
    d = 2 * 3 * (f + 5) + 7                                              # every k_c and sign pattern, ragged last tile
    extra = 37 if with_rows else 0
    G, Gd = tm_matrix(rng, n + extra, d, f, bf16)
    if with_rows:
        rows = rng.permutation(n + extra)[:n].astype(np.int32)
        got = dev.trimmed_mean(Gd, f, row_index=torch.from_numpy(rows).cuda()).cpu().numpy()
        ref = co.trimmed_mean(G, f, rows=rows)
        Gr = G[rows]
    else:
        got = D.trimmed_mean(Gd, n, f).cpu().numpy()
        ref = co.trimmed_mean(G, f)
        Gr = G
    if not with_rows:
        assert np.isinf(ref).sum() > 0 and np.isnan(ref).sum() > 0      # the inputs reach the kept infinities
    close_cols(got, ref, Gr)
    if n <= 100:
        close_cols(got, orc.trimmed_mean(Gr, n, f), Gr)
    if not bf16 and not with_rows:
        close_cols(D.trimmed_mean(G, n, f), ref, G)                      # host-buffer route


@pytest.mark.parametrize("n", [100, 1500])
def test_trimmed_mean_keep_slice_semantics(api, n):
    """keep = n - f - 1 with Python slice semantics: f = n - 1 -> [] -> NaN; f = n -> all but the last; f = n + 3 ->
    all but the last four; f = 2n - 1 -> [] -> NaN.  Both kernels, finite and infinite columns."""
    D, *_ = api
    rng = np.random.default_rng(5000 + n)
    G, Gd = tm_matrix(rng, n, 64, 4, False)
    for f in (n - 1, n, n + 3, 2 * n - 1):
        ref = co.trimmed_mean(G, f)
        close_cols(D.trimmed_mean(Gd, n, f).cpu().numpy(), ref, G)
        if n <= 100:
            close_cols(D.trimmed_mean(Gd, n, f).cpu().numpy(), orc.trimmed_mean(G, n, f), G)
        assert np.isnan(ref).all() == (f in (n - 1, 2 * n - 1))


# ================================================================== A3: size limits
@pytest.mark.parametrize("d", [2048, 4100])
@pytest.mark.parametrize("n", [1025, 2048, 4096])
def test_gram_at_size_limits(api, n, d):
    _, dev, nat, _ = api
    rng = np.random.default_rng(6000 + n + d)
    G = hetero(rng, n, d)
    Gd = torch.from_numpy(G).cuda()
    ref2 = sqdist_ref(G)
    # Bias caps as at n <= 1000 (tests/test_gpu_scale_parity.py).  The centred bf16x2 error scales with
    # |g_i - c|^2 + |g_j - c|^2 relative to d2 (tests/test_gpu_parity.py), and with 4096 clients the
    # exp(0.25 z) norm scales reach further into their tail, so its spread cap is 5e-6 (measured on an H100: up to
    # 4.2e-6 at n = 4096, d = 2048).  That is 2.5e-6 in the distance, below the 1e-5 margin at which an index is
    # pinned, and a uniform bias cannot change a ranking.  Split TF32 and uncentred bf16x2 keep 3e-6 (measured up to
    # 1.2e-6 and 2.2e-6).
    for flags, spread in ((nat.GRAM_FORCE_TCGEN05, 5e-6), (nat.GRAM_FORCE_TCGEN05 | nat.GRAM_TF32X2, 3e-6),
                          (nat.GRAM_FORCE_TCGEN05 | nat.GRAM_NO_CENTER, 3e-6)):
        table_checks(dev.sqdist_partial(Gd, flags).cpu().numpy(), ref2, 1e-5, spread_cap=spread)
    table_checks(dev.sqdist_partial(Gd, nat.GRAM_FORCE_SIMT).cpu().numpy(), ref2, 1e-6, spread_cap=2e-6)
    d2 = dev.sqdist_partial(Gd, nat.GRAM_FORCE_TCGEN05)
    h = (d // 2) // 32 * 32
    halves = dev.sqdist_partial(Gd[:, :h].contiguous(), nat.GRAM_FORCE_TCGEN05) + \
        dev.sqdist_partial(Gd[:, h:].contiguous(), nat.GRAM_FORCE_TCGEN05)
    off = ~torch.eye(n, dtype=torch.bool, device="cuda")
    assert float(((halves - d2).abs()[off] / d2[off]).max()) < 2e-6
    del d2, halves
    Gb = torch.zeros((n, (d + 7) // 8 * 8), dtype=torch.bfloat16, device="cuda")[:, :d]   # 16-byte pitch
    Gb.copy_(Gd)
    table_checks(dev.sqdist_partial(Gb, nat.GRAM_FORCE_TCGEN05).cpu().numpy(),             # exact products: only
                 sqdist_ref(Gb.float().cpu().numpy()), 6e-6)                                # the fp32 sums round


@pytest.mark.parametrize("n", [1025, 2048, 4096])
def test_krum_scores_at_size_limits(api, n):
    """Both row sources of the Krum kernel (fp32 table with scores, float64 d2 table) against the sorted-row
    sequential fp32 sum, with an ALIE block of identical rows (exact score ties)."""
    _, dev, _, _ = api
    rng = np.random.default_rng(7000 + n)
    f = (n - 3) // 4
    G = hetero(rng, n, 256)
    G[:f] = G[:f].mean(0) - 1.5 * G[:f].std(0)
    Gd = torch.from_numpy(G).cuda()
    d2 = dev.sqdist_partial(Gd)
    dist = dev.sqdist_to_dist(d2)
    idx, scores = dev.krum_select(dist, n, f, want_scores=True)
    ref = ref_krum_scores(dist.cpu().numpy(), min(n - f, n - 1))
    assert np.array_equal(scores.cpu().numpy().view(np.uint32), ref.view(np.uint32))
    want = ref_krum_index(ref)
    assert int(idx.item()) == want
    assert int(dev.krum_from_sqdist(d2, n, f).item()) == want


def test_sharded_krum_past_4096(api):
    """afl_krum_sharded has no 4096 limit (a row of 4-byte keys fits shared memory up to 8192): n = 5000 runs the
    SIMT Gram and the Sqdist Krum kernel."""
    _, _, _, Sharded = api
    rng = np.random.default_rng(8000)
    n, d, f = 5000, 64, 1200
    G = hetero(rng, n, d)
    want, margin = co.krum_select(np.sqrt(co.pairwise_sqdist(G)), n, f, with_margin=True)
    pinned(Sharded().krum(torch.from_numpy(G).cuda(), n, f, return_index=True), want, margin)


@pytest.mark.parametrize("alie", [False, True])
@pytest.mark.parametrize("n", [1100, 2100, 3100, 4096])
def test_bulyan_selection_at_size_limits(api, n, alie):
    """Rows 1024 .. 4095 of the rounds kernel and the 2048- / 4096-key row sorts, against the float64 reference on
    the same fp32 table."""
    from oracle import ref_torch as rt
    _, dev, _, _ = api
    rng = np.random.default_rng(9000 + n + alie)
    f = (n - 3) // 4 - 1
    G = hetero(rng, n, 64)
    if alie:
        G[:f] = G[:f].mean(0) - 1.0 * G[:f].std(0)
    table = torch.from_numpy(np.sqrt(co.pairwise_sqdist(G)).astype(np.float32)).cuda()
    sel = dev.bulyan_select(table, n, f).cpu().tolist()
    want = rt.bulyan_select(table, n, f)
    assert len(want) == n - 2 * f
    assert sel == want, next(i for i, (a, b) in enumerate(zip(sel, want)) if a != b)


def test_bulyan_end_to_end_4096(api):
    """n = 4096, f = 1000: theta = 2096 selected rows, so the second stage runs the large trimmed-mean kernel with
    row_index.  Device and host-buffer routes."""
    from oracle import ref_torch as rt
    D, _, _, _ = api
    rng = np.random.default_rng(9500)
    n, d, f = 4096, 64, 1000
    G = hetero(rng, n, d)
    Gd = torch.from_numpy(G).cuda()
    out, sel = D.bulyan(Gd, n, f, return_selection=True)
    sel = sel.cpu().tolist()
    assert sel == rt.bulyan_select(D._krum_create_distances(Gd).dense, n, f)
    ref = co.trimmed_mean(G, 2 * f, rows=sel)
    close_cols(out.cpu().numpy(), ref, G)
    # pitch 64 = the host route's padded pitch, one slab: the host route makes the same calls on the same data, so its
    # output (the host call does not return its selection) is the device output bit for bit
    host = D.bulyan(G, n, f)
    assert np.array_equal(host.view(np.uint32), out.cpu().numpy().view(np.uint32))


@pytest.mark.parametrize("bf16", [False, True])
@pytest.mark.parametrize("n", [128, 256, 384, 512, 640, 768, 896, 1024, 1025, 4096, 12288])
def test_trimmed_mean_row_count_edges(api, n, bf16):
    """Register kernels at n = 32 S (no padded row), then the shared-memory kernel up to its 12,288-row limit."""
    D, dev, _, _ = api
    rng = np.random.default_rng(10000 + n + bf16)
    f = n // 4
    d = 300
    G = hetero(rng, n, d)
    G[:f // 2] = G[:f // 2].mean(0) - 1.5 * G[:f // 2].std(0)          # ties at the keep boundary
    Gd = torch.from_numpy(G).cuda()
    if bf16:
        Gd = Gd.bfloat16(); G = Gd.float().cpu().numpy()
    close_cols(D.trimmed_mean(Gd, n, f).cpu().numpy(), co.trimmed_mean(G, f), G)
    if n == 4096:
        rows = rng.permutation(n).astype(np.int32)
        got = dev.trimmed_mean(Gd, f, row_index=torch.from_numpy(rows).cuda()).cpu().numpy()
        close_cols(got, co.trimmed_mean(G, f, rows=rows), G[rows])


def test_rejections_past_the_limits(api):
    """Every limit is an argument check that fails before any launch."""
    D, dev, nat, _ = api
    n = 4097
    dist = torch.zeros((n, n), device="cuda")
    d2 = torch.zeros((n, n), dtype=torch.float64, device="cuda")
    with pytest.raises(NotImplementedError):
        dev.krum_select(dist, n, 10)
    with pytest.raises(NotImplementedError):
        dev.krum_from_sqdist(d2, n, 10)
    with pytest.raises(NotImplementedError):
        dev.bulyan_select(dist, n, 0)
    del dist, d2
    rng = np.random.default_rng(11000)
    G = hetero(rng, n, 64)
    with pytest.raises(NotImplementedError):
        D.krum(G, n, 10)
    with pytest.raises(NotImplementedError):
        D.bulyan(G, n, 0)
    Gd = torch.from_numpy(G).cuda()
    with pytest.raises(NotImplementedError):
        dev.sqdist_partial(Gd, nat.GRAM_FORCE_TCGEN05)
    table_checks(dev.sqdist_partial(Gd).cpu().numpy(), co.pairwise_sqdist(G), 1e-6, spread_cap=2e-6)   # SIMT
    with pytest.raises(NotImplementedError):
        dev.trimmed_mean(torch.zeros((12289, 8), device="cuda"), 0)


# ================================================================== A4: one-tile and tiny-D Gram shapes
def gram_formats(nat, bf16):
    if bf16:
        return {"bf16": nat.GRAM_FORCE_TCGEN05, "simt": nat.GRAM_FORCE_SIMT}
    return {"auto": nat.GRAM_FORCE_TCGEN05, "tf32x2": nat.GRAM_FORCE_TCGEN05 | nat.GRAM_TF32X2,
            "no_center": nat.GRAM_FORCE_TCGEN05 | nat.GRAM_NO_CENTER, "simt": nat.GRAM_FORCE_SIMT}


def gram_centre(G):
    """The centre of the centred bf16x2 format: fp32 mean of the last 8 rows (the last row repeated when n < 8),
    0 where it is not finite."""
    n = len(G)
    c = np.zeros(G.shape[1], np.float32)
    for r in range(8):
        c = c + G[min(max(n - 8, 0) + r, n - 1)]
    c = c * np.float32(0.125)
    return np.where(np.isfinite(c), c, np.float32(0))


def check_small_gram(dev, nat, G, Gd, bf16, sym=False):
    n, d = G.shape
    ref2 = co.pairwise_sqdist(G)
    centred = not bf16 and (n > 128 or (64 <= (n + 15) // 16 * 16 <= 112 and d >= 32768))   # "auto" is bf16x2 there
    for name, flags in gram_formats(nat, bf16).items():
        d2 = dev.sqdist_partial(Gd, flags).cpu().numpy()
        if name == "simt":
            table_checks(d2, ref2, 1e-6)
        else:
            # Tensor formats, error against ref2 + |x_i|^2 + |x_j|^2 with x the operand rows (g - c when centred).  At
            # tiny D two rows can be far closer than their norms, and the Gram form's error scales with the norms.
            # Split x = b1 + b2 + r, |b2| <= 2^-9 |x|, |r| <= 2^-17 |x|: the dropped terms are at most
            # (2^-18 + 2 * 2^-17) |x_i||x_j| per column, so the error of d2 = s_ii + s_jj - 2 s_ij is at most
            # 1.9e-5 (|x_i| + |x_j|)^2 <= 3.8e-5 (|x_i|^2 + |x_j|^2).  Split TF32 is far inside this.
            x = G - gram_centre(G) if (name == "auto" and centred) else G
            table_checks(d2, ref2, 4e-5, norms=(x.astype(np.float64) ** 2).sum(1))
        if n >= 3:
            assert d2[0, n // 2] == 0.0 and d2[n // 2, 0] == 0.0, name          # duplicate rows: exactly 0
        if sym and name == "auto":                                          # centred: error relative to the distance
            table_checks(d2, ref2, 1e-5, spread_cap=5e-6)


@pytest.mark.parametrize("bf16", [False, True])
@pytest.mark.parametrize("d", [4, 60, 64, 65, 4100])
@pytest.mark.parametrize("n", [1, 2, 7, 8, 9, 63, 64, 65, 112, 113, 127, 128, 129])
def test_gram_one_tile_and_tiny_d(api, n, d, bf16):
    _, dev, nat, _ = api
    rng = np.random.default_rng(12000 + 31 * n + d + bf16)
    ld = (d + 7) // 8 * 8                                                   # 16-byte pitch for fp32 and bf16
    buf = np.zeros((n, ld), np.float32)
    buf[:, :d] = hetero(rng, n, d)
    if n >= 3:
        buf[n // 2] = buf[0]
    Gd = torch.from_numpy(buf).cuda()
    if bf16:
        Gd = Gd.bfloat16()
    Gd = Gd[:, :d]
    check_small_gram(dev, nat, Gd.float().cpu().numpy(), Gd, bf16)


@pytest.mark.parametrize("d,n", [(1, 2), (1, 9), (1, 100), (1, 129), (1, 300), (3, 2), (3, 9), (3, 100), (3, 129)])
def test_gram_d_below_one_word(api, d, n):
    """d = 1 and d = 3 as views of a pitch-4 buffer: every k-block is mostly TMA zero fill."""
    _, dev, nat, _ = api
    rng = np.random.default_rng(13000 + d + n)
    buf = np.zeros((n, 4), np.float32)
    buf[:, :d] = hetero(rng, n, d)
    buf[n // 2] = buf[0]
    Gd = torch.from_numpy(buf).cuda()[:, :d]
    check_small_gram(dev, nat, Gd.cpu().numpy(), Gd, False)


@pytest.mark.parametrize("n", [49, 56, 57, 63, 64, 65, 105, 111, 112])
def test_gram_symmetric_form_row_rounding(api, n):
    """The one-tile symmetric bf16x2 form (64 <= N_pad <= 112, D >= 32768): boxes of N rounded up to 8 rows."""
    _, dev, nat, _ = api
    rng = np.random.default_rng(14000 + n)
    d = 32768 + 36
    buf = np.zeros((n, d + 4), np.float32)
    buf[:, :d] = hetero(rng, n, d)
    buf[n // 2] = buf[0]
    Gd = torch.from_numpy(buf).cuda()[:, :d]
    check_small_gram(dev, nat, Gd.cpu().numpy(), Gd, False, sym=True)
