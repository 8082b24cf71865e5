"""The trimmed mean (csrc/trimmed_mean.cu) against the reference's own fp32 arithmetic, bit for bit, at every kernel
instance, and on columns spread over many binades (-m gpu).

1. Exact oracle.  Columns of small integers with n * 2 max|x| < 2^23: the median is an integer or a half-integer, every
   deviation and every partial sum of kept deviations is exact in fp32, in any order.  So whatever the lane order and
   whichever selection path ran, the kernel must return the bits of `ref_numpy.trimmed_mean` (the reference's fp32
   NumPy arithmetic): one kept |dev| too many, or a tie group resolved out of row order, changes the result.
   Instances: trimmed_mean_kernel<S, DT, false> for S = 4 .. 32 (n at the first and last row count of each class) and
   fp32, bf16, fp16; <4, DT, true> through batched calls with one corrupted count per problem; the n > 1024 kernel.
   Column families, one per tile so that each meets every word-column and both halves of a 16-bit word: wide
   integers (fast path), a few distinct values (tie groups wider than a warp), two clusters with the median in the gap,
   constant columns, and +-T pairs cut by the keep boundary (only the row-order rule gets the sign of the sum right).
2. Wide spreads.  Attacker rows one per binade above (and below) honest rows, log-uniform columns over +-100 binades,
   signed zeros and subnormals around the median: the selection's bisection fallback must finish on every column.
   Against the C oracle with the parity tests' tolerance; every finite oracle entry must be finite.
"""
import warnings

import numpy as np
import pytest

from oracle import c_oracle as co
from oracle import ref_numpy as orc

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

DTYPES = {"f32": torch.float32, "bf16": torch.bfloat16, "f16": torch.float16}
# first and last row count of every kernel class: S = 4, 8, ..., 32 slots per lane, then the shared-memory kernel
ROW_COUNTS = [1, 2, 3, 33, 128, 129, 256, 257, 384, 385, 512, 513, 640, 641, 768, 769, 896, 897, 1024, 1025, 2048]
FAMILIES = ["wide", "few", "clusters", "const", "pm_t"]


@pytest.fixture(scope="module")
def api():
    if not torch.cuda.is_available():
        pytest.skip("no GPU")
    from attacking_federate_learning_b200 import batched, defences, _device, _native
    _native.lib()
    return batched, defences, _device


def ref_tm(G, f):
    """ref_numpy.trimmed_mean (fp32 NumPy, the reference's arithmetic); keep <= 0 gives NaN like np.mean([])."""
    with warnings.catch_warnings(), np.errstate(invalid="ignore", divide="ignore"):
        warnings.simplefilter("ignore", RuntimeWarning)
        return orc.trimmed_mean(G, len(G), f)


def assert_same_bits(got, want, what):
    """Bit for bit after -0 -> +0; NaN where the reference is NaN (its payload is the platform's)."""
    got = np.asarray(got, np.float32)
    want = np.asarray(want, np.float32)
    nan = np.isnan(want)
    assert np.array_equal(np.isnan(got), nan), (what, np.flatnonzero(np.isnan(got) != nan)[:10])
    g = np.where(got == 0, np.float32(0), got)[~nan].view(np.uint32)
    w = np.where(want == 0, np.float32(0), want)[~nan].view(np.uint32)
    bad = np.flatnonzero(g != w)
    assert bad.size == 0, (what, np.flatnonzero(~nan)[bad[:10]], g[bad[:10]].view(np.float32), w[bad[:10]].view(np.float32))


def value_cap(dtype, n):
    """max |x| such that the values are exact in the format and n * 2 max|x| < 2^23."""
    if dtype == "bf16":
        return 2 ** 7
    if dtype == "f16" or n > 1024:
        return 2 ** 10
    return 2 ** 11


def f_values(n):
    """corrupted counts giving keep = n - 1, about 3n/4 and 1, and f = n - 1 (keep 0: NaN)."""
    return sorted({f for f in (0, n - 1 - round(3 * n / 4), n - 2, n - 1) if 0 <= f <= n - 1})


def pm_t_column(rng, n, keep, M):
    """Median exactly 0 (>= 2 zero rows in the middle), L rows with |x| < T, g rows at +-T with random signs and
    rows, keep boundary inside the +-T group (L < keep < L + g), the rest with T < |x| <= M."""
    g = min(max(2, n // 8), 96)
    r_lo, r_hi = max(1, keep + g - n), min(g - 1, keep - 2)
    if n < 8 or r_lo > r_hi:
        return rng.integers(-M, M + 1, n)
    L = keep - int(rng.integers(r_lo, r_hi + 1))
    T = int(rng.integers(2, M // 2 + 1))
    z = max(2, L // 3)
    s = L - z
    b = n - L - g
    mag = np.concatenate([rng.integers(1, T, s), np.full(g, T), rng.integers(T + 1, M + 1, b)])
    m = len(mag)
    signs = np.ones(m, np.int64)
    signs[:m // 2] = -1                         # as many negative as positive rows: the zeros hold the middle
    rng.shuffle(signs)
    col = np.concatenate([np.zeros(z, np.int64), signs * mag])
    return col[rng.permutation(n)]


def family_column(rng, fam, n, M, keep):
    if fam == "wide":
        return rng.integers(-M, M + 1, n)
    if fam == "few":
        vals = rng.choice(np.arange(-M // 4, M // 4 + 1), size=3, replace=False)
        return vals[rng.choice(3, size=n, p=[0.25, 0.5, 0.25])]
    if fam == "clusters":
        lo_n = n // 2 + int(rng.integers(0, 2)) * (n % 2)
        lo = rng.integers(-M, -M // 2, lo_n)
        hi = rng.integers(M // 2 + 1, M + 1, n - lo_n)
        return np.concatenate([lo, hi])[rng.permutation(n)]
    if fam == "const":
        return np.full(n, rng.integers(-M, M + 1))
    return pm_t_column(rng, n, keep, M)


def exact_matrix(rng, n, dtype, cols_per_tile, keeps):
    """[n, d] fp32 integers: tile t holds family t % 5 in all its columns, then one more tile and a ragged tail of 7
    columns (families by column); +-T columns aim the keep boundary at keeps[column % len(keeps)]."""
    M = value_cap(dtype, n)
    d = (len(FAMILIES) + 1) * cols_per_tile + 7
    G = np.empty((n, d), np.float32)
    for c in range(d):
        t = c // cols_per_tile
        fam = FAMILIES[t % len(FAMILIES)] if t <= len(FAMILIES) else FAMILIES[c % len(FAMILIES)]
        G[:, c] = family_column(rng, fam, n, M, keeps[c % len(keeps)])
    assert np.abs(G).max() <= M
    return G


def on_device(G, dtype, pitch):
    """The matrix in `dtype` on the GPU, either at a 16-byte-aligned pitch (vector staging) or packed at the odd d
    (element-wise staging)."""
    n, d = G.shape
    ld = d if pitch == "packed" else d + (-d) % 16 + 16
    buf = torch.zeros((n, ld), dtype=DTYPES[dtype], device="cuda")
    buf[:, :d] = torch.from_numpy(G).cuda().to(DTYPES[dtype])
    out = buf[:, :d]
    assert np.array_equal(out.float().cpu().numpy(), G)          # every value exact in the format
    return out


# ================================================================== 1. exact oracle
@pytest.mark.parametrize("dtype", list(DTYPES))
@pytest.mark.parametrize("n", ROW_COUNTS)
def test_trimmed_mean_exact_every_instance(api, n, dtype):
    bt, D, dev = api
    rng = np.random.default_rng(31000 + 7 * n + list(DTYPES).index(dtype))
    fs = f_values(n)
    keeps = [max(n - f - 1, 0) for f in fs]
    cols = 16 if dtype == "f32" else 32
    G = exact_matrix(rng, n, dtype, cols, keeps)
    perm = rng.permutation(n).astype(np.int32)                  # Bulyan's stage 2: rows in selection order
    sub = perm[:max(n - n // 8, 1)]
    Gd = {p: on_device(G, dtype, p) for p in ("aligned", "packed")}
    for f in fs:
        want = ref_tm(G, f)
        got = {p: D.trimmed_mean(Gd[p], n, f).cpu().numpy() for p in Gd}
        assert_same_bits(got["aligned"], want, ("aligned", f))
        assert_same_bits(got["packed"], got["aligned"], ("packed", f))
        if dtype == "f32":                                        # the host-buffer route on the same NumPy matrix
            assert_same_bits(D.trimmed_mean(G, n, f), got["aligned"], ("host", f))
        for rows in (perm, sub):
            ff = min(f, len(rows) - 1)
            want_r = ref_tm(G[rows], ff)
            for p in Gd:
                ri = torch.from_numpy(rows).cuda()
                assert_same_bits(dev.trimmed_mean(Gd[p], ff, row_index=ri).cpu().numpy(), want_r, ("rows", p, len(rows), ff))


@pytest.mark.parametrize("dtype", list(DTYPES))
@pytest.mark.parametrize("n", [1, 2, 3, 33, 100, 128])
def test_trimmed_mean_exact_per_problem_counts(api, n, dtype):
    """trimmed_mean_kernel<4, DT, true>: every problem with its own corrupted count (and its own data)."""
    bt, D, dev = api
    rng = np.random.default_rng(32000 + 7 * n + list(DTYPES).index(dtype))
    fs = (f_values(n) * 2)[:max(len(f_values(n)), 3)]
    keeps = [max(n - f - 1, 0) for f in f_values(n)]
    cols = 16 if dtype == "f32" else 32
    mats = [exact_matrix(rng, n, dtype, cols, keeps) for _ in fs]
    d = mats[0].shape[1]
    for pitch, ld in (("aligned", d + (-d) % 16), ("packed", d)):   # packed: odd row and problem strides
        buf = torch.zeros((len(fs), n, ld), dtype=DTYPES[dtype], device="cuda")
        buf[:, :, :d] = torch.from_numpy(np.stack(mats)).cuda().to(DTYPES[dtype])
        Gb = buf[:, :, :d]
        out = bt.trimmed_mean(Gb, n, fs).cpu().numpy()
        for b, (G, f) in enumerate(zip(mats, fs)):
            assert_same_bits(out[b], ref_tm(G, f), (pitch, b, f))
        # the same batch with one count: the scalar instance
        out1 = bt.trimmed_mean(Gb, n, fs[0]).cpu().numpy()
        for b, G in enumerate(mats):
            assert_same_bits(out1[b], ref_tm(G, fs[0]), (pitch, b, fs[0]))


# ================================================================== 2. wide spreads
# one n per register class (S = 4, 8, ..., 32) and a corrupted count of at least 100 where n allows it
WIDE_SHAPES = [(100, 80), (200, 100), (300, 100), (500, 120), (600, 150), (700, 170), (800, 200), (1000, 240)]
WIDE_FAMILIES = ["attack_above", "attack_both", "log_uniform", "zeros_subnormals"]


def wide_matrix(rng, n, f, dtype, d=48):
    """Column c has family c % 4; rows 0..f-1 are the attackers of the attack families."""
    top = 15.9 if dtype == "f16" else 127.0                     # fp16 spans 40 binades, fp32 and bf16 254
    tiny = 2.0 ** (-24 if dtype == "f16" else -133 if dtype == "bf16" else -149)     # smallest subnormal
    G = np.empty((n, d), np.float32)
    for c in range(d):
        fam = WIDE_FAMILIES[c % len(WIDE_FAMILIES)]
        if fam.startswith("attack"):
            col = rng.standard_normal(n)
            col[:f] = 2.0 ** np.linspace(2.0, top, f)[rng.permutation(f)]
            if fam == "attack_both":
                col[:f] *= rng.choice([-1.0, 1.0], f)
        elif fam == "log_uniform":
            col = rng.choice([-1.0, 1.0], n) * 2.0 ** rng.uniform(-100, 100, n)
            if dtype == "f16":
                col = rng.choice([-1.0, 1.0], n) * 2.0 ** rng.uniform(-24, 15.9, n)
        else:
            kind = rng.choice(4, n, p=[0.2, 0.2, 0.4, 0.2])
            col = np.select([kind == 0, kind == 1, kind == 2],
                            [np.full(n, 0.0), np.full(n, -0.0), rng.integers(-50, 51, n) * tiny],
                            rng.choice([-1.0, 1.0], n) * 2.0 ** rng.uniform(-20, 0, n))
        G[:, c] = col
    Gd = torch.from_numpy(G).cuda().to(DTYPES[dtype])
    return Gd, Gd.float().cpu().numpy()


def close_cols(got, ref, G):
    """rtol 1e-5 + 1e-6 x each column's mean |finite value| (the tolerance of the parity tests); non-finite entries
    must be the same, so every finite oracle entry is finite."""
    got = np.asarray(got, np.float64); ref = np.asarray(ref, np.float64)
    assert np.isfinite(got[np.isfinite(ref)]).all(), np.flatnonzero(np.isfinite(ref) & ~np.isfinite(got))[:10]
    assert np.array_equal(np.isnan(got), np.isnan(ref)), np.flatnonzero(np.isnan(got) != np.isnan(ref))[:10]
    assert np.array_equal(np.isposinf(got), np.isposinf(ref))
    assert np.array_equal(np.isneginf(got), np.isneginf(ref))
    fin = np.isfinite(ref)
    A = np.where(np.isfinite(G), np.abs(G.astype(np.float64)), 0.0)
    scale = A.sum(0) / np.maximum(np.isfinite(G).sum(0), 1) + 1e-30
    err = np.abs(got[fin] - ref[fin])
    bound = 1e-5 * np.abs(ref[fin]) + 1e-6 * scale[fin]
    assert (err <= bound).all(), (np.flatnonzero(fin)[err > bound][:10], (err / bound).max())


@pytest.mark.parametrize("dtype", list(DTYPES))
@pytest.mark.parametrize("n,f", WIDE_SHAPES)
def test_trimmed_mean_wide_spread(api, n, f, dtype):
    bt, D, dev = api
    rng = np.random.default_rng(33000 + n + list(DTYPES).index(dtype))
    Gd, G = wide_matrix(rng, n, f, dtype)
    ref = co.trimmed_mean(G, f)
    close_cols(D.trimmed_mean(Gd, n, f).cpu().numpy(), ref, G)
    if dtype == "f32":
        close_cols(D.trimmed_mean(G, n, f), ref, G)               # host-buffer route
    # Bulyan's second stage: theta = n - 2 fb rows in selection order, 2 fb of them trimmed
    fb = (n - 3) // 4
    rows = rng.permutation(n)[:n - 2 * fb].astype(np.int32)
    got = dev.trimmed_mean(Gd, 2 * fb, row_index=torch.from_numpy(rows).cuda()).cpu().numpy()
    close_cols(got, co.trimmed_mean(G, 2 * fb, rows=rows), G[rows])


@pytest.mark.parametrize("dtype", list(DTYPES))
def test_trimmed_mean_wide_spread_batched(api, dtype):
    """n = 128 with up to 110 attackers per problem: the per-problem (EACH) and scalar S = 4 instances."""
    bt, D, dev = api
    rng = np.random.default_rng(34000 + list(DTYPES).index(dtype))
    n, fs = 128, [100, 90, 110, 64]
    mats = [wide_matrix(rng, n, f, dtype) for f in fs]
    Gb = torch.stack([m[0] for m in mats])
    out = bt.trimmed_mean(Gb, n, fs).cpu().numpy()
    out1 = bt.trimmed_mean(Gb, n, fs[0]).cpu().numpy()
    for b, ((_, G), f) in enumerate(zip(mats, fs)):
        close_cols(out[b], co.trimmed_mean(G, f), G)
        close_cols(out1[b], co.trimmed_mean(G, fs[0]), G)
