"""Batched aggregation against float64 and exact oracles, problem by problem, including the batched forms that no single
call runs (-m gpu).  The other batched tests pin each problem to the single device call; where a batch runs an operand
format or a kernel instance that a single call of the same problem would not, only an oracle can say it is right:

A. Per-problem distance tables, read out of the "batched" workspace (DESIGN 1b), against co.pairwise_sqdist (float64):
   exact symmetry, a zero diagonal, an exact zero and identical table rows for the copy of row 0 at rows_b // 2 (in the
   three-product forms, outside the columns between the two rows: DESIGN 2.1), and the operand-norm bound of
   test_gpu_edges.check_small_gram (error < 4e-5 (|x_i|^2 + |x_j|^2), x = g - the problem's own Gram centre in the
   centred bf16x2 forms, x = g elsewhere).  Centred forms with rows_b >= 9 also keep the distance-relative caps that
   the suite uses for the same form.  In the centred forms every problem carries a common component of its own,
   s_b mu_b with s_b = 0, 1, 8 or 30 times the noise: with its own centre the component cancels; centred on rows of
   another problem's count (padding, so no centre) a problem at s_b = 30 fails the norm bound tens of times over.
     1. fp32, N = 1000, rows_b = 1 ... 1000: the multi-tile bf16x2 form with one centre per problem, also for problems
        of at most 128 rows, whose single call would run split TF32.
     2. fp32, D >= 32768, N = 49 ... 112: the ragged one-tile symmetric bf16x2 form, one box height kSymN = 56 ... 112
        per case, every problem centred on its own last rows inside a box sized by N.
     3. The uncentred batched forms at the suite's usual data: split TF32, bf16 and fp16 operands, SIMT.
B. Selections on the device's own tables, exactly: Krum's index is the sorted-row fp32 score argmin over problem b's
   block (and the C oracle's wherever its float64 top-1 / top-2 margin exceeds 1e-5), Bulyan's selection is
   co.bulyan_select on the block of its fp32 distance table, then -2 up to theta_max.
C. The per-class trimmed-mean instances (trimmed_mean_kernel<S, DT, true, true>, S = 4 ... 32) on the exact-integer
   columns of test_gpu_trimmed_mean_exact, at every class boundary, in fp32, bf16 and fp16, at an aligned and a packed
   pitch: ref_numpy bit for bit, the mean too; and Bulyan's second stage (rows picked by the returned selection, row
   stride theta_max) with theta_b on every class boundary.
"""
import contextlib
import os

import numpy as np
import pytest

from oracle import c_oracle as co
from oracle import ref_numpy as orc
from test_gpu_edges import gram_centre, hetero, ref_krum_index, ref_krum_scores, table_checks
from test_gpu_trimmed_mean_exact import assert_same_bits, exact_matrix, f_values, ref_tm

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

MARGIN = 1e-5
NORM_BOUND = 4e-5        # test_gpu_edges.check_small_gram: proven for the split bf16x2 operands, looser for the others
SPLITS = "2"
DTYPES = {"f32": torch.float32, "bf16": torch.bfloat16, "f16": torch.float16}


@pytest.fixture(scope="module")
def api():
    if not torch.cuda.is_available():
        pytest.skip("no GPU")
    from attacking_federate_learning_b200 import batched, _device, _native
    _native.lib()
    return batched, _device


@pytest.fixture
def splits():
    saved = os.environ.get("AFL_GRAM_SPLITS")
    os.environ["AFL_GRAM_SPLITS"] = SPLITS
    yield
    if saved is None:
        os.environ.pop("AFL_GRAM_SPLITS", None)
    else:
        os.environ["AFL_GRAM_SPLITS"] = saved


@contextlib.contextmanager
def collect(failures, what):
    """Run one problem's checks and record a failure instead of stopping, so that a run reports every bad problem."""
    try:
        yield
    except AssertionError as e:
        failures.append(f"{what}: {e!r}"[:600])


def align_up(x, a):
    return (x + a - 1) // a * a


def fk(r):            # the sweep's malicious share
    return int(0.24 * r)


def fb(r):            # the largest f with r >= 4 f + 3
    return (r - 3) // 4


def slot_class(r):    # tmean::slot_class: the trimmed-mean instance S = 4 (class + 1)
    return 0 if r <= 128 else (r - 1) // 128


def workspace_tables(dev, G, rows, with_dist=False):
    """Problem b's leading rows_b x rows_b blocks of the last Krum or Bulyan call's tables, read out of the "batched"
    workspace (DESIGN 1b): the ProblemParams table (40 bytes per problem, and with more than 128 slot rows int perm[B]
    after it) padded to 256 bytes, then d2 [B][N][N] float64, then (Bulyan) dist [B][N][N] fp32."""
    B, N = G.shape[0], G.shape[1]
    t = align_up((40 if N <= 128 else 44) * B, 256)
    nn = B * N * N
    ws = dev.Workspace.get(G.device, "batched", 0)
    d2 = ws[t:t + 8 * nn].view(torch.float64).view(B, N, N).cpu().numpy()
    d2 = [d2[b, :r, :r] for b, r in enumerate(rows)]
    if not with_dist:
        return d2
    t2 = t + align_up(8 * nn, 256)
    dist = ws[t2:t2 + 4 * nn].view(torch.float32).view(B, N, N).cpu().numpy()
    return d2, [dist[b, :r, :r] for b, r in enumerate(rows)]


def dist32(d2):
    """The fp32 distances the selection kernels form from d2 (gram::sqdist_to_dist, select.cu krum_key)."""
    return np.sqrt(np.maximum(d2, 0.0)).astype(np.float32)


def problems(rng, rows, N, D, ld, offsets=None):
    """[B, N, ld] fp32 host buffer: problem b is hetero(rows_b, D) plus offsets[b] * mu_b (its own common component,
    in units of the noise), with row rows_b // 2 a copy of row 0; padding rows and columns are zero."""
    buf = np.zeros((len(rows), N, ld), np.float32)
    for b, r in enumerate(rows):
        X = hetero(rng, r, D)
        if offsets is not None and offsets[b]:
            X = X + np.float32(offsets[b]) * rng.standard_normal(D).astype(np.float32)
        X[r // 2] = X[0]
        buf[b, :r, :D] = X
    return buf


def check_table(d2, G, centred, caps=None, three_products=False):
    """A.: the device block d2 of problem G (fp32 rows as the kernel read them) against float64.
    three_products: a form that adds b1_I b2_J before b2_I b1_J, with I the pair's higher row (multi-tile bf16x2,
    split TF32; DESIGN 2.1).  The copy k = rows_b // 2 of row 0 then shares row 0's table entries wherever the pairs
    (0, j) and (k, j) have the same higher row, j > k; for 0 < j < k the two cross products are added in the other
    order, and an entry may differ in its last bits (the norm bound still holds for it)."""
    r = len(G)
    ref2 = co.pairwise_sqdist(G)
    x = G - gram_centre(G) if centred else G
    table_checks(d2, ref2, NORM_BOUND, norms=(x.astype(np.float64) ** 2).sum(1))
    k = r // 2
    assert d2[0, k] == 0.0 and d2[k, 0] == 0.0, ("duplicate rows", d2[0, k])
    diff = np.flatnonzero(d2[0] != d2[k])
    if three_products:
        diff = diff[(diff == 0) | (diff >= k)]
    assert diff.size == 0, ("duplicate rows, table rows differ at", diff[:10], d2[0, diff[:3]], d2[k, diff[:3]])
    if caps is not None and r >= 9:
        table_checks(d2, ref2, caps[0], spread_cap=caps[1])
    return ref2


def check_rules(bt, dev, G, Gh, rows, centred, caps=None, three_products=False, label=""):
    """A. and B. for one batch: Krum over every problem (its tables checked against float64, its index against the
    device table and the C oracle), then Bulyan over the problems with rows_b >= 3 (its selection against the device
    table).  G: the device batch; Gh: its rows as fp32 host arrays; caps(b): the distance-relative caps of problem b."""
    failures = []
    fs = [fk(r) for r in rows]
    idx = bt.krum(G, None, fs, return_index=True, rows=rows).cpu().tolist()
    d2s = workspace_tables(dev, G, rows)
    for b, r in enumerate(rows):
        with collect(failures, f"{label} problem {b} rows {r}"):
            ref2 = check_table(d2s[b], Gh[b], centred, None if caps is None else caps(b), three_products)
            take = min(r - fs[b], r - 1)
            want = ref_krum_index(ref_krum_scores(dist32(d2s[b]), take))
            assert idx[b] == want, ("krum on the device table", idx[b], want)
            if r >= 3:
                o, margin = co.krum_select(np.sqrt(ref2), r, fs[b], with_margin=True)
                assert margin <= MARGIN or idx[b] == o, ("krum vs the oracle", idx[b], o, margin)
    keep = [b for b, r in enumerate(rows) if r >= 3]
    brows = [rows[b] for b in keep]
    bfs = [fb(r) for r in brows]
    _, sel = bt.bulyan(G[keep], None, bfs, return_selection=True, rows=brows)
    sel = sel.cpu().numpy()
    d2s, dists = workspace_tables(dev, G[keep], brows, with_dist=True)
    assert sel.shape[1] == max(r - 2 * f for r, f in zip(brows, bfs))
    for j, b in enumerate(keep):
        r, f = brows[j], bfs[j]
        with collect(failures, f"{label} bulyan problem {b} rows {r}"):
            assert np.array_equal(dists[j], dist32(d2s[j]))
            theta = r - 2 * f
            want = co.bulyan_select(dists[j].astype(np.float64), r, f)
            assert sel[j, :theta].tolist() == want, ("bulyan on the device table", sel[j, :theta][:8], want[:8])
            assert (sel[j, theta:] == -2).all()
    assert not failures, "\n".join(failures)


# ================================================================== A.1 / B: multi-tile bf16x2 with per-problem centres
# rows_b <= 128 inside an N = 1000 batch run this form, not their single call's split TF32; the last k-block is ragged
A1_ROWS = [129, 7, 1000, 64, 2, 256, 9, 128, 1, 127, 8, 3]
A1_OFFSETS = [8, 30, 30, 30, 1, 0, 30, 8, 0, 30, 8, 1]
TILE_PAIR_CAPS = (1e-5, 3e-6)          # test_gpu_scale_parity / test_gpu_edges, multi-tile bf16x2
SYM_CAPS = (1e-5, 5e-6)                # test_gpu_edges.test_gram_symmetric_form_row_rounding
OFFSET_CAPS = (2e-5, 1.5e-5)           # test_gpu_scale_parity.test_gram_shared_mean_and_heterogeneous_norms


def test_large_ragged_fp32_centred_per_problem(api):
    bt, dev = api
    N, D = 1000, 2048 + 36
    rng = np.random.default_rng(41000)
    buf = problems(rng, A1_ROWS, N, D, D, A1_OFFSETS)
    G = torch.from_numpy(buf).cuda()
    Gh = [buf[b, :r] for b, r in enumerate(A1_ROWS)]
    check_rules(bt, dev, G, Gh, A1_ROWS, centred=True, three_products=True, label="fp32 N=1000",
                caps=lambda b: OFFSET_CAPS if A1_OFFSETS[b] else TILE_PAIR_CAPS)


# ================================================================== A.2 / B: ragged one-tile symmetric bf16x2
SYM_D = 32768 + 36
SYM_N = [49, 64, 65, 80, 88, 96, 100, 112]          # box heights kSymN = N rounded up to 8: 56, 64, ..., 112


def sym_rows(N):
    """rows_b from 1 to N in a mixed order, the full slot first."""
    return [N, 9, N - 1, 1, N // 2 + 1, 2, N - 8, 7]


@pytest.mark.parametrize("N", SYM_N, ids=[f"kSymN{(n + 7) // 8 * 8}-N{n}" for n in SYM_N])
def test_ragged_one_tile_symmetric_per_problem(api, N):
    bt, dev = api
    nb = (N + 15) // 16 * 16
    assert 64 <= nb <= 112 and SYM_D >= 32768           # gram.cu make_plan: the one-tile symmetric bf16x2 form
    rows = sym_rows(N)
    offsets = [(0, 30, 1, 8)[b % 4] for b in range(len(rows))]
    rng = np.random.default_rng(42000 + N)
    buf = problems(rng, rows, N, SYM_D, SYM_D + 4, offsets)
    G = torch.from_numpy(buf).cuda()[:, :, :SYM_D]
    Gh = [buf[b, :r, :SYM_D] for b, r in enumerate(rows)]
    check_rules(bt, dev, G, Gh, rows, centred=True, label=f"fp32 N={N}",
                caps=lambda b: OFFSET_CAPS if offsets[b] else SYM_CAPS)


# ================================================================== A.3 / B: uncentred batched forms
UNCENTRED = [("float32", "tf32x2", 100, 4096 + 36), ("bfloat16", "tensor", 100, 4096 + 40),
             ("bfloat16", "tensor", 300, 4096 + 40), ("float16", "tensor", 100, 4096 + 40),
             ("float16", "tensor", 300, 4096 + 40), ("float32", "simt", 100, 4099), ("float32", "simt", 300, 4099)]


@pytest.mark.parametrize("dtype,form,N,D", UNCENTRED, ids=[f"{d}-{f}-N{n}" for d, f, n, _ in UNCENTRED])
def test_uncentred_forms_per_problem(api, dtype, form, N, D):
    """No common offsets: these formats do not centre (DESIGN 2.1)."""
    bt, dev = api
    rows = [N, 8, N - 1, 1, N // 2 + 3, 2, 64, 9]
    rng = np.random.default_rng(43000 + N + D)
    buf = problems(rng, rows, N, D, D)
    G = torch.from_numpy(buf).cuda().to(getattr(torch, dtype))
    Gh = G.float().cpu().numpy()
    Gh = [np.ascontiguousarray(Gh[b, :r]) for b, r in enumerate(rows)]
    caps = (lambda b: (1e-6, 3e-6)) if form == "simt" else None          # check_small_gram's SIMT cap
    check_rules(bt, dev, G, Gh, rows, centred=False, caps=caps, three_products=form == "tf32x2",
                label=f"{dtype} {form} N={N}")


# ================================================================== B: one bf16 large ragged batch, anchored
def test_large_ragged_bf16_selections(api, splits):
    """The workspace reading is anchored here: with the split count pinned, a problem with rows_b = N is the single
    call's table bit for bit (bf16 operands: S_ij depends on rows i and j only)."""
    bt, dev = api
    N, D = 1000, 2048 + 40
    rng = np.random.default_rng(44000)
    buf = problems(rng, A1_ROWS, N, D, D)
    G = torch.from_numpy(buf).cuda().bfloat16()
    Gh = G.float().cpu().numpy()
    Gh = [np.ascontiguousarray(Gh[b, :r]) for b, r in enumerate(A1_ROWS)]
    full = A1_ROWS.index(N)
    bt.krum(G, None, [fk(r) for r in A1_ROWS], return_index=True, rows=A1_ROWS)
    got = workspace_tables(dev, G, A1_ROWS)[full]
    one = dev.sqdist_partial(G[full]).cpu().numpy()
    assert np.array_equal(got.view(np.uint64), one.view(np.uint64))
    check_rules(bt, dev, G, Gh, A1_ROWS, centred=False, label="bf16 N=1000")


# ================================================================== C: per-class trimmed mean, exact
# every class boundary; neighbours are never of one class, so the class permutation is not the identity
TM_ROWS = [1, 129, 257, 385, 513, 641, 769, 897, 2, 256, 384, 512, 640, 768, 896, 1024, 128]


def class_order_checks(rows):
    cls = [slot_class(r) for r in rows]
    assert sorted(set(cls)) == list(range(8))
    assert all(a != b for a, b in zip(cls, cls[1:]))


def batch_of(mats, N, dtype, pitch):
    """[B, N, d] device view of the exact matrices at an aligned (16-element) or packed (odd) pitch, padding NaN."""
    d = mats[0].shape[1]
    ld = d if pitch == "packed" else d + (-d) % 16
    buf = np.full((len(mats), N, ld), np.nan, np.float32)
    for b, M in enumerate(mats):
        buf[b, :len(M), :d] = M
    G = torch.from_numpy(buf).cuda().to(DTYPES[dtype])[:, :, :d]
    for b, M in enumerate(mats):
        assert np.array_equal(G[b, :len(M)].float().cpu().numpy(), M)          # every value exact in the format
    return G


@pytest.mark.parametrize("pitch", ["aligned", "packed"])
@pytest.mark.parametrize("dtype", list(DTYPES))
def test_trimmed_mean_every_class_exact(api, dtype, pitch):
    bt, _ = api
    rows = TM_ROWS
    class_order_checks(rows)
    rng = np.random.default_rng(45000 + 7 * list(DTYPES).index(dtype))
    cols = 16 if dtype == "f32" else 32
    mats = [exact_matrix(rng, r, dtype, cols, [max(r - f - 1, 0) for f in f_values(r)]) for r in rows]
    G = batch_of(mats, max(rows), dtype, pitch)
    failures = []
    for k in range(4):                         # keep = rows_b - 1, about 3/4, 1, 0 (NaN)
        fs = [f_values(r)[min(k, len(f_values(r)) - 1)] for r in rows]
        out = bt.trimmed_mean(G, None, fs, rows=rows).cpu().numpy()
        for b, (M, f) in enumerate(zip(mats, fs)):
            with collect(failures, f"trimmed mean problem {b} rows {rows[b]} f {f}"):
                assert_same_bits(out[b], ref_tm(M, f), (b, rows[b], f))
    mean = bt.no_defense(G, None, 0, rows=rows).cpu().numpy()
    for b, M in enumerate(mats):
        with collect(failures, f"mean problem {b} rows {rows[b]}"):
            assert_same_bits(mean[b], orc.no_defense(M), (b, rows[b]))
    assert not failures, "\n".join(failures)


# Bulyan's second stage: theta_b = rows_b - 2 f_b on every class boundary (theta >= 2 f + 3 >= 3), classes interleaved
BULYAN_THETAS = [3, 129, 257, 385, 513, 641, 769, 897, 128, 256, 384, 512, 640, 768, 896, 1024]


@pytest.mark.parametrize("pitch", ["aligned", "packed"])
@pytest.mark.parametrize("dtype", list(DTYPES))
def test_bulyan_second_stage_every_class_exact(api, dtype, pitch):
    """Whatever selection comes back, out[b] is the trimmed mean of the selected rows with 2 f_b, bit for bit."""
    bt, _ = api
    class_order_checks(BULYAN_THETAS)
    fs = [min((t - 3) // 2, (1024 - t) // 2, (0, 17, 40, 63)[i % 4]) for i, t in enumerate(BULYAN_THETAS)]
    rows = [t + 2 * f for t, f in zip(BULYAN_THETAS, fs)]
    assert all(r >= 4 * f + 3 for r, f in zip(rows, fs)) and max(rows) == 1024
    rng = np.random.default_rng(46000 + 7 * list(DTYPES).index(dtype))
    cols = 16 if dtype == "f32" else 32
    mats = [exact_matrix(rng, r, dtype, cols, [max(t - 2 * f - 1, 0)]) for r, t, f in zip(rows, BULYAN_THETAS, fs)]
    G = batch_of(mats, max(rows), dtype, pitch)
    out, sel = bt.bulyan(G, None, fs, return_selection=True, rows=rows)
    out, sel = out.cpu().numpy(), sel.cpu().numpy()
    assert sel.shape[1] == max(BULYAN_THETAS)
    failures = []
    for b, (M, t, f) in enumerate(zip(mats, BULYAN_THETAS, fs)):
        with collect(failures, f"bulyan problem {b} rows {rows[b]} theta {t} f {f}"):
            s = sel[b, :t]
            assert (sel[b, t:] == -2).all() and len(set(s.tolist())) == t and s.min() >= 0 and s.max() < rows[b]
            assert_same_bits(out[b], ref_tm(M[s], 2 * f), (b, t, f))
    assert not failures, "\n".join(failures)
