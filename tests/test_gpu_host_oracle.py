"""The host-buffer engine (csrc/capi.cu, DESIGN 1c) against float64 and exact oracles over several slabs (-m gpu).
test_gpu_host_surface and test_gpu_host_streaming pin each host entry point to a slab-wise route built from the
device entry points; a mistake both routes share passes there.  Here every result is held to an oracle instead, at
client counts up to 12288, with narrow slabs (4 to 12 of them, the last one ragged) and a host pitch ld > d:

A. afl_sqdist_host at N = 129 ... 4096 (centred bf16x2 slabs) against float64 sums: exact symmetry, a zero diagonal,
   exact zeros between the ALIE-crafted rows 0 ... f-1, and the operand-norm bound of test_gpu_edges.check_small_gram
   (x = G - gram_centre(G): the centre is per column, so every slab's table keeps the bound for its own columns and
   the slab sum keeps the whole-matrix bound).  The Krum index of afl_defend_host is the sorted-row fp32 argmin over
   that table, the C oracle's index wherever its float64 margin exceeds 1e-5, and 1 (the reference's tie-break)
   whenever a crafted row wins.  N = 4500 and 6000 run the SIMT Gram kernel on every slab (its caps 1e-6 / 2e-6).
   The table must also be the per-slab device tables added in slab order, bit for bit.  Every slab's entries are
   float64 sums of a few fp32 partial sums (MMA accumulators, or the SIMT kernel's 32-column chunks), so at these
   shapes the float64 sum over the slabs is exact and gives the same bits in any slab order.
B. afl_bulyan_host with theta = N - 2f on every trimmed-mean class boundary from 128 to 2096 (the large kernel past
   1024).  2f far outlier rows at random positions keep the selected set known, so the exact-integer columns of
   test_gpu_trimmed_mean_exact (the +-T family aimed at the keep boundary of the theta selected rows) are built on
   exactly those rows.  The selection is the float64 reference on the device's own fp32 table; the output is ref_numpy
   bit for bit on the integer columns and co.trimmed_mean within close_cols on the hetero columns.  The partial
   budget ends the resident prefix between the two integer blocks, so the resident pass (row_index = sel) and the
   packed re-streamed pass (theta rows in selection order at pitch w2 > slab_cols) each cover a block of every family.
C. afl_defend_host("TrimmedMean" / "NoDefense") at N = 129 ... 12288 on exact-integer columns: ref_numpy bit for bit
   for every corrupted count of f_values(N), the mean too.
D. afl_alie_host at f = 1025 and 4096 separate user arrays, with an inf and an inf - inf column: the C oracle within
   test_gpu_parity's RTOL with NaN exactly where it has NaN, and one whole-matrix afl_alie bit for bit, aliased or not.
E. krum(..., distances=..., return_index=True) on a table the caller pops users from, as the reference's Bulyan loop
   does (defences.py:57-68): a reference-style dict-of-dicts and a DistanceTable, every round against
   ref_numpy.krum_select on the same alive users.

Each case runs under three budgets (AFL_HOST_DEVICE_BYTES): ring only, then a partial resident prefix (Bulyan) or a
third ring slot (the others), then unlimited, each after a call on other data of the same shape.  The engine keeps its
device output vector between calls, so a column that a call fails to write shows the other call's value instead of
the previous budget's correct one.  Failures are collected per case and budget and reported together.
"""
import ctypes as C
import os
from collections import defaultdict

import numpy as np
import pytest

from oracle import c_oracle as co
from oracle import ref_numpy as orc
from test_gpu_batched_oracle import collect, dist32
from test_gpu_edges import (close_cols, gram_centre, hetero, pinned, ref_krum_index, ref_krum_scores, sqdist_ref,
                            table_checks)
from test_gpu_host_surface import (budgets, call_alie, call_bulyan, call_sqdist, host_matrix, slab_width,
                                   slabwise_sqdist, user_arrays)
from test_gpu_trimmed_mean_exact import assert_same_bits, exact_matrix, f_values, ref_tm

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

ENV = "AFL_HOST_DEVICE_BYTES"
NORM_BOUND = 4e-5        # test_gpu_edges.check_small_gram: the centred bf16x2 operand-norm bound
SIMT_CAPS = (1e-6, 2e-6)  # test_gpu_edges: the SIMT Gram kernel's bias and spread caps
RTOL = 1e-5              # test_gpu_parity.test_golden_alie
EXTRA = 5                # host pitch ld = d + EXTRA
POISON = np.float32(12345.0)
ORDER = ("ring", "partial", "unlimited")


@pytest.fixture(scope="module")
def api():
    if not torch.cuda.is_available():
        pytest.skip("no GPU")
    from attacking_federate_learning_b200 import defences, _device, _native
    _native.lib()
    return defences, _device, _native


@pytest.fixture
def budget():
    """Setter for AFL_HOST_DEVICE_BYTES (None = unset); the variable is restored when the test ends."""
    saved = os.environ.get(ENV)

    def set_budget(nbytes):
        if nbytes is None:
            os.environ.pop(ENV, None)
        else:
            os.environ[ENV] = str(int(nbytes))
    yield set_budget
    if saved is None:
        os.environ.pop(ENV, None)
    else:
        os.environ[ENV] = saved


def run_budgets(call, set_budget, who, slab_bytes, nslab, poison=None):
    """call() -> (rc, result, message) under ring only, partial, unlimited (in that order), each after poison() (the
    same entry point on other data of the same shape, unlimited budget)."""
    assert nslab >= 3
    sizes = budgets(call, set_budget, who, slab_bytes, nslab)
    got = {}
    for name in ORDER:
        set_budget(None)
        if poison is not None:
            assert poison()[0] == 0
        set_budget(sizes[name])
        rc, res, msg = call()
        assert rc == 0, (name, msg)
        got[name] = res
    set_budget(None)
    return got


def same_bits(a, b):
    a, b = np.asarray(a), np.asarray(b)
    return a.shape == b.shape and np.array_equal(a.view(np.uint32), b.view(np.uint32))


def nslabs(rows, d, slab_cols):
    w = slab_width(rows, d, slab_cols)
    return w, -(-d // w)


def defend_call(nat, rule, Gh, ld, f, slab_cols):
    n, d = Gh.shape
    out = np.full(d, np.nan, np.float32)
    idx = C.c_int(-7)
    rc = nat.lib().afl_defend_host(rule, Gh.ctypes.data, n, d, ld, n, f, out.ctypes.data, C.byref(idx), slab_cols)
    return rc, out, nat.lib().afl_last_error().decode() if rc else ""


def krum_call(nat, Gh, ld, f, slab_cols):
    n, d = Gh.shape
    idx = C.c_int(-7)
    rc = nat.lib().afl_defend_host(b"Krum", Gh.ctypes.data, n, d, ld, n, f, None, C.byref(idx), slab_cols)
    return rc, idx.value, nat.lib().afl_last_error().decode() if rc else ""


def crafted_rows(G, f, z=0.5):
    """Rows 0 .. f-1 set to one ALIE vector from the honest rows' statistics, close enough to their mean to win Krum."""
    if f:
        H = G[f:]
        G[:f] = H.mean(0) - np.float32(z) * H.std(0)
    return G


# ================================================================== A. distance tables and Krum
# (n, d, slab_cols): 11, 9, 5, 8 and 5 slabs, every last slab ragged
A_SHAPES = [(129, 1000, 96), (500, 805, 96), (1000, 611, 128), (2100, 700, 96), (4096, 517, 128)]


@pytest.mark.parametrize("n,d,slab_cols", A_SHAPES, ids=[f"N{s[0]}" for s in A_SHAPES])
def test_sqdist_and_krum_several_slabs(api, budget, n, d, slab_cols):
    D, dev, nat = api
    rng = np.random.default_rng(51000 + n)
    f = int(0.24 * n)
    G = crafted_rows(hetero(rng, n, d), f)
    Gh, ld = host_matrix(G, EXTRA)
    w, ns = nslabs(n, d, slab_cols)
    assert 4 <= ns <= 12 and d % w
    failures = []
    tables = run_budgets(lambda: call_sqdist(nat, Gh, ld, slab_cols), budget, "afl_sqdist_host", n * w * 4, ns)
    for name in ORDER[1:]:
        with collect(failures, f"N={n} table {name}"):
            assert torch.equal(tables[name], tables["ring"]), "the table depends on the budget"
    with collect(failures, f"N={n} slab order"):
        assert torch.equal(tables["ring"], slabwise_sqdist(dev, G, slab_cols)), "not the slab tables summed in order"
    d2 = tables["ring"].cpu().numpy()
    del tables
    ref2 = sqdist_ref(G)
    with collect(failures, f"N={n} table vs float64"):
        x = (G - gram_centre(G)).astype(np.float64)
        table_checks(d2, ref2, NORM_BOUND, norms=(x ** 2).sum(1))
    with collect(failures, f"N={n} crafted rows"):
        assert not d2[:f, :f].any(), np.argwhere(d2[:f, :f])[:5]

    take = min(n - f, n - 1)
    want = ref_krum_index(ref_krum_scores(dist32(d2), take))
    o, margin = co.krum_select(np.sqrt(ref2), n, f, with_margin=True)
    idx = run_budgets(lambda: krum_call(nat, Gh, ld, f, slab_cols), budget, "afl_defend_host", n * w * 4, ns)
    for name, i in idx.items():
        with collect(failures, f"N={n} krum {name}"):
            assert i == want, ("krum on the device table", i, want)
            pinned(i, o, margin)
            assert want >= f or i == 1, ("a crafted row wins: the reference visits row 1 first", i)
    assert not failures, "\n".join(failures)


@pytest.mark.parametrize("n", [4500, 6000])
def test_sqdist_simt_several_slabs(api, budget, n):
    """Past 4096 clients every slab runs the SIMT Gram kernel: direct float64 sums of squared fp32 differences."""
    D, dev, nat = api
    rng = np.random.default_rng(52000 + n)
    d, slab_cols, f = 200, 64, int(0.24 * n)
    G = crafted_rows(hetero(rng, n, d), f)
    Gh, ld = host_matrix(G, EXTRA)
    w, ns = nslabs(n, d, slab_cols)
    assert ns == 4 and d % w
    failures = []
    tables = run_budgets(lambda: call_sqdist(nat, Gh, ld, slab_cols), budget, "afl_sqdist_host", n * w * 4, ns)
    for name in ORDER[1:]:
        with collect(failures, f"N={n} table {name}"):
            assert torch.equal(tables[name], tables["ring"]), "the table depends on the budget"
    with collect(failures, f"N={n} slab order"):
        assert torch.equal(tables["ring"], slabwise_sqdist(dev, G, slab_cols)), "not the slab tables summed in order"
    d2 = tables["ring"].cpu().numpy()
    del tables
    with collect(failures, f"N={n} table vs float64"):
        table_checks(d2, sqdist_ref(G), SIMT_CAPS[0], spread_cap=SIMT_CAPS[1])
    with collect(failures, f"N={n} crafted rows"):
        assert not d2[:f, :f].any()
    assert not failures, "\n".join(failures)


# ================================================================== B. Bulyan, theta on every class boundary
B_THETAS = [128, 129, 256, 257, 512, 513, 1024, 1025, 2096]
B_SLAB = 128
B_NSLAB = 6
B_D = B_NSLAB * B_SLAB - 19                # ragged last slab
B_RES = B_NSLAB // 2 * B_SLAB              # the partial budget's resident columns (R = nslab // 2 slabs)
INT_COLS = 16                              # columns per family tile: exact_matrix blocks of 6 * 16 + 7 columns
HETERO_SCALE = np.float32(2.0 ** 12)       # the hetero columns dominate the honest rows' distances
OUTLIER_SCALE = np.float32(2.0 ** 16)      # outliers: about ten times further from every row than honest rows are


def bulyan_matrix(rng, theta, f):
    """[n, B_D] matrix with n = theta + 2f: integer block E1 at columns [0, 103), E2 at [B_RES, B_RES + 103), hetero
    columns elsewhere.  The 2f outlier rows (zero integer columns, huge independent hetero columns) are never selected,
    so the integer blocks are exact_matrix blocks of the theta honest rows with the +-T boundary at theta - 2f - 1."""
    n = theta + 2 * f
    out_rows = rng.choice(n, 2 * f, replace=False)
    honest = np.setdiff1d(np.arange(n), out_rows)
    G = np.zeros((n, B_D), np.float32)
    ints = np.zeros(B_D, bool)
    for c0 in (0, B_RES):
        E = exact_matrix(rng, theta, "f32", INT_COLS, [theta - 2 * f - 1])
        G[honest, c0:c0 + E.shape[1]] = E
        ints[c0:c0 + E.shape[1]] = True
    het = ~ints
    G[np.ix_(honest, het)] = hetero(rng, theta, het.sum()) * HETERO_SCALE
    G[np.ix_(out_rows, het)] = rng.standard_normal((2 * f, het.sum())).astype(np.float32) * OUTLIER_SCALE
    return G, honest, ints


def ref_selection(dist, n, f):
    """The float64 selection on the device's fp32 table: the C oracle where it takes seconds, else ref_torch."""
    if n <= 800:
        return co.bulyan_select(dist.cpu().numpy().astype(np.float64), n, f)
    from oracle import ref_torch as rt
    return rt.bulyan_select(dist, n, f)


@pytest.mark.parametrize("theta", B_THETAS)
def test_bulyan_every_class_several_slabs(api, budget, theta):
    D, dev, nat = api
    rng = np.random.default_rng(53000 + theta)
    f = theta // 4                         # n / theta = 1.5: the re-streamed slabs (w2) are wider than slab_cols
    n = theta + 2 * f
    assert n >= 4 * f + 3 and n <= 4096
    G, honest, ints = bulyan_matrix(rng, theta, f)
    Gh, ld = host_matrix(G, EXTRA)
    Gp, _ = host_matrix(np.full_like(G, POISON), EXTRA)
    w, ns = nslabs(n, B_D, B_SLAB)
    assert w == B_SLAB and ns == B_NSLAB
    assert ints[:B_RES].any() and ints[B_RES:].any()
    rc, d2, msg = call_sqdist(nat, Gh, ld, B_SLAB)
    assert rc == 0, msg
    want = ref_selection(dev.sqdist_to_dist(d2), n, f)
    assert sorted(want) == honest.tolist(), "an outlier was selected: the integer blocks are not on the selected rows"
    S = G[want]
    want_int = ref_tm(S, 2 * f)
    want_het = co.trimmed_mean(G, 2 * f, rows=want)
    # the +-T columns tell selection order from ascending row order in both blocks
    order_cols = np.flatnonzero(ints & (ref_tm(G[np.sort(want)], 2 * f) != want_int))
    assert (order_cols < B_RES).any() and (order_cols >= B_RES).any(), order_cols

    got = run_budgets(lambda: call_bulyan(nat, Gh, ld, f, B_SLAB), budget, "afl_bulyan_host", n * w * 4, ns,
                      poison=lambda: call_bulyan(nat, Gp, ld, f, B_SLAB))
    failures = []
    for name, (out, sel) in got.items():
        with collect(failures, f"theta={theta} {name} selection"):
            assert sel.tolist() == want, ("first difference at", next(i for i, (a, b) in enumerate(zip(sel, want))
                                                                   if a != b))
        with collect(failures, f"theta={theta} {name} integer columns"):
            assert_same_bits(out[ints], want_int[ints], name)
        with collect(failures, f"theta={theta} {name} hetero columns"):
            close_cols(out[~ints], want_het[~ints], S[:, ~ints])
        with collect(failures, f"theta={theta} {name} against ring only"):
            assert same_bits(out, got["ring"][0])
    assert not failures, "\n".join(failures)


# ================================================================== C. TrimmedMean and NoDefense
C_ROWS = [129, 1024, 1025, 4096, 12288]
C_SLAB = 32                                # 103 columns: slabs of 32, 32, 32 and 7 at pitch 32


def cap_format(n):
    """exact_matrix's value cap by format name: 2^11 ("f32") or 2^10 ("f16", n > 1024) up to 2048 rows, 2^7 ("bf16")
    beyond, so that n * 2 max|x| < 2^23 and every partial sum is exact."""
    return "f32" if n <= 2048 else "bf16"


@pytest.mark.parametrize("n", C_ROWS)
def test_trimmed_mean_and_mean_several_slabs(api, budget, n):
    D, dev, nat = api
    rng = np.random.default_rng(54000 + n)
    fs = f_values(n)
    M = exact_matrix(rng, n, cap_format(n), INT_COLS, [max(n - f - 1, 0) for f in fs])
    d = M.shape[1]
    Gh, ld = host_matrix(M, EXTRA)
    Gp, _ = host_matrix(np.full_like(M, POISON), EXTRA)
    w, ns = nslabs(n, d, C_SLAB)
    assert ns >= 3 and d % w
    failures = []
    for f in fs:
        got = run_budgets(lambda: defend_call(nat, b"TrimmedMean", Gh, ld, f, C_SLAB), budget, "afl_defend_host",
                          n * w * 4, ns, poison=lambda: defend_call(nat, b"TrimmedMean", Gp, ld, f, C_SLAB))
        want = ref_tm(M, f)
        for name, out in got.items():
            with collect(failures, f"N={n} trimmed mean f={f} {name}"):
                assert_same_bits(out, want, (name, f))
    got = run_budgets(lambda: defend_call(nat, b"NoDefense", Gh, ld, 0, C_SLAB), budget, "afl_defend_host",
                      n * w * 4, ns, poison=lambda: defend_call(nat, b"NoDefense", Gp, ld, 0, C_SLAB))
    want = orc.no_defense(M)
    for name, out in got.items():
        with collect(failures, f"N={n} mean {name}"):
            assert same_bits(out, want)
    assert not failures, "\n".join(failures)


# ================================================================== D. ALIE past 240 attackers
@pytest.mark.parametrize("f", [1025, 4096])
def test_alie_host_many_attackers(api, budget, f):
    D, dev, nat = api
    rng = np.random.default_rng(55000 + f)
    d, slab_cols, z = 1000, 256, 1.5
    rows = user_arrays(rng, f, d, "contiguous")
    rows[1][5] = np.inf                                   # sigma NaN (inf - inf in the variance), crafted NaN
    rows[0][7] = -np.inf
    rows[1][7] = np.inf                                   # mu NaN too
    poison = [np.full(d, POISON) for _ in range(f)]
    w, ns = nslabs(f, d, slab_cols)
    assert ns >= 3 and d % w
    stack = np.stack(rows)
    cr, mu64, sd64 = co.alie(stack, z)
    with np.errstate(invalid="ignore"):
        mu32, sd32 = orc.alie_stats(stack)
    failures = []
    got = {}
    for alias in (True, False):
        res = run_budgets(lambda: call_alie(nat, rows, z, slab_cols, alias=alias), budget, "afl_alie_host",
                          f * w * 4, ns, poison=lambda: call_alie(nat, poison, z, slab_cols, alias=alias))
        got[alias] = res["ring"]
        whole = dict(zip(("crafted", "mu", "sigma"), (t.cpu().numpy() for t in dev.alie(
            torch.from_numpy(stack).cuda(), z, None, alias_mean=alias))))
        for name, (mu, sigma, crafted) in res.items():
            what = f"f={f} alias={alias} {name}"
            with collect(failures, what + " whole-matrix afl_alie"):
                assert same_bits(sigma, whole["sigma"]) and same_bits(crafted, whole["crafted"])
                assert same_bits(mu, whole["mu"])
            with collect(failures, what + " oracle"):
                for got_v, ref64, ref32, atol in ((sigma, sd64, sd32, 1e-7), (crafted, cr, None, 1e-6),
                                                  (mu, cr if alias else mu64, None if alias else mu32, 1e-6)):
                    nan = np.isnan(ref64)
                    assert np.array_equal(np.isnan(got_v), nan), np.flatnonzero(np.isnan(got_v) != nan)
                    np.testing.assert_allclose(got_v, ref64, rtol=RTOL, atol=atol)
                    if ref32 is not None:
                        np.testing.assert_allclose(got_v, ref32, rtol=RTOL, atol=atol)
    with collect(failures, f"f={f} aliased against not aliased"):
        (mu_a, s_a, c_a), (mu_n, s_n, c_n) = got[True], got[False]
        assert same_bits(s_a, s_n) and same_bits(c_a, c_n) and same_bits(mu_a, c_n)
    with collect(failures, f"f={f} the inf columns"):
        sigma = got[False][1]
        assert np.isnan(sigma[5]) and np.isnan(sigma[7]) and np.isnan(got[False][0][7]) and got[False][0][5] == np.inf
    assert not failures, "\n".join(failures)


# ================================================================== E. the reference's popped-table Krum
def reference_distances(G):
    """defences.py:16-21: a defaultdict of dicts of fp32 norms, keys in the order the reference creates them."""
    distances = defaultdict(dict)
    for i in range(len(G)):
        for j in range(i):
            distances[i][j] = distances[j][i] = np.linalg.norm(G[i] - G[j])
    return distances


def dense_of(distances, n):
    t = np.zeros((n, n), np.float32)
    for u in distances.keys():
        for v, x in distances[u].items():
            t[u, v] = x
    return t


@pytest.mark.parametrize("where", ["cuda", "numpy"])
@pytest.mark.parametrize("n", [11, 100, 129])
def test_popped_table_krum(api, n, where):
    """Bulyan's selection loop of the reference (defences.py:57-68) with krum(..., distances) on the GPU.  The crafted
    rows 0 .. f-1 tie exactly, so the first two rounds (keys [1, 0, 2, ...], then [0, 2, ...]) also pin the order in
    which the compacted table is visited."""
    D, dev, nat = api
    rng = np.random.default_rng(56000 + n)
    f = (n - 3) // 4
    G = crafted_rows(hetero(rng, n, 64), f)
    Gx = torch.from_numpy(G).cuda() if where == "cuda" else G
    failures = []
    for kind in ("dict", "DistanceTable"):
        if kind == "dict":
            distances = reference_distances(G)
            dense = dense_of(distances, n)
        else:
            distances = D._krum_create_distances(Gx)
            dense = distances.dense.cpu().numpy()
        chosen = []
        while len(chosen) < n - 2 * f:
            users_count = n - len(chosen)
            alive = list(distances.keys())
            got = D.krum(Gx, users_count, f, distances, True)
            want = orc.krum_select(dense, alive, users_count, f)
            with collect(failures, f"{kind} round {len(chosen)} alive {alive[:4]}..."):
                assert got == want, (got, want)
            if got != want:
                break
            chosen.append(got)
            distances.pop(got)
            if kind == "dict":                 # a DistanceTable's pop already removes the user from every row
                for remaining_user in distances.keys():
                    distances[remaining_user].pop(got)
        with collect(failures, f"{kind}: the tied crafted rows win the first rounds in key order"):
            assert chosen[:2] == [1, 0], chosen[:2]
    assert not failures, "\n".join(failures)
