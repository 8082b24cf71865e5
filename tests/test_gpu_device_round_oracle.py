"""batched.DeviceRound against float64 and exact oracles, problem by problem (-m gpu).  test_gpu_device_round holds
the device-parameter calls to the host-parameter calls; a mistake both routes shared would pass there.  Here every
result is held to oracle/c_oracle.py, oracle/ref_numpy.py or exact NumPy arithmetic instead:

A. ALIE's in-kernel 16-bit write (alie_write16_kernel), bf16 and fp16, at every instance: a 16-byte-aligned pitch with
   D % 8 = 0 (VEC = 8, full width) and D % 8 != 0 (VEC = 8, the last thread's scalar tail), an odd pitch and a batch
   stride that is not a multiple of 8 elements (VEC = 1).  Pad columns, rows past N and the gap between problems hold
   a sentinel NaN.  Oracle: the float64 statistics of the upcast rows, each rounded once to fp32, and
   crafted = fl(mu - fl(z sigma)) (DESIGN 2.3); values with |x| >= 2^-6 keep the float64 sums exact.  Rows 0..f_b-1
   must hold crafted rounded to nearest even (np.float16, or the bf16 carry rule on the fp32 bits; NaN as NaN), every
   other element its old bits.  Problems: f = 0, f = N, z = 0 (statistics only), negative z, fp16 overflow to +-inf,
   and +-inf in the malicious rows (mu +-inf or NaN, sigma NaN as np.var gives, crafted NaN).
B. ALIE and the attack metrics past one tile (N = 129, 500, 1000; fp32, bf16; whole slot and ragged): ALIE against
   co.alie, the honest mean bit for bit against the fp32 mean of rows f_b..rows_b-1, the relative deviation and its
   two sums against float64, krum_success and the selection counts exactly for host-built indices and selections
   holding -1 and -2.
C. One round at B = 200 > 128 problems (two table CTAs), N = 40, every problem with its own rows, f and users count
   per rule, on the exact-integer columns of test_gpu_trimmed_mean_exact: Krum against co.krum_select and Bulyan's
   selection against co.bulyan_select where the float64 margins are clear, the trimmed mean, the mean and Bulyan's
   second stage against ref_numpy bit for bit, ALIE against co.alie.
D. One captured round (alie, krum rows, bulyan, trimmed_mean, attack_metrics) replayed over a valid grid, the same grid
   with four problems flagged (rows_b = N + 1 on an all-+inf slot, Krum's precondition, Bulyan's users_count != rows,
   NaN rows), the valid grid again without clearing (codes sticky, outputs back on the oracles), and after
   clear_status.
"""
import numpy as np
import pytest

from oracle import c_oracle as co
from oracle import ref_numpy as orc
from test_gpu_batched_oracle import collect
from test_gpu_edges import hetero
from test_gpu_metrics import oracle_deviation
from test_gpu_trimmed_mean_exact import assert_same_bits, close_cols, exact_matrix, ref_tm, value_cap

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

MARGIN = 1e-5
TORCH16 = {"bf16": torch.bfloat16, "f16": torch.float16}
SENTINEL = 0x7FA5                  # a NaN in both formats, which no kernel writes


@pytest.fixture(scope="module")
def api():
    if not torch.cuda.is_available():
        pytest.skip("no GPU")
    from attacking_federate_learning_b200 import batched, _native
    _native.lib()
    return batched, _native


def dev_i32(v):
    return torch.as_tensor(np.asarray(v, np.int32), device="cuda")


def fill(rm, f=None, z=None, rows=None, users=None):
    for t, v, dt in ((rm.f, f, np.int32), (rm.z, z, np.float64), (rm.rows, rows, np.int32),
                     (rm.users_count, users, np.int32)):
        if v is not None:
            t.copy_(torch.as_tensor(np.asarray(v, dt), device="cuda"))


# ---- exact ALIE oracle -------------------------------------------------------------------------------------------
def fma_neg_sq(m, t):
    """t - m*m with one rounding (the kernel's fma(-m, m, t)): Dekker's exact product and a TwoSum."""
    p = m * m
    c = 134217729.0 * m
    hi = c - (c - m)
    lo = m - hi
    e = ((hi * hi - p) + 2.0 * hi * lo) + lo * lo             # m*m = p + e exactly
    r = t - p
    bv = r - t
    es = (t - (r - bv)) + (-p - bv)                           # r + es = t - p exactly
    return r + (es - e)


def alie_exact(X, f, z):
    """(crafted, mu, sigma) fp32 of rows 0..f-1 of X (fp32): float64 sums, m = s1 (1/f), var = fma(-m, m, s2 (1/f))
    clamped at 0 (NaN stays NaN, as np.var), each statistic rounded once to fp32, crafted = fl(mu - fl(z sigma))."""
    with np.errstate(all="ignore"):
        x = X[:f].astype(np.float64)
        inv = np.float64(1.0) / np.float64(f)
        m = x.sum(0) * inv
        var = fma_neg_sq(m, (x * x).sum(0) * inv)
        var = np.where(var < 0.0, 0.0, var)
        mu, sigma = m.astype(np.float32), np.sqrt(var).astype(np.float32)
        crafted = (mu - np.float32(z) * sigma).astype(np.float32)
    return crafted, mu, sigma


def bits16(x32, dt):
    """fp32 -> 16-bit bits, round to nearest even (NaN payloads are not compared)."""
    x32 = np.ascontiguousarray(x32, np.float32)
    if dt == "f16":
        with np.errstate(over="ignore"):
            return x32.astype(np.float16).view(np.uint16)
    u = x32.view(np.uint32).astype(np.uint64)
    return ((u + 0x7FFF + ((u >> 16) & 1)) >> 16).astype(np.uint16)


def isnan16(b, dt):
    b = np.asarray(b).view(np.uint16)
    exp, man = (0x7C00, 0x03FF) if dt == "f16" else (0x7F80, 0x007F)
    return ((b & exp) == exp) & ((b & man) != 0)


def magnitudes_at_least(x, lo=2.0 ** -6):
    """|x| >= lo: squares of 16-bit values then span few enough binades that the float64 sums are exact."""
    return np.where(np.abs(x) < lo, np.copysign(lo, x), x).astype(np.float32)


# ================================================================== A. ALIE's 16-bit write
A_N = 40
# name: (D, ld, extra elements between problems after N + 2 rows)
A_LAYOUTS = {"aligned": (1024, 1024, 0), "tail": (1003, 1008, 0), "odd_pitch": (1003, 1005, 0),
             "odd_batch": (1000, 1008, 3)}
A_PROBLEMS = [(0, 1.5, None),          # no malicious row: NaN statistics, nothing written
              (A_N, 1.0, None),        # every row
              (5, 0.0, None),          # statistics only
              (7, -1.25, None),        # negative z
              (3, 7e4, None),          # fp16: crafted below -65504 -> -inf
              (4, -7e4, None),         # fp16: +inf
              (6, 1.5, "inf"),         # +inf, -inf and both in malicious rows; +inf in an honest row
              (1, 2.0, None),          # one row: sigma = 0
              (A_N - 1, 0.5, None)]


@pytest.mark.parametrize("layout", list(A_LAYOUTS))
@pytest.mark.parametrize("dt", list(TORCH16))
def test_alie_write16_against_exact_rounding(api, dt, layout):
    bt, _ = api
    D, ld, extra = A_LAYOUTS[layout]
    B, N = len(A_PROBLEMS), A_N
    bs = (N + 2) * ld + extra
    buf = torch.full((B * bs,), SENTINEL, dtype=torch.int16, device="cuda").view(TORCH16[dt])
    G = buf.as_strided((B, N, D), (bs, ld, 1))
    rng = np.random.default_rng(50000 + 10 * list(TORCH16).index(dt) + list(A_LAYOUTS).index(layout))
    X = magnitudes_at_least(hetero(rng, B * N, D)).reshape(B, N, D)
    for b, (_, _, special) in enumerate(A_PROBLEMS):
        if special == "inf":
            X[b, 1, 3], X[b, 2, 5], X[b, 0, 9], X[b, 3, 9], X[b, 10, 11] = np.inf, -np.inf, np.inf, -np.inf, np.inf
    G.copy_(torch.from_numpy(X).cuda())
    Xu = G.float().cpu().numpy()                          # the upcast values the kernel reads
    before = buf.view(torch.int16).cpu().numpy().view(np.uint16)
    rm = bt.DeviceRound(G, rules=())
    fs, zs = [p[0] for p in A_PROBLEMS], [p[1] for p in A_PROBLEMS]
    fill(rm, fs, zs)
    crafted, mu, sigma = (t.cpu().numpy() for t in rm.alie())
    after = buf.view(torch.int16).cpu().numpy().view(np.uint16)
    assert not rm.status.any()
    failures = []
    for b, (f, z, special) in enumerate(A_PROBLEMS):
        with collect(failures, f"{dt} {layout} problem {b} f {f} z {z}"):
            want_c, want_mu, want_s = alie_exact(Xu[b], f, z)
            assert_same_bits(mu[b], want_mu, "mu")
            assert_same_bits(sigma[b], want_s, "sigma")
            assert_same_bits(crafted[b], want_c, "crafted")
            if special == "inf":
                assert np.isnan(want_c[[3, 5, 9]]).all() and np.isnan(want_s[[3, 5, 9]]).all()
            lo, hi = b * bs, min((b + 1) * bs, len(after))
            want = before[lo:hi].copy()
            nan_ok = np.zeros(hi - lo, bool)
            if f > 0 and z != 0:
                w16 = bits16(want_c, dt)
                if dt == "f16" and abs(z) > 65504:
                    assert ((w16 & 0x7FFF) == 0x7C00)[np.isfinite(want_c)].any(), "no column overflows fp16"
                for r in range(f):
                    want[r * ld:r * ld + D] = w16
                    nan_ok[r * ld:r * ld + D] = np.isnan(want_c)
            got = after[lo:hi]
            bad = (got != want) & ~nan_ok
            bad |= nan_ok & ~isnan16(got, dt)
            where = np.flatnonzero(bad)
            assert where.size == 0, ("elements (row, column) that differ", [divmod(int(i), ld) for i in where[:8]],
                                     got[where[:4]], want[where[:4]])
    assert not failures, "\n".join(failures)


# ================================================================== B. ALIE and metrics past one tile
B_D = 520


def selection_counts(nat, rm, sel):
    """(malicious, selected) per problem from afl_attack_metrics_batched_dev with DeviceRound's own arguments."""
    mal, cnt = (torch.empty(rm.B, dtype=torch.int32, device="cuda") for _ in range(2))
    nat.check(nat.lib().afl_attack_metrics_batched_dev(
        rm.G.data_ptr(), rm.B, rm._bs, rm.N, rm.D, rm._ld, rm._code, rm._ptr(rm.rows), rm.f.data_ptr(), None, None,
        sel.data_ptr(), sel.shape[1], None, None, None, None, mal.data_ptr(), cnt.data_ptr(), rm._ws.data_ptr(),
        rm._ws.numel(), rm.status.data_ptr(), torch.cuda.current_stream().cuda_stream))
    return mal.cpu().numpy(), cnt.cpu().numpy()


def check_written_rows(G_after, G_before, crafted, f, z, dt, what):
    """Rows 0..f-1 hold crafted in G's dtype (written when f > 0 and z != 0), every other row its old values."""
    k = f if (f > 0 and z != 0) else 0
    if k:
        if dt == "f32":
            assert_same_bits(G_after[:k], np.broadcast_to(crafted, G_after[:k].shape), (what, "written rows"))
        else:
            got = G_after[:k].view(np.uint16)
            want = np.broadcast_to(bits16(crafted, dt), got.shape)
            nan = np.broadcast_to(np.isnan(crafted), got.shape)
            assert np.array_equal(got[~nan], want[~nan]) and isnan16(got[nan], dt).all(), (what, "written rows")
    assert np.array_equal(G_after[k:].view(np.uint8), G_before[k:].view(np.uint8)), (what, "rows left alone")


def host_view(G, dt):
    """G as NumPy: fp32 values, or the raw 16-bit words."""
    return G.cpu().numpy() if dt == "f32" else G.view(torch.int16).cpu().numpy().view(np.uint16)


B_CASES = [(n, dt, ragged) for n in (129, 500, 1000) for dt in ("f32", "bf16") for ragged in (False, True)]


@pytest.mark.parametrize("N,dt,ragged", B_CASES,
                         ids=[f"N{n}-{dt}-{'ragged' if r else 'whole'}" for n, dt, r in B_CASES])
def test_alie_and_metrics_past_one_tile(api, N, dt, ragged):
    bt, nat = api
    rows = [N, N - 1, 1, N // 2 + 1, 129] if ragged else [N] * 5
    B = len(rows)
    fs = [0, rows[1] - 1, rows[2], rows[3] // 4, min(rows[4] + 3, N)]       # 0, rows_b - 1, >= rows_b
    zs = [1.5, -0.8, 1.0, 0.0, 2.5]
    rng = np.random.default_rng(51000 + N + 7 * ragged + 3 * (dt == "bf16"))
    X = hetero(rng, B * N, B_D).reshape(B, N, B_D)
    G = torch.from_numpy(X).cuda().to(torch.float32 if dt == "f32" else torch.bfloat16)
    before_vals, before_raw = G.float().cpu().numpy(), host_view(G, dt)
    rm = bt.DeviceRound(G, rules=(), rows=ragged)
    fill(rm, fs, zs, rows if ragged else None)
    crafted, mu, sigma = (t.cpu().numpy() for t in rm.alie())
    Gh, after_raw = G.float().cpu().numpy(), host_view(G, dt)
    agg = torch.from_numpy(Gh.mean(1) + 0.05 * rng.standard_normal((B, B_D)).astype(np.float32)).cuda()
    idx = [-1, fs[1] - 1, rows[2] - 1, -2, rows[4]]            # malicious, honest, -1, -2, past rows_b
    sel = np.stack([rng.integers(-2, N, 24) for _ in range(B)]).astype(np.int32)
    sel[:, 0], sel[:, 1], sel[:, 2] = -1, -2, 0
    idx_d, sel_d = dev_i32(idx), torch.from_numpy(sel).cuda()
    met = {k: v.cpu().numpy() for k, v in rm.attack_metrics(aggregated=agg, return_honest_mean=True).items()}
    met_k = {k: v.cpu().numpy() for k, v in rm.attack_metrics(krum_index=idx_d, selection=sel_d).items()}
    mal, cnt = selection_counts(nat, rm, sel_d)
    assert not rm.status.any()
    agg = agg.cpu().numpy()
    failures = []
    for b, (r, f, z) in enumerate(zip(rows, fs, zs)):
        with collect(failures, f"N {N} {dt} problem {b} rows {r} f {f} z {z}"):
            if f == 0:
                assert np.isnan(crafted[b]).all() and np.isnan(mu[b]).all() and np.isnan(sigma[b]).all()
            else:
                ref_c, ref_mu, ref_s = co.alie(np.ascontiguousarray(before_vals[b, :f]), z)
                np.testing.assert_allclose(crafted[b], ref_c, rtol=1e-5, atol=1e-6)
                np.testing.assert_allclose(mu[b], ref_mu, rtol=1e-5, atol=1e-6)
                np.testing.assert_allclose(sigma[b], ref_s, rtol=1e-5, atol=1e-7)
            check_written_rows(after_raw[b], before_raw[b], crafted[b], f, z, dt, "alie")
            honest = met["honest_mean"][b]
            if f >= r:
                assert np.isnan(honest).all() and np.isnan(met["rel_deviation"][b])
                assert np.isnan(met_k["rel_deviation"][b])
            else:
                h = orc.no_defense(Gh[b, f:r])
                assert_same_bits(honest, h, "honest mean")
                want = oracle_deviation(Gh[b, :r], f, agg[b])
                assert abs(float(met["rel_deviation"][b]) - want) <= 1e-6 * want, ("rel", met["rel_deviation"][b], want)
                h64 = h.astype(np.float64)
                sums = (((agg[b].astype(np.float64) - h64) ** 2).sum(), (h64 ** 2).sum())
                np.testing.assert_allclose(met["deviation_sums"][b], sums, rtol=1e-11)
                if 0 <= idx[b] < r:
                    want = oracle_deviation(Gh[b, :r], f, Gh[b, idx[b]])
                    assert abs(float(met_k["rel_deviation"][b]) - want) <= 1e-6 * want, ("rel krum", idx[b])
                else:
                    assert np.isnan(met_k["rel_deviation"][b]), ("an index outside the rows reads no row", idx[b])
            assert bool(met_k["krum_success"][b]) == (0 <= idx[b] < f)
            s = sel[b]
            want_cnt, want_mal = int((s >= 0).sum()), int(((s >= 0) & (s < f)).sum())
            assert (int(mal[b]), int(cnt[b])) == (want_mal, want_cnt)
            frac = np.float32(want_mal) / np.float32(max(want_cnt, 1))
            assert met_k["bulyan_malicious_fraction"][b] == frac
    assert not failures, "\n".join(failures)


# ================================================================== C. a whole round at B > 128
C_N, C_B = 40, 200
C_ROWS = [1, 2, 3, C_N - 1, C_N, 5, 12, 23, 33, 17]


def c_params(r, k):
    """Per-rule (f, users_count) of a problem with r rows, variant k: the largest legal f of each rule, uc = 2f + 1."""
    kf = [((r - 1) // 2, r), (0, r), (r // 2, 2 * (r // 2) + 1), ((r - 1) // 4, 2 * ((r - 1) // 4) + 1)][k % 4]
    bf = ((r - 3) // 4 if k % 2 == 0 else 0, r) if r >= 3 else (0, r)
    tf = [r - 1, (r - 1) // 2, 0, max(r - 1 - round(3 * r / 4), 0)][k % 4]
    af, az = [(0, 1.5), (r, -0.7), (C_N, 3.0), (r // 2, 0.0)][k % 4]
    return dict(krum=kf, bulyan=bf, tm=tf, alie=(af, az))


def test_whole_round_past_one_table_cta(api):
    bt, nat = api
    N, B = C_N, C_B
    rows = [C_ROWS[b % len(C_ROWS)] for b in range(B)]
    ps = [c_params(r, b // len(C_ROWS)) for b, r in enumerate(rows)]
    rng = np.random.default_rng(52000)
    mats = [exact_matrix(rng, r, "f32", 16, [max(r - p["tm"] - 1, 0)]) for r, p in zip(rows, ps)]
    D = mats[0].shape[1]
    M = value_cap("f32", N)
    buf = rng.integers(-M, M + 1, (B, N, D)).astype(np.float32)          # padding rows: exact integers too
    for b, X in enumerate(mats):
        buf[b, :len(X)] = X
    G = torch.from_numpy(buf).cuda()
    rm = bt.DeviceRound(G, rows=True, per_problem_users_count=True)
    fill(rm, rows=rows)
    st = {}
    fill(rm, [p["krum"][0] for p in ps], users=[p["krum"][1] for p in ps])
    idx = rm.krum(return_index=True).clone()
    krow = rm.krum().clone()
    st["krum"] = rm.status.clone()
    rm.clear_status()
    fill(rm, [p["bulyan"][0] for p in ps], users=[p["bulyan"][1] for p in ps])
    out_b, sel = (t.clone() for t in rm.bulyan(return_selection=True))
    st["bulyan"] = rm.status.clone()
    rm.clear_status()
    fill(rm, [p["tm"] for p in ps], users=rows)
    tm, mean = rm.trimmed_mean().clone(), rm.no_defense().clone()
    st["tm"] = rm.status.clone()
    fill(rm, [p["alie"][0] for p in ps], [p["alie"][1] for p in ps])
    crafted, mu, sigma = (t.cpu().numpy() for t in rm.alie())
    st["alie"] = rm.status.clone()
    after = G.cpu().numpy()
    idx, krow, out_b, sel, tm, mean = (t.cpu().numpy() for t in (idx, krow, out_b, sel, tm, mean))
    st = {k: v.cpu().numpy() for k, v in st.items()}
    assert not st["krum"].any() and not st["tm"].any() and not st["alie"].any(), st
    want_b = [nat.AFL_ERR_PRECONDITION if r < 3 else 0 for r in rows]       # Bulyan needs rows >= 4 f + 3 >= 3
    assert st["bulyan"].tolist() == want_b
    failures = []
    for b, (X, r, p) in enumerate(zip(mats, rows, ps)):
        with collect(failures, f"problem {b} rows {r} {p}"):
            dist = np.sqrt(co.pairwise_sqdist(X))
            f, uc = p["krum"]
            o, margin = co.krum_select(dist, uc, f, with_margin=True)
            assert margin <= MARGIN or idx[b] == o, ("krum", idx[b], o, margin)
            assert_same_bits(krow[b], X[idx[b] if idx[b] >= 0 else r - 1], "krum row")
            f = p["bulyan"][0]
            theta = r - 2 * f
            if r >= 3:
                want, margins = co.bulyan_select(dist, r, f, with_margins=True)
                k = next((j for j, m in enumerate(margins) if not m > MARGIN), theta)
                assert sel[b, :k].tolist() == want[:k], ("bulyan", sel[b, :k][:8], want[:k][:8])
                assert (sel[b, theta:] == -2).all()
                s = sel[b, :theta]
                assert len(set(s.tolist())) == theta and s.min() >= 0 and s.max() < r
                assert_same_bits(out_b[b], ref_tm(X[s], 2 * f), "bulyan second stage")
            else:                                                            # the safe row: N rows, f = 0
                assert sel[b].min() >= 0 and sel[b].max() < N
            assert_same_bits(tm[b], ref_tm(X, p["tm"]), "trimmed mean")
            assert_same_bits(mean[b], orc.no_defense(X), "mean")
            f, z = p["alie"]
            if f == 0:
                assert np.isnan(crafted[b]).all()
            else:
                ref_c, ref_mu, ref_s = co.alie(np.ascontiguousarray(buf[b, :f]), z)
                np.testing.assert_allclose(crafted[b], ref_c, rtol=1e-5, atol=1e-6)
                np.testing.assert_allclose(mu[b], ref_mu, rtol=1e-5, atol=1e-6)
                np.testing.assert_allclose(sigma[b], ref_s, rtol=1e-5, atol=1e-7)
            check_written_rows(after[b], buf[b], crafted[b], f, z, "f32", "alie")
    assert not failures, "\n".join(failures)


# ================================================================== D. status across replays of one captured round
D_N, D_D = 32, 1000
D_ROWS = [32, 31, 20, 9, 32, 3, 27, 16]
D_F = [7, 2, 4, 1, 0, 0, 6, 3]                        # Bulyan's largest f or less: legal for every call
D_Z = [1.5, 0.5, 0.0, -1.0, 2.0, 1.0, 0.7, 3.0]


def d_grid(seed):
    rng = np.random.default_rng(seed)
    return hetero(rng, len(D_ROWS) * D_N, D_D).reshape(len(D_ROWS), D_N, D_D)


def check_round(outs, G, X, rows, fs, zs, ucs, problems, what):
    """Every listed problem's outputs of one replay against the oracles; X: the slots before ALIE wrote them."""
    o = {k: v.cpu().numpy() for k, v in outs.items()}
    Gh = G.cpu().numpy()
    failures = []
    for b in problems:
        r, f, z, uc = rows[b], fs[b], zs[b], ucs[b]
        with collect(failures, f"{what} problem {b} rows {r} f {f} z {z}"):
            if f == 0:
                assert np.isnan(o["crafted"][b]).all()
            else:
                ref_c, ref_mu, ref_s = co.alie(np.ascontiguousarray(X[b, :f]), z)
                np.testing.assert_allclose(o["crafted"][b], ref_c, rtol=1e-5, atol=1e-6)
                np.testing.assert_allclose(o["sigma"][b], ref_s, rtol=1e-5, atol=1e-7)
            check_written_rows(Gh[b], X[b], o["crafted"][b], f, z, "f32", "alie")
            Y = np.ascontiguousarray(Gh[b, :r])
            dist = np.sqrt(co.pairwise_sqdist(Y))
            i = int(o["idx"][b])
            want, margin = co.krum_select(dist, uc, f, with_margin=True)
            assert margin <= MARGIN or i == want, ("krum", i, want, margin)
            assert_same_bits(o["krow"][b], Y[i if i >= 0 else r - 1], "krum row")
            theta = r - 2 * f
            want, margins = co.bulyan_select(dist, r, f, with_margins=True)
            k = next((j for j, m in enumerate(margins) if not m > MARGIN), theta)
            s = o["sel"][b]
            assert s[:k].tolist() == want[:k] and (s[theta:] == -2).all(), ("bulyan", s[:8], want[:8])
            close_cols(o["bulyan"][b], co.trimmed_mean(Y, 2 * f, rows=s[:theta]), Y[s[:theta]])
            close_cols(o["tm"][b], co.trimmed_mean(Y, f), Y)
            h = orc.no_defense(Y[f:])
            assert_same_bits(o["honest"][b], h, "honest mean")
            rel = oracle_deviation(Y, f, o["bulyan"][b])
            assert abs(float(o["rel"][b]) - rel) <= 1e-6 * rel, ("rel", o["rel"][b], rel)
            mal, cnt = int(((s >= 0) & (s < f)).sum()), int((s >= 0).sum())
            assert o["frac"][b] == np.float32(mal) / np.float32(max(cnt, 1))
            assert bool(o["hit"][b]) == (0 <= i < f)
            if 0 <= i < r:
                rel = oracle_deviation(Y, f, Y[i])
                assert abs(float(o["rel_k"][b]) - rel) <= 1e-6 * rel, ("rel krum", o["rel_k"][b], rel)
    assert not failures, "\n".join(failures)


def test_status_across_replays_of_one_captured_round(api):
    bt, nat = api
    B, N = len(D_ROWS), D_N
    X = d_grid(53000)
    G = torch.from_numpy(X).cuda()
    rm = bt.DeviceRound(G, rows=True, per_problem_users_count=True)

    def round_():
        crafted, mu, sigma = rm.alie()
        krow = rm.krum()
        out_b, sel = rm.bulyan(return_selection=True)
        tm = rm.trimmed_mean()
        met = rm.attack_metrics(aggregated=out_b, selection=sel, return_honest_mean=True)
        met_k = rm.attack_metrics(krum_index=rm.krum_index)
        return dict(crafted=crafted, sigma=sigma, krow=krow, idx=rm.krum_index, bulyan=out_b, sel=sel, tm=tm,
                    honest=met["honest_mean"], rel=met["rel_deviation"], frac=met["bulyan_malicious_fraction"],
                    rel_k=met_k["rel_deviation"], hit=met_k["krum_success"])

    def refill(Xs, rows, fs, zs, ucs):
        G.copy_(torch.from_numpy(Xs).cuda())
        fill(rm, fs, zs, rows, ucs)

    refill(X, D_ROWS, D_F, D_Z, D_ROWS)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        round_()                                                 # eager warm-up
    torch.cuda.current_stream().wait_stream(s)
    torch.cuda.synchronize()
    assert not rm.status.any()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        outs = round_()

    def replay(Xs, rows, fs, zs, ucs):
        refill(Xs, rows, fs, zs, ucs)
        graph.replay()
        torch.cuda.synchronize()
        return rm.status.cpu().tolist()

    every = range(B)
    failures = []                                                # every step runs, whatever an earlier one found
    with collect(failures, "1. valid grid"):
        assert replay(X, D_ROWS, D_F, D_Z, D_ROWS) == [0] * B
        check_round(outs, G, X, D_ROWS, D_F, D_Z, D_ROWS, every, "valid")
    # 2. four problems flagged, each with its own code
    Xb, rows, fs, zs, ucs = X.copy(), list(D_ROWS), list(D_F), list(D_Z), list(D_ROWS)
    rows[1], zs[1], Xb[1] = N + 1, 0.0, np.inf                  # rows_b outside [1, N], on an all-+inf slot
    fs[3] = 5                                                   # Krum: users_count 9 < 2 f + 1
    ucs[6] = rows[6] + 1                                        # Bulyan: users_count != rows (and >= 4 f + 3)
    Xb[7] = np.nan                                              # Bulyan's first round finds no eligible user
    codes = [0, nat.AFL_ERR_BAD_ARG, 0, nat.AFL_ERR_PRECONDITION, 0, 0, nat.AFL_ERR_UNSUPPORTED, nat.AFL_ERR_NO_WINNER]
    with collect(failures, "2. flagged grid"):
        assert replay(Xb, rows, fs, zs, ucs) == codes
    with collect(failures, "2. flagged grid, outputs"):
        assert int(outs["idx"][1]) == -1                        # the safe row's Krum finds nobody on +inf rows
        assert torch.equal(outs["krow"][1], G[1, N - 1]) and bool(torch.isposinf(outs["krow"][1]).all())
        check_round(outs, G, Xb, rows, fs, zs, ucs, [0, 2, 4, 5], "flagged grid")
    # 3. the valid grid again without clearing: the codes stay, the outputs follow the valid values
    with collect(failures, "3. valid grid, codes kept"):
        assert replay(X, D_ROWS, D_F, D_Z, D_ROWS) == codes
    with collect(failures, "3. valid grid, outputs"):
        check_round(outs, G, X, D_ROWS, D_F, D_Z, D_ROWS, every, "valid again, codes kept")
    # 4. cleared
    rm.clear_status()
    with collect(failures, "4. cleared"):
        assert replay(X, D_ROWS, D_F, D_Z, D_ROWS) == [0] * B
        check_round(outs, G, X, D_ROWS, D_F, D_Z, D_ROWS, every, "cleared")
    assert not failures, "\n".join(failures)
