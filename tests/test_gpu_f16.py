"""fp16 client matrices (AFL_F16) on an H100 (-m gpu).  An fp16 matrix must give the reference's result on its values
upcast to fp32: every fp16 value and every product of two is exact in fp32.

  * Column kernels (mean, ALIE, row gather): bit for bit the fp32 call on G.float().
  * Trimmed mean: against the fp32 kernel on G.float() next to the same comparison for bf16 (so a difference is
    measured, not assumed), and against the C oracle.
  * Distance tables: the bias and spread caps bf16 clients meet, against float64 and against the SIMT kernel;
    duplicate rows give bit-identical table rows and exact zeros; Krum and Bulyan select what the C oracle selects
    wherever its top-1 / top-2 margin exceeds 1e-5; rows holding an inf are never selected.
  * Batched calls: bit for bit the single calls (AFL_GRAM_SPLITS pinned); the sharded path at world size 1: the
    single calls' results.
"""
import os

import numpy as np
import pytest

from oracle import c_oracle as co

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

MARGIN = 1e-5
SPLITS = "3"


@pytest.fixture(scope="module")
def api():
    if not torch.cuda.is_available():
        pytest.skip("no GPU")
    from attacking_federate_learning_b200 import batched, defences, malicious, _device, _native
    from attacking_federate_learning_b200.sharded import ShardedAggregator
    _native.lib()
    return batched, defences, malicious, _device, _native, ShardedAggregator


@pytest.fixture
def splits():
    saved = os.environ.get("AFL_GRAM_SPLITS")

    def set_splits(v):
        if v is None:
            os.environ.pop("AFL_GRAM_SPLITS", None)
        else:
            os.environ["AFL_GRAM_SPLITS"] = v
    yield set_splits
    set_splits(saved)


def hetero(rng, n, d):
    return (0.1 * rng.standard_normal(d) + np.exp(0.25 * rng.standard_normal((n, 1))) * rng.standard_normal((n, d))).astype(np.float32)


def same_bits(a, b):
    a, b = a.contiguous(), b.contiguous()
    return a.shape == b.shape and a.dtype == b.dtype and torch.equal(a.view(torch.uint8), b.view(torch.uint8))


def diff_count(a, b):
    return int((a.contiguous().view(torch.int32) != b.contiguous().view(torch.int32)).sum())


def close_cols(got, ref, G):
    """rtol 1e-5 + 1e-6 x each column's mean |finite value| (the tolerance of the parity tests); non-finite entries
    must be the same."""
    got = np.asarray(got, np.float64); ref = np.asarray(ref, np.float64)
    assert np.array_equal(np.isnan(got), np.isnan(ref)), np.flatnonzero(np.isnan(got) != np.isnan(ref))[:10]
    assert np.array_equal(np.isposinf(got), np.isposinf(ref))
    assert np.array_equal(np.isneginf(got), np.isneginf(ref))
    fin = np.isfinite(ref)
    A = np.where(np.isfinite(G), np.abs(G.astype(np.float64)), 0.0)
    scale = A.sum(0) / np.maximum(np.isfinite(G).sum(0), 1) + 1e-30
    err = np.abs(got[fin] - ref[fin])
    bound = 1e-5 * np.abs(ref[fin]) + 1e-6 * scale[fin]
    assert (err <= bound).all(), (np.flatnonzero(fin)[err > bound][:10], (err / bound).max())


def table_checks(d2, ref2, cap, spread_cap=3e-6):
    """Bias and pair-to-pair spread of the relative error off the diagonal, exact symmetry, zero diagonal (the caps of
    the bf16 client tests)."""
    n = len(d2)
    assert np.array_equal(d2, d2.T) and not d2.diagonal().any()
    off = ~np.eye(n, dtype=bool) & (ref2 > 0) & np.isfinite(ref2)
    rel = (d2[off] - ref2[off]) / ref2[off]
    assert np.abs(rel).max() < cap, np.abs(rel).max()
    assert rel.max() - rel.min() < spread_cap, (rel.min(), rel.max())


def f16_matrix(rng, n, d, ld, f, special):
    """fp16 [n, d] at pitch ld with ALIE ties (rows 0..f-1 identical), and with `special`: +-inf entries in a few
    rows and columns (fewer than f per column, so the trimmed mean's median stays finite) and columns of fp16
    subnormals (|x| < 2^-14)."""
    G = hetero(rng, n, d)
    if f > 1:
        G[:f] = G[f:2 * f].mean(0) - 1.5 * G[f:2 * f].std(0)
    if special:
        G[:, 5::11] *= np.float32(2.0 ** -18)                      # subnormal in fp16, exact in fp32
        G[:, 7::13] = np.float32(2.0 ** -24) * rng.integers(-900, 900, size=(n, len(range(7, d, 13))))
        k = max(min(f - 1, 4), 1)
        for j, c in enumerate(range(3, d, 17)):
            rows = rng.choice(np.arange(f, n), size=k, replace=False)
            G[rows, c] = np.float32(np.inf) if j % 2 else -np.float32(np.inf)
    buf = torch.zeros((n, ld), dtype=torch.float16, device="cuda")
    buf[:, :d] = torch.from_numpy(G).cuda().half()
    return buf[:, :d]


# ================================================================== 1. column kernels
@pytest.mark.parametrize("pitch", ["aligned", "packed"])
@pytest.mark.parametrize("special", [False, True])
@pytest.mark.parametrize("n", [10, 100, 129, 300, 640, 1000, 1025])
def test_f16_column_kernels(api, n, special, pitch):
    bt, D, M, dev, nat, _ = api
    rng = np.random.default_rng(20000 + n + 7 * special + 3 * (pitch == "packed"))
    d = 1003                                                               # d % 8 != 0: a ragged last tile
    ld = 1008 if pitch == "aligned" else d                                 # packed: 16-byte loads do not apply
    f = max(n // 4, 2)
    G16 = f16_matrix(rng, n, d, ld, f, special)
    G32 = G16.float()                                                      # the upcast values (exact)
    G = G32.cpu().numpy()
    if special:
        assert ((G != 0) & (np.abs(G) < 2.0 ** -14)).any() and np.isinf(G).any()

    # mean, ALIE statistics, row gather: bit for bit the fp32 kernels on the upcast matrix
    assert same_bits(D.no_defense(G16, n, f), D.no_defense(G32, n, f))
    for z in (1.5, 0.0):
        r16 = dev.alie(G16[:f], z, None, alias_mean=False)
        r32 = dev.alie(G32[:f], z, None, alias_mean=False)
        assert all(same_bits(a, b) for a, b in zip(r16, r32)), z
    for k in (0, n // 2, n - 1, -1):
        idx = torch.tensor([k], dtype=torch.int32, device="cuda")
        assert same_bits(dev.gather_row(G16, idx), dev.gather_row(G32, idx)), k
    # ALIE written back into rows 0..f-1 (through a cast) and its crafted vector, against the fp32 route
    A16, A32 = G16.clone(), G32.clone()
    c16 = M.DriftAttack(1.5).attack_rows(A16, f)
    c32 = M.DriftAttack(1.5).attack_rows(A32, f)
    assert same_bits(c16, c32)
    assert same_bits(A16[:f], A32[:f].half()) and same_bits(A16[f:], G16[f:])
    assert all(torch.equal(A16[i].view(torch.int16), A16[0].view(torch.int16)) for i in range(f))

    # trimmed mean (the ALIE ties sit at the keep boundary), all rows and a row_index subset in a shuffled order
    rows = rng.permutation(n)[:max(n - n // 5, 3)].astype(np.int32)
    ri = torch.from_numpy(rows).cuda()
    Gb = G32.bfloat16()
    Gbf = Gb.float()
    tm = {"f16": D.trimmed_mean(G16, n, f), "f16/fp32": D.trimmed_mean(G32, n, f),
          "bf16": D.trimmed_mean(Gb, n, f), "bf16/fp32": D.trimmed_mean(Gbf, n, f),
          "f16 rows": dev.trimmed_mean(G16, f, row_index=ri), "f16 rows/fp32": dev.trimmed_mean(G32, f, row_index=ri),
          "bf16 rows": dev.trimmed_mean(Gb, f, row_index=ri), "bf16 rows/fp32": dev.trimmed_mean(Gbf, f, row_index=ri)}
    # A 16-bit tile holds a column in a different word-column than the fp32 tile, which permutes the order in which the
    # kept deviations are summed: bit-identical unless an fp32 sum rounds differently in that order.  Measured on an
    # H100: bf16 never differed here (its 8-bit values mostly sum exactly), fp16 in 1 of 1,003 columns in 2 of the 56
    # comparisons.  Both are held to the same tolerance against the fp32 kernel, and the counts are printed (-s).
    diffs = {k: diff_count(tm[k], tm[k + "/fp32"]) for k in ("f16", "bf16", "f16 rows", "bf16 rows")}
    print(f"n={n} special={special} pitch={pitch}: columns differing from the fp32 kernel on the upcast matrix {diffs}")
    Gbh = Gbf.cpu().numpy()
    for k in ("f16", "f16 rows", "bf16", "bf16 rows"):
        Gk = G if k.startswith("f16") else Gbh
        close_cols(tm[k].cpu().numpy(), tm[k + "/fp32"].cpu().numpy(), Gk[rows] if "rows" in k else Gk)
        assert diffs[k] <= d // 100, diffs
    ref = co.trimmed_mean(G, f)
    close_cols(tm["f16"].cpu().numpy(), ref, G)
    close_cols(tm["f16/fp32"].cpu().numpy(), ref, G)
    ref_rows = co.trimmed_mean(G, f, rows=rows)
    close_cols(tm["f16 rows"].cpu().numpy(), ref_rows, G[rows])
    close_cols(tm["bf16"].cpu().numpy(), co.trimmed_mean(Gbh, f), Gbh)


# ================================================================== 2. distances and selection
SEL_SHAPES = {                  # n, d, ld, f (Krum), f (Bulyan)
    "one_tile_100": (100, 32768, 32768, 24, 24),
    "one_tile_128": (128, 8200, 8200, 31, 31),
    "tiles_200": (200, 8192, 8192, 48, 48),
    "tiles_1000": (1000, 4096, 4096, 240, 240),
    "simt_unaligned": (100, 4099, 4099, 24, 24),            # pitch 8198 bytes: the SIMT kernel
}


@pytest.mark.parametrize("shape", list(SEL_SHAPES))
def test_f16_distances_and_selection(api, shape):
    bt, D, M, dev, nat, _ = api
    n, d, ld, f, fb = SEL_SHAPES[shape]
    rng = np.random.default_rng(21000 + n + d)
    G16 = torch.from_numpy(hetero(rng, n, d)).cuda().half()
    G = G16.float().cpu().numpy()
    ref2 = co.pairwise_sqdist(G)
    simt = dev.sqdist_partial(G16, nat.GRAM_FORCE_SIMT).cpu().numpy()
    table_checks(simt, ref2, 1e-6, spread_cap=2e-6)
    auto = dev.sqdist_partial(G16).cpu().numpy()
    if shape == "simt_unaligned":
        assert np.array_equal(auto, simt)
        with pytest.raises(NotImplementedError):
            dev.sqdist_partial(G16, nat.GRAM_FORCE_TCGEN05)
    else:
        tc = dev.sqdist_partial(G16, nat.GRAM_FORCE_TCGEN05).cpu().numpy()
        assert np.array_equal(auto, tc)
        table_checks(tc, ref2, 6e-6)                           # the bf16 clients' caps (tests/test_gpu_scale_parity.py)
        table_checks(tc, simt, 6e-6)
        # the fp32 operand flags do not apply to 16-bit clients
        for flags in (nat.GRAM_TF32X2, nat.GRAM_SINGLE_PASS, nat.GRAM_BF16X2, nat.GRAM_NO_CENTER):
            assert np.array_equal(dev.sqdist_partial(G16, flags).cpu().numpy(), tc), flags
    want, margin = co.krum_select(np.sqrt(ref2), n, f, with_margin=True)
    got = D.krum(G16, n, f, return_index=True)
    if margin > MARGIN or margin == 0.0:
        assert got == want, (got, want, margin)
    assert same_bits(D.krum(G16, n, f), G16[got])
    out, sel = D.bulyan(G16, n, fb, return_selection=True)
    sel = sel.cpu().tolist()
    gpu_table = D._krum_create_distances(G16).dense.cpu().numpy().astype(np.float64)
    assert sel == co.bulyan_select(gpu_table, n, fb)
    want_sel, margins = co.bulyan_select(np.sqrt(ref2), n, fb, with_margins=True)
    first_close = next((i for i, m in enumerate(margins) if 0.0 < m <= MARGIN), len(margins))
    assert sel[:first_close] == want_sel[:first_close]
    close_cols(out.cpu().numpy(), co.trimmed_mean(G, 2 * fb, rows=sel), G)


@pytest.mark.parametrize("n,d,f", [(80, 40960, 19), (128, 8192, 31), (200, 8192, 48), (1000, 4096, 240),
                                   (100, 4099, 24)])
def test_f16_alie_rows_tie_to_user_1(api, n, d, f):
    """ALIE makes rows 0..f-1 one vector (at n = 1000 they span the first two 128-row tiles): bit-identical table
    rows, exact zeros between them, and Krum's [1, 0, 2, ...] tie-break picks user 1."""
    bt, D, M, dev, nat, _ = api
    rng = np.random.default_rng(22000 + n)
    G = 5.0 * hetero(rng, n, d)
    G[:f] = 0.002 * G[f]
    G16 = torch.from_numpy(G).cuda().half()
    M.DriftAttack(1.5).attack_rows(G16, f)
    assert all(torch.equal(G16[i], G16[0]) for i in range(1, f))
    flags = [nat.GRAM_FORCE_SIMT] + ([nat.GRAM_FORCE_TCGEN05] if d % 8 == 0 else [])
    for fl in flags:
        d2 = dev.sqdist_partial(G16, fl)
        assert float(d2[:f, :f].abs().max()) == 0.0, fl
        assert bool((d2[:f, f:] == d2[0:1, f:]).all()), fl
        assert bool((d2[f:, :f] == d2[f:, 0:1]).all()), fl
    assert D.krum(G16, n, f, return_index=True) == 1


@pytest.mark.parametrize("n,d,f", [(12, 1000, 2), (100, 32768, 24), (300, 4096, 70), (100, 4099, 24)])
def test_f16_rows_with_inf_never_selected(api, n, d, f):
    bt, D, M, dev, nat, Sharded = api
    rng = np.random.default_rng(23000 + n)
    G = hetero(rng, n, d)
    bad = list(range(max(f - 1, 1)))
    for k, u in enumerate(bad):
        G[u, (3 * k + np.arange(3)) % d] = np.array([(1, 1, 1), (-1, -1, -1), (1, -1, 1)][k % 3], np.float32) * np.inf
    G16 = torch.from_numpy(G).cuda().half()
    routes = {"device": D.krum(G16, n, f, return_index=True), "sharded": Sharded().krum(G16, n, f, return_index=True)}
    for name, fl in (("simt", nat.GRAM_FORCE_SIMT), ("auto", 0)):
        d2 = dev.sqdist_partial(G16, fl)
        routes[name] = int(dev.krum_from_sqdist(d2, n, f).item())
        t = d2.cpu().numpy()
        assert np.isposinf(t[bad][:, len(bad):]).all(), name
    assert not set(routes.values()) & set(bad), routes
    want, margin = co.krum_select(np.sqrt(co.pairwise_sqdist(G16.float().cpu().numpy())), n, f, with_margin=True)
    assert want not in bad
    for route, idx in routes.items():
        if margin > MARGIN or margin == 0.0:
            assert idx == want, (route, idx, want, margin)
    if n >= 4 * f + 3:
        _, sel = D.bulyan(G16, n, f, return_selection=True)
        assert not set(sel.cpu().tolist()) & set(bad)


# ================================================================== 3. batched
def f16_batch(shape_id):
    rng = np.random.default_rng(24000 + len(shape_id))
    if shape_id == "tensor_one_tile":              # 4 x 51 x 8,192: the one-tile map {d, n, B}
        B, n, d, ld = 4, 51, 8_192, 8_192
    else:                                          # 5 x 10 x 79,510: pitch 159,020 bytes, the SIMT kernel
        B, n, d, ld = 5, 10, 79_510, 79_510
    G = (0.1 * rng.standard_normal((B, 1, d)) + np.exp(0.25 * rng.standard_normal((B, n, 1)))
         * rng.standard_normal((B, n, d))).astype(np.float32)
    buf = torch.zeros((B, n, ld), dtype=torch.float16, device="cuda")
    buf[:, :, :d] = torch.from_numpy(G).cuda().half()
    return buf[:, :, :d]


@pytest.mark.parametrize("shape_id", ["tensor_one_tile", "simt"])
def test_f16_batch_matches_single_calls(api, splits, shape_id):
    bt, D, M, dev, nat, _ = api
    G = f16_batch(shape_id)
    B, n, _ = G.shape
    f = 2 if n == 10 else 12
    fb = 1 if n == 10 else 12
    splits(SPLITS)
    idx = bt.krum(G, n, f, return_index=True)
    ws = dev.Workspace.get(G.device, "batched", 0)
    tables = ws[:B * n * n * 8].view(torch.float64).view(B, n, n).clone()
    rows = bt.krum(G, n, f)
    out, sel = bt.bulyan(G, n, fb, return_selection=True)
    tm, mean = bt.trimmed_mean(G, n, f), bt.no_defense(G, n, f)
    idx_h = idx.cpu().tolist()
    for b in range(B):
        assert same_bits(tables[b], dev.sqdist_partial(G[b])), b
        assert idx_h[b] == D.krum(G[b], n, f, return_index=True), b
        assert same_bits(rows[b], G[b, idx_h[b]])
        out1, sel1 = D.bulyan(G[b], n, fb, return_selection=True)
        assert same_bits(sel[b].cpu(), sel1.cpu()) and same_bits(out[b], out1), b
        assert same_bits(tm[b], D.trimmed_mean(G[b], n, f)) and same_bits(mean[b], D.no_defense(G[b], n, f)), b
    # per-problem corrupted counts and attack strengths
    fs = [b % (f + 1) for b in range(B)]
    fbs = [b % (fb + 1) for b in range(B)]
    idx_e = bt.krum(G, n, fs, return_index=True).cpu().tolist()
    out_e, sel_e = bt.bulyan(G, n, fbs, return_selection=True)
    tm_e = bt.trimmed_mean(G, n, fs)
    for b in range(B):
        assert idx_e[b] == D.krum(G[b], n, fs[b], return_index=True), b
        out1, sel1 = D.bulyan(G[b], n, fbs[b], return_selection=True)
        assert same_bits(sel_e[b, :len(sel1)].cpu(), sel1.cpu()) and same_bits(out_e[b], out1), b
        assert same_bits(tm_e[b], D.trimmed_mean(G[b], n, fs[b])), b
    # ALIE, scalar and per problem, written back through a cast: each problem as the single attack_rows call
    zs = [1.5, 0.0, 0.5, 2.0, 1.0][:B]
    for fa, za in ((f, 1.5), (fs, zs)):
        Gb = torch.empty_strided(G.shape, G.stride(), dtype=G.dtype, device=G.device).copy_(G)
        crafted, mu, sigma = bt.alie_rows(Gb, fa, za)
        for b in range(B):
            fb_, zb = (fa[b], za[b]) if isinstance(fa, list) else (fa, za)
            one = G[b].clone()
            if fb_ > 0:
                _, mu1, sigma1 = dev.alie(G[b, :fb_], zb, None, alias_mean=False)
                crafted1 = M.DriftAttack(zb).attack_rows(one, fb_)
                assert same_bits(mu[b], mu1) and same_bits(sigma[b], sigma1), b
                if zb != 0:
                    assert same_bits(crafted[b], crafted1), b
            assert same_bits(Gb[b], one), b


# ================================================================== 4. sharded (world size 1) and the server
@pytest.mark.parametrize("n,d,f", [(100, 32768, 24), (200, 8192, 48), (100, 4099, 24)])
def test_f16_sharded_world_1(api, n, d, f):
    bt, D, M, dev, nat, Sharded = api
    rng = np.random.default_rng(25000 + n)
    G16 = torch.from_numpy(hetero(rng, n, d)).cuda().half()
    agg = Sharded()
    assert agg.krum(G16, n, f, return_index=True) == D.krum(G16, n, f, return_index=True)
    out, sel = agg.bulyan(G16, n, f, return_selection=True)
    out1, sel1 = D.bulyan(G16, n, f, return_selection=True)
    assert same_bits(sel.cpu(), sel1.cpu()) and same_bits(out, out1)
    assert same_bits(agg.trimmed_mean(G16, n, f), D.trimmed_mean(G16, n, f))
    assert same_bits(agg.no_defense(G16), D.no_defense(G16, n, f))


def test_f16_aggregation_server(api):
    from attacking_federate_learning_b200.server import AggregationServer
    bt, D, M, dev, nat, _ = api
    rng = np.random.default_rng(26)
    n, d = 10, 79510
    G = hetero(rng, n, d)
    srv = AggregationServer(n, d, mal_prop=0.24, learning_rate=0.1, momentum=0.9, dtype=torch.float16)

    class U:
        def __init__(self, g): self.grads = g
    srv.collect_gradients([U(torch.from_numpy(g).half()) for g in G])
    torch.cuda.synchronize()
    G16 = srv.users_grads
    assert G16.dtype == torch.float16
    for rule in ("Krum", "TrimmedMean", "NoDefense"):
        want = D.defend[rule](G16, n, int(n * 0.24)).float()
        assert same_bits(srv.defend(rule), want), rule
