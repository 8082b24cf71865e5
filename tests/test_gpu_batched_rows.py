"""Ragged batched aggregation (batched.py with `rows=`, afl_defend_batched_rows, afl_attack_metrics_batched_rows) on an
H100 (-m gpu).  Problem b is G[b, :rows_b] of a [B, N, D] batch:
  * its results are, bit for bit, the single device call's on G[b, :rows_b] with users_count_b and f_b (Krum's index
    and row, Bulyan's output and selection, the trimmed mean, the mean), for fp32, bf16 and fp16, on the tensor-core
    and the SIMT Gram paths (split count pinned; fp32 at D < 32768, where both sides run split-TF32 operands);
  * rows past rows_b never change a result (zeros, NaN, +-inf, +-1e30), also in the default fp32 format at N = 100,
    D >= 32768, whose bf16x2 operands are centred on each problem's own last rows;
  * with rows_b = N everywhere it is afl_defend_batched_each, distance tables included;
  * in the default format its selections match the C oracle wherever the oracle's top-1 / top-2 margin exceeds 1e-5;
  * its metrics are the single-problem metrics of G[b, :rows_b].
"""
import os

import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

SPLITS = "3"
MARGIN = 1e-5
ROWS = [1, 2, 3, 7, 8, 9, 10, 16, 51, 64, 100]


@pytest.fixture(scope="module")
def api():
    if not torch.cuda.is_available():
        pytest.skip("no GPU")
    from attacking_federate_learning_b200 import batched, defences, _device, _native
    _native.lib()
    return batched, defences, _device, _native


@pytest.fixture
def splits():
    saved = os.environ.get("AFL_GRAM_SPLITS")
    os.environ["AFL_GRAM_SPLITS"] = SPLITS
    yield
    if saved is None:
        os.environ.pop("AFL_GRAM_SPLITS", None)
    else:
        os.environ["AFL_GRAM_SPLITS"] = saved


def same_bits(a, b):
    a, b = a.contiguous(), b.contiguous()
    return a.shape == b.shape and a.dtype == b.dtype and torch.equal(a.view(torch.uint8), b.view(torch.uint8))


def make(rows, N, D, ld, dtype, seed=0):
    """[B, N, D] view of a [B, N, ld] buffer: heterogeneous clients around a common component, padding rows = 0."""
    rng = np.random.default_rng(seed)
    B = len(rows)
    common = 0.1 * rng.standard_normal((B, 1, ld), dtype=np.float32)
    scale = np.exp(0.25 * rng.standard_normal((B, N, 1))).astype(np.float32)
    G = common + scale * rng.standard_normal((B, N, ld), dtype=np.float32)
    for b, r in enumerate(rows):
        G[b, r:] = 0.0
    return torch.from_numpy(G).cuda().to(dtype)[:, :, :D]


def fill_padding(G, rows, kind):
    """Padding rows of every problem: zeros, or a mix of NaN, +-inf and +-1e30."""
    G = G.clone()
    for b, r in enumerate(rows):
        if r == G.shape[1]:
            continue
        if kind == "zero":
            G[b, r:] = 0
        else:
            pad = torch.tensor([float("nan"), float("inf"), -float("inf"), 1e30, -1e30], device=G.device)
            k = torch.arange((G.shape[1] - r) * G.shape[2], device=G.device) % 5
            G[b, r:] = pad[k].view(G.shape[1] - r, G.shape[2]).to(G.dtype)
    return G


def fk(r):            # the sweep's malicious share: f = int(0.24 n)
    return int(0.24 * r)


def fb(r):            # the largest f with r >= 4 f + 3
    return (r - 3) // 4


def run_all(bt, G, rows):
    """Every rule's results on one ragged batch (Bulyan over the problems with rows_b >= 3)."""
    kf, tf = [fk(r) for r in rows], [fk(r) for r in rows]
    idx = bt.krum(G, None, kf, return_index=True, rows=rows)
    krow = bt.krum(G, None, kf, rows=rows)
    tm = bt.trimmed_mean(G, None, tf, rows=rows)
    mean = bt.no_defense(G, None, 0, rows=rows)
    keep = [b for b, r in enumerate(rows) if r >= 3]
    brows = [rows[b] for b in keep]
    out, sel = bt.bulyan(G[keep], None, [fb(r) for r in brows], return_selection=True, rows=brows)
    return dict(idx=idx, krow=krow, tm=tm, mean=mean, bout=out, bsel=sel), keep


CASES = [(dt, path) for dt in ("float32", "bfloat16", "float16") for path in ("tensor", "simt")]


@pytest.mark.parametrize("dtype,path", CASES, ids=[f"{d}-{p}" for d, p in CASES])
@pytest.mark.parametrize("N", [100, 128])
def test_rows_match_single_calls(api, splits, dtype, path, N):
    bt, Dm, _, _ = api
    rows = ROWS + ([128, 127] if N == 128 else [])
    D, ld = (4096, 4096) if path == "tensor" else (4099, 4099)
    G = make(rows, N, D, ld, getattr(torch, dtype), seed=N)
    res, keep = run_all(bt, G, rows)
    idx = res["idx"].cpu().tolist()
    for b, r in enumerate(rows):
        Gb = G[b, :r]
        assert idx[b] == Dm.krum(Gb, r, fk(r), return_index=True), (b, r)
        want_row = Gb[idx[b]] if idx[b] >= 0 else Gb[r - 1]
        assert same_bits(res["krow"][b], want_row), (b, r)
        assert same_bits(res["tm"][b], Dm.trimmed_mean(Gb, r, fk(r))), (b, r)
        assert same_bits(res["mean"][b], Dm.no_defense(Gb, r, 0)), (b, r)
    sel = res["bsel"].cpu()
    for j, b in enumerate(keep):
        r = rows[b]
        out1, sel1 = Dm.bulyan(G[b, :r], r, fb(r), return_selection=True)
        theta = r - 2 * fb(r)
        assert same_bits(sel[j, :theta], sel1.cpu()) and bool((sel[j, theta:] == -2).all()), (b, r)
        assert same_bits(res["bout"][j], out1), (b, r)


@pytest.mark.parametrize("dtype", ["float32", "bfloat16", "float16"])
def test_padding_is_inert(api, dtype):
    bt = api[0]
    N, D = 100, 32768 + 64                     # fp32: the default format is the centred one-tile bf16x2 form
    rows = ROWS
    G = make(rows, N, D, D, getattr(torch, dtype), seed=7)
    ref, _ = run_all(bt, fill_padding(G, rows, "zero"), rows)
    for kind in ("zero", "special"):
        Gp = fill_padding(G, rows, kind)
        got, _ = run_all(bt, Gp, rows)
        for k in ref:
            assert same_bits(got[k], ref[k]), (kind, k)
        fs = [fk(r) for r in rows]
        m1 = bt.attack_metrics(Gp, fs, krum_index=got["idx"], return_honest_mean=True, rows=rows)
        m0 = bt.attack_metrics(fill_padding(G, rows, "zero"), fs, krum_index=ref["idx"], return_honest_mean=True,
                               rows=rows)
        for k in m0:
            assert same_bits(m1[k], m0[k]), (kind, k)


def test_rectangular_rows_equal_each(api, splits):
    bt, _, dev, nat = api
    N, D, B = 100, 32768 + 64, 6
    G = make([N] * B, N, D, D, torch.float32, seed=3)
    rows, fs, fbs = [N] * B, [0, 5, 12, 24, 30, 49], [0, 3, 7, 12, 20, 24]
    L = nat.lib()

    def tables(rule):
        off = L.afl_batched_each_workspace_bytes(rule, B, N, D, nat.AFL_F32) - \
            L.afl_batched_workspace_bytes(rule, B, N, D, nat.AFL_F32)
        ws = dev.Workspace.get(G.device, "batched", 0)
        return ws[off:off + B * N * N * 8].view(torch.float64).view(B, N, N).clone()
    a = bt.krum(G, N, fs, return_index=True, rows=rows); ta = tables(b"Krum")
    e = bt.krum(G, N, fs, return_index=True); te = tables(b"Krum")
    assert same_bits(a, e) and same_bits(ta, te)
    ao, asel = bt.bulyan(G, N, fbs, return_selection=True, rows=rows); ta = tables(b"Bulyan")
    eo, esel = bt.bulyan(G, N, fbs, return_selection=True); te = tables(b"Bulyan")
    assert same_bits(ao, eo) and same_bits(asel, esel) and same_bits(ta, te)
    assert same_bits(bt.trimmed_mean(G, N, fs, rows=rows), bt.trimmed_mean(G, N, fs))
    assert same_bits(bt.no_defense(G, N, fs, rows=rows), bt.no_defense(G, N, fs))


def test_default_format_matches_c_oracle(api):
    bt = api[0]
    from oracle import c_oracle as co
    N, D = 100, 32768 + 64
    rows = [r for r in ROWS if r >= 3]
    G = make(rows, N, D, D, torch.float32, seed=11)
    G = fill_padding(G, rows, "special")
    idx = bt.krum(G, None, [fk(r) for r in rows], return_index=True, rows=rows).cpu().tolist()
    out, sel = bt.bulyan(G, None, [fb(r) for r in rows], return_selection=True, rows=rows)
    tm = bt.trimmed_mean(G, None, [fk(r) for r in rows], rows=rows).cpu().numpy()
    sel, out = sel.cpu().tolist(), out.cpu().numpy()
    for b, r in enumerate(rows):
        Gh = G[b, :r].cpu().numpy()
        table = np.sqrt(co.pairwise_sqdist(Gh))
        want, margin = co.krum_select(table, r, fk(r), with_margin=True)
        assert idx[b] == want or margin <= MARGIN, (b, idx[b], want, margin)
        want_sel, margins = co.bulyan_select(table, r, fb(r), with_margins=True)
        first_close = next((i for i, m in enumerate(margins) if 0.0 < m <= MARGIN), len(margins))
        assert sel[b][:first_close] == want_sel[:first_close], b
        if first_close == len(margins):
            np.testing.assert_allclose(out[b], co.trimmed_mean(Gh, 2 * fb(r), rows=sel[b][:r - 2 * fb(r)]),
                                       rtol=1e-5, atol=1e-6)
        np.testing.assert_allclose(tm[b], co.trimmed_mean(Gh, fk(r)), rtol=1e-5, atol=1e-6)


@pytest.mark.parametrize("dtype", ["float32", "bfloat16"])
def test_metrics_rows(api, splits, dtype):
    bt, Dm, _, _ = api
    N, D = 100, 4096
    rows = ROWS
    G = fill_padding(make(rows, N, D, D, getattr(torch, dtype), seed=5), rows, "special")
    fs = [min(fk(r) + 1, r) for r in rows]                           # rows_b = 1, 2: f_b = rows_b, no honest row
    idx = bt.krum(G, None, [fk(r) for r in rows], return_index=True, rows=rows)
    agg = bt.trimmed_mean(G, None, fs, rows=rows)
    m = bt.attack_metrics(G, fs, krum_index=idx, return_honest_mean=True, rows=rows)
    ma = bt.attack_metrics(G, fs, aggregated=agg, rows=rows)
    for b, r in enumerate(rows):
        Gb = G[b, :r][None]
        if fs[b] >= r:
            assert torch.isnan(m["honest_mean"][b]).all() and torch.isnan(m["rel_deviation"][b]), b
        else:
            assert same_bits(m["honest_mean"][b], Dm.no_defense(G[b, fs[b]:r], r - fs[b], 0)), b
        one = bt.attack_metrics(Gb, [fs[b]], krum_index=idx[b:b + 1], return_honest_mean=True)
        for k in one:
            assert same_bits(m[k][b:b + 1], one[k]), (b, k)
        onea = bt.attack_metrics(Gb, [fs[b]], aggregated=agg[b:b + 1])
        for k in onea:
            assert same_bits(ma[k][b:b + 1], onea[k]), (b, k)
    # Bulyan's selection statistics
    keep = [b for b, r in enumerate(rows) if r >= 3]
    brows = [rows[b] for b in keep]
    _, sel = bt.bulyan(G[keep], None, [fb(r) for r in brows], return_selection=True, rows=brows)
    ms = bt.attack_metrics(G[keep], [fb(r) for r in brows], selection=sel, rows=brows)
    for j, b in enumerate(keep):
        one = bt.attack_metrics(G[b:b + 1, :brows[j]], [fb(brows[j])], selection=sel[j:j + 1])
        assert same_bits(ms["bulyan_malicious_fraction"][j:j + 1], one["bulyan_malicious_fraction"]), b


def test_failed_round_and_single_row(api):
    bt = api[0]
    N, D = 16, 256
    rows = [1, 11, 16]
    G = make(rows, N, D, D, torch.float32, seed=9)
    idx = bt.krum(G, None, 0, return_index=True, rows=rows).cpu().tolist()
    assert idx[0] == -1
    row = bt.krum(G, None, 0, rows=rows)
    assert same_bits(row[0], G[0, 0])
    # a problem whose every distance is NaN: its first Bulyan round finds no eligible user
    Gn = G[1:].clone()
    Gn[0, :11, 0] = float("nan")
    with pytest.raises(KeyError):
        bt.bulyan(Gn, None, [2, 3], rows=[11, 16])
    out = bt.bulyan(G[1:], None, [2, 3], rows=[11, 16])
    assert torch.isfinite(out).all()
    with pytest.raises(TypeError):
        bt.krum(G, None, 0, rows=torch.tensor(rows, device="cuda"))
    with pytest.raises(TypeError):
        bt.attack_metrics(G, torch.tensor([0, 0, 0], device="cuda"), rows=rows)
