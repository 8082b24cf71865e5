"""Batched aggregation with more than 128 clients per problem (batched.py at 128 < N <= 1024, afl_defend_batched_large,
afl_alie_batched_large) on an H100 (-m gpu):
  * problem b's results are the single device call's bit for bit (Krum's index and row, Bulyan's output and selection,
    the trimmed mean, the mean) with per-problem f_b, at N = 129 ... 1000 (2 ... 8 Gram tiles, every trimmed-mean class
    S = 8 ... 32, Bulyan's theta_b crossing classes in one batch), for fp32 on the tensor-core path (multi-tile bf16x2
    with per-problem centres) and on SIMT, and for bf16 and fp16 (split count pinned);
  * ragged N = 1000 batches: padding (NaN, +-inf, +-1e30) never changes a result, problem b equals the single call on
    G[b, :rows_b] wherever both run the same operand format, and Krum's selection matches the C oracle in the default
    format wherever the oracle's top-1 / top-2 margin exceeds 1e-5;
  * the exact-integer trimmed-mean columns in one batch that mixes classes equal ref_numpy bit for bit;
  * ALIE at N = 1000, f = 240 equals the single attack_rows, and Krum on the attacked batch the single call;
  * afl_defend_batched_large at n <= 128 is afl_defend_batched_rows, and the metrics of a large batch are the
    per-problem metrics;
  * a failed Bulyan round raises KeyError(-1) and N = 1025 NotImplementedError.
"""
import ctypes
import os

import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

SPLITS = "2"
MARGIN = 1e-5


@pytest.fixture(scope="module")
def api():
    if not torch.cuda.is_available():
        pytest.skip("no GPU")
    from attacking_federate_learning_b200 import batched, defences, malicious, _native
    _native.lib()
    return batched, defences, malicious, _native


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


def make(B, N, D, ld, dtype, seed=0):
    """[B, N, D] view of a [B, N, ld] buffer: heterogeneous clients around a common component."""
    rng = np.random.default_rng(seed)
    common = 0.1 * rng.standard_normal((B, 1, ld), dtype=np.float32)
    scale = np.exp(0.25 * rng.standard_normal((B, N, 1))).astype(np.float32)
    G = common + scale * rng.standard_normal((B, N, ld), dtype=np.float32)
    return torch.from_numpy(G).cuda().to(dtype)[:, :, :D]


def fill_padding(G, rows):
    """Rows past rows_b of every problem: a mix of NaN, +-inf and +-1e30."""
    G = G.clone()
    pad = torch.tensor([float("nan"), float("inf"), -float("inf"), 1e30, -1e30], device=G.device)
    for b, r in enumerate(rows):
        if r < G.shape[1]:
            k = torch.arange((G.shape[1] - r) * G.shape[2], device=G.device) % 5
            G[b, r:] = pad[k].view(G.shape[1] - r, G.shape[2]).to(G.dtype)
    return G


def fb(r):            # the largest f with r >= 4 f + 3
    return (r - 3) // 4


# per-problem Krum / trimmed-mean counts and Bulyan counts whose theta_b = N - 2 f_b crosses trimmed-mean classes
KF = {129: [0, 30, 64], 256: [1, 61, 127], 300: [72, 10, 149], 640: [153, 0, 300], 1000: [240, 100, 499]}
BF = {129: [31, 0, 20], 256: [63, 20, 0], 300: [74, 30, 5], 640: [159, 60, 0], 1000: [245, 190, 120, 60, 10]}
CASES = [("float32", "tensor"), ("float32", "simt"), ("bfloat16", "tensor"), ("float16", "tensor")]


@pytest.mark.parametrize("dtype,path", CASES, ids=[f"{d}-{p}" for d, p in CASES])
@pytest.mark.parametrize("N", [129, 256, 300, 640, 1000])
def test_large_match_single_calls(api, splits, dtype, path, N):
    bt, Dm, _, _ = api
    kf, bf = KF[N], BF[N]
    D, ld = (4096, 4096) if path == "tensor" else (4099, 4099)
    G = make(max(len(kf), len(bf)), N, D, ld, getattr(torch, dtype), seed=N)
    Gk = G[:len(kf)]
    idx = bt.krum(Gk, N, kf, return_index=True).cpu().tolist()
    krow = bt.krum(Gk, N, kf)
    tm = bt.trimmed_mean(Gk, N, kf)
    mean = bt.no_defense(Gk, N, 0)
    for b, f in enumerate(kf):
        assert idx[b] == Dm.krum(Gk[b], N, f, return_index=True), (b, f)
        assert same_bits(krow[b], Gk[b, idx[b]]), (b, f)
        assert same_bits(tm[b], Dm.trimmed_mean(Gk[b], N, f)), (b, f)
        assert same_bits(mean[b], Dm.no_defense(Gk[b], N, 0)), (b, f)
    Gb = G[:len(bf)]
    out, sel = bt.bulyan(Gb, N, bf, return_selection=True)
    sel = sel.cpu()
    assert sel.shape[1] == N - 2 * min(bf)
    for b, f in enumerate(bf):
        out1, sel1 = Dm.bulyan(Gb[b], N, f, return_selection=True)
        theta = N - 2 * f
        assert same_bits(sel[b, :theta], sel1.cpu()) and bool((sel[b, theta:] == -2).all()), (b, f)
        assert same_bits(out[b], out1), (b, f)


RAGGED = [1, 2, 127, 128, 129, 500, 1000]


@pytest.mark.parametrize("dtype", ["float32", "bfloat16", "float16"])
def test_large_ragged(api, splits, dtype):
    bt, Dm, _, _ = api
    N, D = 1000, 2048
    rows = RAGGED
    G = make(len(rows), N, D, D, getattr(torch, dtype), seed=5)
    Gp = fill_padding(G, rows)
    kf = [int(0.24 * r) for r in rows]
    res = {}
    for name, M in (("clean", G), ("padded", Gp)):
        res[name] = dict(idx=bt.krum(M, None, kf, return_index=True, rows=rows), krow=bt.krum(M, None, kf, rows=rows),
                         tm=bt.trimmed_mean(M, None, kf, rows=rows), mean=bt.no_defense(M, None, 0, rows=rows))
    for k in res["clean"]:
        assert same_bits(res["clean"][k], res["padded"][k]), k
    keep = [b for b, r in enumerate(rows) if r >= 3]
    brows = [rows[b] for b in keep]
    bouts = [bt.bulyan(M[keep], None, [fb(r) for r in brows], return_selection=True, rows=brows) for M in (G, Gp)]
    assert same_bits(bouts[0][0], bouts[1][0]) and same_bits(bouts[0][1], bouts[1][1])
    idx = res["clean"]["idx"].cpu().tolist()
    for b, r in enumerate(rows):
        if dtype == "float32" and r <= 128:           # a single call at rows_b <= 128 runs another operand format
            continue
        Gb = G[b, :r]
        assert idx[b] == Dm.krum(Gb, r, kf[b], return_index=True), (b, r)
        assert same_bits(res["clean"]["krow"][b], Gb[idx[b]] if idx[b] >= 0 else Gb[r - 1]), (b, r)
        assert same_bits(res["clean"]["tm"][b], Dm.trimmed_mean(Gb, r, kf[b])), (b, r)
        assert same_bits(res["clean"]["mean"][b], Dm.no_defense(Gb, r, 0)), (b, r)
    sel = bouts[0][1].cpu()
    for j, b in enumerate(keep):
        r = rows[b]
        if dtype == "float32" and r <= 128:
            continue
        out1, sel1 = Dm.bulyan(G[b, :r], r, fb(r), return_selection=True)
        theta = r - 2 * fb(r)
        assert same_bits(sel[j, :theta], sel1.cpu()) and bool((sel[j, theta:] == -2).all()), (b, r)
        assert same_bits(bouts[0][0][j], out1), (b, r)


def test_large_ragged_oracle(api):
    """Default format (no pinned splits), fp32: Krum's index against the C oracle where its margin exceeds 1e-5."""
    from oracle import c_oracle as co
    bt = api[0]
    N, D = 1000, 1024
    rows = [129, 500, 1000]
    G = fill_padding(make(len(rows), N, D, D, torch.float32, seed=11), rows)
    kf = [int(0.24 * r) for r in rows]
    idx = bt.krum(G, None, kf, return_index=True, rows=rows).cpu().tolist()
    checked = 0
    for b, r in enumerate(rows):
        Gn = G[b, :r].cpu().numpy()
        want, margin = co.krum_select(np.sqrt(co.pairwise_sqdist(Gn)), r, kf[b], with_margin=True)
        if margin > MARGIN:
            assert idx[b] == want, (b, r, margin)
            checked += 1
    assert checked >= 2


def test_large_trimmed_mean_exact_mixed_classes(api):
    """The exact-integer columns of test_gpu_trimmed_mean_exact in one ragged batch whose problems fall in every
    trimmed-mean class: ref_numpy bit for bit."""
    from test_gpu_trimmed_mean_exact import exact_matrix, f_values, ref_tm, assert_same_bits
    bt = api[0]
    rng = np.random.default_rng(33000)
    rows = [100, 129, 256, 300, 500, 640, 700, 896, 1000]
    N = max(rows)
    fs = [f_values(r)[1] for r in rows]
    mats = [exact_matrix(rng, r, "f32", 16, [max(r - f - 1, 0)]) for r, f in zip(rows, fs)]
    d = mats[0].shape[1]
    buf = np.full((len(rows), N, d), np.nan, np.float32)
    for b, M in enumerate(mats):
        buf[b, :rows[b]] = M
    out = bt.trimmed_mean(torch.from_numpy(buf).cuda(), None, fs, rows=rows).cpu().numpy()
    for b, (M, f) in enumerate(zip(mats, fs)):
        assert_same_bits(out[b], ref_tm(M, f), (b, rows[b], f))


def test_large_alie_and_krum_tie_break(api):
    bt, Dm, Mal, _ = api
    N, D, f = 1000, 4096, 240
    G = make(2, N, D, D, torch.float32, seed=13)
    G1 = [G[b].clone() for b in range(2)]
    crafted, mu, sigma = bt.alie_rows(G, f, 1.5)
    for b in range(2):
        c1 = Mal.DriftAttack(1.5).attack_rows(G1[b], f)
        assert same_bits(crafted[b], c1)
        assert same_bits(G[b], G1[b])                   # rows 0..239 written, nothing else
        assert same_bits(G[b, :f], crafted[b].expand(f, D))
    # Krum on the attacked batch: 240 identical rows across two tiles, the [1, 0, 2, ...] tie-break
    idx = bt.krum(G, N, f, return_index=True).cpu().tolist()
    for b in range(2):
        assert idx[b] == Dm.krum(G1[b], N, f, return_index=True)
    # per-problem counts at N > 128 take the large entry too
    Gs = make(2, N, D, D, torch.float32, seed=14)
    Gs1 = [Gs[b].clone() for b in range(2)]
    crafted2, _, _ = bt.alie_rows(Gs, [240, 100], [1.0, 2.0])
    for b, (ff, z) in enumerate(((240, 1.0), (100, 2.0))):
        assert same_bits(crafted2[b], Mal.DriftAttack(z).attack_rows(Gs1[b], ff))
        assert same_bits(Gs[b], Gs1[b])


def test_large_entry_equals_rows_entry_at_one_tile(api, splits):
    bt, _, _, nat = api
    L = nat.lib()
    N, D, B = 100, 4096, 3
    G = make(B, N, D, D, torch.float32, seed=17)
    rows = (ctypes.c_int * B)(100, 60, 9)
    ucs = (ctypes.c_int * B)(100, 60, 9)
    fs = (ctypes.c_int * B)(24, 14, 1)
    for rule in (b"Krum", b"Bulyan", b"TrimmedMean", b"NoDefense"):
        outs = []
        for ws_fn, call in ((L.afl_batched_rows_workspace_bytes, L.afl_defend_batched_rows),
                            (L.afl_batched_large_workspace_bytes, L.afl_defend_batched_large)):
            nbytes = ws_fn(rule, B, N, D, nat.AFL_F32)
            assert nbytes == L.afl_batched_rows_workspace_bytes(rule, B, N, D, nat.AFL_F32)
            ws = torch.empty(nbytes, dtype=torch.uint8, device="cuda")
            out = torch.full((B, D), -7.0, device="cuda")
            idx = torch.full((B,), -7, dtype=torch.int32, device="cuda")
            sel = torch.full((B, 100), -7, dtype=torch.int32, device="cuda")
            nat.check(call(rule, G.data_ptr(), B, N * D, N, D, D, nat.AFL_F32, rows, ucs, fs, out.data_ptr(),
                           idx.data_ptr(), sel.data_ptr(), ws.data_ptr(), nbytes, None))
            torch.cuda.synchronize()
            outs.append((out, idx, sel))
        for a, b in zip(*outs):
            assert same_bits(a, b), rule


def test_large_metrics(api):
    bt = api[0]
    N, D = 600, 2048
    rows, fs = [600, 300, 129], [144, 72, 30]
    G = make(3, N, D, D, torch.float32, seed=19)
    agg = bt.trimmed_mean(G, None, fs, rows=rows)
    idx = bt.krum(G, None, fs, return_index=True, rows=rows)
    met = bt.attack_metrics(G, fs, aggregated=agg, rows=rows, return_honest_mean=True)
    metk = bt.attack_metrics(G, fs, krum_index=idx, rows=rows)
    for b, r in enumerate(rows):
        one = bt.attack_metrics(G[b:b + 1, :r], fs[b], aggregated=agg[b:b + 1], return_honest_mean=True)
        assert same_bits(met["rel_deviation"][b:b + 1], one["rel_deviation"])
        assert same_bits(met["honest_mean"][b:b + 1], one["honest_mean"])
        onek = bt.attack_metrics(G[b:b + 1, :r], fs[b], krum_index=idx[b:b + 1])
        assert same_bits(metk["krum_success"][b:b + 1], onek["krum_success"])
        assert same_bits(metk["rel_deviation"][b:b + 1], onek["rel_deviation"])


def test_large_errors(api):
    bt = api[0]
    N, D = 200, 256
    G = make(2, N, D, D, torch.float32, seed=23)
    Gn = G.clone()
    Gn[1, :, 0] = float("nan")                         # every distance of problem 1 is NaN: its first round fails
    with pytest.raises(KeyError):
        bt.bulyan(Gn, N, [40, 40])
    with pytest.raises(NotImplementedError, match="1024"):
        bt.krum(torch.zeros((1, 1025, 8), device="cuda"), 1025, 10)
    with pytest.raises(NotImplementedError, match="1024"):
        bt.trimmed_mean(torch.zeros((1, 1025, 8), device="cuda"), 1025, 10)
