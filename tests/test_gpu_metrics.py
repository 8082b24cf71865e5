"""Attack-success metrics of a batch (batched.attack_metrics, afl_attack_metrics_batched / _each) on an H100
(-m gpu).  The honest mean must equal afl_mean on rows f_b..n-1 bit for bit; the relative deviation is held to a
float64 NumPy oracle on the upcast matrix; the flags and fractions must equal metrics.krum_attack_success and
metrics.bulyan_attack_success evaluated per problem on the host.  Results must not depend on the pitch, the alignment,
the batch size or the run.
"""
import numpy as np
import pytest

from oracle import ref_numpy as orc

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

DTYPES = [torch.float32, torch.bfloat16, torch.float16]
# name: (problems, clients, params, pitch, take every second problem of a batch twice as long)
LAYOUTS = {
    "c1_padded": (6, 10, 79_510, 79_520, False),
    "c1_packed": (5, 10, 79_510, 79_510, False),        # d % 8 != 0 and a pitch no 16-byte load can use
    "n51_odd_d": (4, 51, 8_195, 8_200, False),
    "n100_packed": (3, 100, 4_099, 4_099, False),
    "n300": (2, 300, 2_048, 2_048, False),              # past the one Gram tile of the defence batches
    "strided": (4, 10, 4_096, 4_096, True),
}


@pytest.fixture(scope="module")
def api():
    if not torch.cuda.is_available():
        pytest.skip("no GPU")
    from attacking_federate_learning_b200 import batched, metrics, _device, _native
    _native.lib()
    return batched, metrics, _device, _native


def same_bits(a, b):
    a, b = a.contiguous(), b.contiguous()
    return a.shape == b.shape and a.dtype == b.dtype and torch.equal(a.view(torch.uint8), b.view(torch.uint8))


def hetero(rng, B, n, d):
    common = 0.1 * rng.standard_normal((B, 1, d), dtype=np.float32)
    scale = np.exp(0.25 * rng.standard_normal((B, n, 1))).astype(np.float32)
    return common + scale * rng.standard_normal((B, n, d), dtype=np.float32)


def make(layout, dtype, seed=0):
    B, n, d, ld, strided = LAYOUTS[layout]
    rng = np.random.default_rng(seed)
    buf = torch.zeros((2 * B if strided else B, n, ld), dtype=dtype, device="cuda")
    G = buf[::2] if strided else buf
    G = G[:, :, :d]
    G.copy_(torch.from_numpy(hetero(rng, B, n, d)).cuda())
    return G


def cycle(B, values):
    return [values[b % len(values)] for b in range(B)]


def oracle_deviation(Gb, f, a):
    """float64 ||a - h|| / ||h|| with h the reference's fp32 mean of the honest rows (defences.py:13-14)."""
    h = orc.no_defense(Gb[f:]).astype(np.float64)
    return np.linalg.norm(a.astype(np.float64) - h) / np.linalg.norm(h)


@pytest.mark.parametrize("dtype", DTYPES, ids=["f32", "bf16", "f16"])
@pytest.mark.parametrize("layout", LAYOUTS)
def test_honest_mean_is_afl_mean_of_the_honest_rows(api, layout, dtype):
    bt, _, dev, _ = api
    G = make(layout, dtype)
    B, n, _ = G.shape
    f = max(1, n // 4)
    got = bt.attack_metrics(G, f, return_honest_mean=True)
    assert set(got) == {"honest_mean"}
    if n - f <= 128:
        assert same_bits(got["honest_mean"], bt.no_defense(G[:, f:], n - f, 0))
    fs = cycle(B, [0, 1, n // 4, n - 1, n // 2])
    each = bt.attack_metrics(G, fs, return_honest_mean=True)["honest_mean"]
    for b in range(B):
        assert same_bits(got["honest_mean"][b], dev.mean(G[b, f:])), b
        assert same_bits(each[b], dev.mean(G[b, fs[b]:])), (b, fs[b])


@pytest.mark.parametrize("dtype", DTYPES, ids=["f32", "bf16", "f16"])
@pytest.mark.parametrize("layout", LAYOUTS)
def test_relative_deviation_matches_float64_oracle(api, layout, dtype):
    bt = api[0]
    G = make(layout, dtype, seed=1)
    B, n, _ = G.shape
    Gh = G.float().cpu().numpy()
    fs = cycle(B, [n // 4, 0, 1, n // 2, n - 1])
    agg = G.float().mean(dim=1) + 0.01                       # any fp32 [B, D] aggregate
    idx = torch.tensor(cycle(B, [n - 1, 0, n // 2]), dtype=torch.int32, device="cuda")
    rows = G[torch.arange(B, device="cuda"), idx.long()].float()
    for f in (fs[0], fs):                                    # one count for the batch, then one per problem
        fb = [f] * B if isinstance(f, int) else f
        by_agg = bt.attack_metrics(G, f, aggregated=agg)
        by_idx = bt.attack_metrics(G, f, krum_index=idx)
        by_rows = bt.attack_metrics(G, f, aggregated=rows)
        assert same_bits(by_idx["rel_deviation"], by_rows["rel_deviation"])
        assert same_bits(by_idx["deviation_sums"], by_rows["deviation_sums"])
        for b in range(B):
            want = oracle_deviation(Gh[b], fb[b], agg[b].cpu().numpy())
            assert abs(float(by_agg["rel_deviation"][b]) - want) <= 1e-6 * want, (b, fb[b])
            want = oracle_deviation(Gh[b], fb[b], Gh[b, int(idx[b])])
            assert abs(float(by_idx["rel_deviation"][b]) - want) <= 1e-6 * want, (b, fb[b])
        s = by_agg["deviation_sums"]
        assert same_bits(by_agg["rel_deviation"], torch.sqrt(s[:, 0] / s[:, 1]).float())


@pytest.mark.parametrize("dtype", DTYPES, ids=["f32", "bf16", "f16"])
def test_bits_do_not_depend_on_run_batch_or_pitch(api, dtype):
    bt = api[0]
    G = make("c1_padded", dtype, seed=2)
    B, n, _ = G.shape
    fs = cycle(B, [1, 2, 0, 3])
    agg = G.float().mean(dim=1)
    idx = torch.tensor(cycle(B, [3, 0, 9]), dtype=torch.int32, device="cuda")
    keys = ("rel_deviation", "deviation_sums", "honest_mean")
    for kw in ({"aggregated": agg}, {"krum_index": idx}):
        one = bt.attack_metrics(G, fs, return_honest_mean=True, **kw)
        two = bt.attack_metrics(G, fs, return_honest_mean=True, **kw)
        packed = bt.attack_metrics(G.contiguous(), fs, return_honest_mean=True, **kw)    # pitch 79,510: scalar loads
        for k in keys:
            assert same_bits(one[k], two[k]), k
            assert same_bits(one[k], packed[k]), k
        for b in range(B):
            sub = {k: v[b:b + 1] for k, v in kw.items()}
            alone = bt.attack_metrics(G[b:b + 1], fs[b], return_honest_mean=True, **sub)
            for k in keys:
                assert same_bits(one[k][b:b + 1], alone[k]), (k, b)


def test_edge_problems(api):
    bt = api[0]
    n, d = 10, 3_000
    rng = np.random.default_rng(3)
    fs = [0, n, n + 5, 2, 2, 2, 3]
    B = len(fs)
    Gh = hetero(rng, B, n, d)
    Gh[4, 2:] = 0.0                                  # problem 4: an all-zero honest mean
    Gh[4, 2:, 7] = [1.0, -1.0] + [0.0] * (n - 4)
    Gh[5, 6, 11] = np.inf                            # problem 5: an inf in an honest row
    Gh[6, 1, 11] = np.inf                            # problem 6: an inf in a malicious row only
    G = torch.from_numpy(Gh).cuda()
    idx = torch.tensor([3, 3, 3, -1, 0, 0, 5], dtype=torch.int32, device="cuda")
    got = bt.attack_metrics(G, fs, krum_index=idx, return_honest_mean=True)
    torch.cuda.synchronize()                         # f_b >= n and idx = -1 read no row: nothing faults
    rel, h = got["rel_deviation"].cpu().numpy(), got["honest_mean"].cpu().numpy()
    np.testing.assert_array_equal(h[0], orc.no_defense(Gh[0]))                  # f = 0: every row is honest
    want = oracle_deviation(Gh[0], 0, Gh[0, 3])
    assert abs(rel[0] - want) <= 1e-6 * want
    assert np.isnan(rel[1]) and np.isnan(h[1]).all()                            # f = n: no honest row
    assert np.isnan(rel[2]) and np.isnan(h[2]).all()                            # f > n
    assert np.isnan(rel[3]) and np.isfinite(h[3]).all()                         # Krum found no eligible user
    assert np.isnan(got["deviation_sums"].cpu().numpy()[3, 0])
    assert (h[4] == 0).all() and np.isposinf(rel[4])                            # x / 0, as NumPy divides
    with np.errstate(invalid="ignore"):
        assert np.isnan(oracle_deviation(Gh[5], 2, Gh[5, 0])) and np.isnan(rel[5])   # inf / inf
    want = oracle_deviation(Gh[6], 3, Gh[6, 5])
    assert abs(rel[6] - want) <= 1e-6 * want
    assert got["krum_success"].cpu().tolist() == [False, True, True, False, True, True, False]
    zero = bt.attack_metrics(G[4:5], 2, aggregated=torch.zeros((1, d), device="cuda"))["rel_deviation"]
    assert torch.isnan(zero).all()                                              # 0 / 0


def test_bulyan_selection_rows(api):
    bt, metrics, _, _ = api
    G = torch.zeros((5, 12, 64), device="cuda")
    fs = [2, 2, 0, 3, 12]
    sel = torch.tensor([[5, 1, 0, 7, 11, 3],          # two malicious of six
                        [4, 1, 9, -1, -1, -1],        # a failed round: the -1 tail is not counted
                        [4, 1, 9, 0, -2, -2],         # f = 0: nobody is malicious; -2 = no such round
                        [-2, -2, -2, -2, -2, -2],     # nothing selected: 0 / max(1, 0)
                        [4, 1, 9, 0, 11, 2]],         # f = n: everybody is
                       dtype=torch.int32, device="cuda")
    got = bt.attack_metrics(G, fs, selection=sel)
    assert set(got) == {"bulyan_malicious_fraction"}
    frac = got["bulyan_malicious_fraction"]
    assert frac.dtype == torch.float32
    want = [2 / 6, 1 / 3, 0.0, 0.0, 1.0]
    assert frac.cpu().tolist() == [float(np.float32(w)) for w in want]
    for b in (0, 2, 4):                               # rows without failed rounds: the host bookkeeping's figure
        run = [i for i in sel[b].cpu().tolist() if i != -2]
        assert float(frac[b]) == float(np.float32(metrics.bulyan_attack_success(run, fs[b])))
    # a column slice of a wider selection tensor
    wide = torch.full((5, 9), 7, dtype=torch.int32, device="cuda")
    wide[:, :6] = sel
    assert same_bits(bt.attack_metrics(G, fs, selection=wide[:, :6])["bulyan_malicious_fraction"], frac)


def test_selection_statistics_need_no_workspace(api):
    _, _, _, nat = api
    L = nat.lib()
    G = torch.zeros((3, 10, 64), device="cuda")
    idx = torch.tensor([1, 2, -1], dtype=torch.int32, device="cuda")
    hit = torch.empty(3, dtype=torch.int32, device="cuda")
    nat.check(L.afl_attack_metrics_batched(G.data_ptr(), 3, 640, 10, 64, 64, nat.AFL_F32, 2, None, idx.data_ptr(), None, 0,
                                           None, None, None, hit.data_ptr(), None, None, None, 0,
                                           torch.cuda.current_stream().cuda_stream))
    assert hit.cpu().tolist() == [1, 0, 0]


def test_sweep_end_to_end_at_c1(api):
    """alie_rows -> rule -> attack_metrics with one (f_b, z_b) per problem against the per-problem host bookkeeping."""
    bt, metrics, dev, _ = api
    n, d, S = 10, 79_510, 2
    zs = [0.25, 0.5, 1.0, 1.5, 2.0, 3.0]
    rng = np.random.default_rng(4)
    for rule, f_values in (("Krum", (1, 2)), ("Bulyan", (0, 1))):
        f = np.repeat([fv for _ in zs for fv in f_values], S).astype(np.int32)
        z = np.repeat([zv for zv in zs for _ in f_values], S)
        B = len(f)
        buf = torch.from_numpy(hetero(rng, B, n, 79_520)).cuda()
        G = buf[:, :, :d]
        bt.alie_rows(G, f, z)
        if rule == "Krum":
            idx = bt.krum(G, n, f, return_index=True)
            got = bt.attack_metrics(G, f, krum_index=idx)
            idx_h = idx.cpu().tolist()
        else:
            agg, sel = bt.bulyan(G, n, f, return_selection=True)
            got = bt.attack_metrics(G, f, aggregated=agg, selection=sel)
            sel_h = sel.cpu().tolist()
        for b in range(B):
            fb = int(f[b])
            honest = dev.mean(G[b, fb:])
            if rule == "Krum":
                assert bool(got["krum_success"][b]) == metrics.krum_attack_success(idx_h[b], fb), b
                want = metrics.relative_deviation(G[b, idx_h[b]], honest)
            else:
                run = sel_h[b][:n - 2 * fb]
                assert sel_h[b][n - 2 * fb:] == [-2] * (2 * fb - 2 * int(f.min())), b
                assert float(got["bulyan_malicious_fraction"][b]) == \
                    float(np.float32(metrics.bulyan_attack_success(run, fb))), b
                want = metrics.relative_deviation(agg[b], honest)
            assert abs(float(got["rel_deviation"][b]) - want) <= 1e-5 * want, (b, want)


def test_arguments_are_refused(api):
    bt = api[0]
    G = torch.zeros((2, 10, 64), device="cuda")
    agg = torch.zeros((2, 64), device="cuda")
    idx = torch.zeros(2, dtype=torch.int32, device="cuda")
    with pytest.raises(TypeError):
        bt.attack_metrics(G, torch.tensor([1, 2], device="cuda"), aggregated=agg)
    with pytest.raises(ValueError):
        bt.attack_metrics(G, [1, 2, 3], aggregated=agg)
    with pytest.raises(ValueError, match="not both"):
        bt.attack_metrics(G, 2, aggregated=agg, krum_index=idx)
    with pytest.raises(ValueError):
        bt.attack_metrics(G, 2, aggregated=agg[:, :32])
    with pytest.raises(ValueError):
        bt.attack_metrics(G, 2, krum_index=idx.long())
    with pytest.raises(ValueError):
        bt.attack_metrics(G, -1, aggregated=agg)
    assert bt.attack_metrics(G, 2) == {}
