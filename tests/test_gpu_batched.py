"""Batched aggregation (attacking_federate_learning_b200/batched.py, afl_defend_batched, afl_alie_batched) on an
H100 (-m gpu).  Every problem of a batch must give, bit for bit, what the existing single device call gives on that
problem: the distance table, the Krum index, Bulyan's selection and output, the trimmed mean, the mean and the ALIE
statistics.  The Gram kernels choose their split count for the whole batch, so the table comparisons pin it with
AFL_GRAM_SPLITS for both arms; the column rules are compared with no override as well.  Selections are also held
to the C oracle wherever its top-1 / top-2 margin exceeds 1e-5.
"""
import os

import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

MARGIN = 1e-5
SPLITS = "3"


@pytest.fixture(scope="module")
def api():
    if not torch.cuda.is_available():
        pytest.skip("no GPU")
    from attacking_federate_learning_b200 import batched, defences, malicious, _device, _native
    _native.lib()
    return batched, defences, malicious, _device, _native


@pytest.fixture
def splits():
    """Setter for AFL_GRAM_SPLITS (None = unset); restored when the test ends."""
    saved = os.environ.get("AFL_GRAM_SPLITS")

    def set_splits(v):
        if v is None:
            os.environ.pop("AFL_GRAM_SPLITS", None)
        else:
            os.environ["AFL_GRAM_SPLITS"] = v
    yield set_splits
    set_splits(saved)


def hetero(rng, B, n, d):
    common = 0.1 * rng.standard_normal((B, 1, d), dtype=np.float32)
    scale = np.exp(0.25 * rng.standard_normal((B, n, 1))).astype(np.float32)
    return common + scale * rng.standard_normal((B, n, d), dtype=np.float32)


def make(shape_id):
    """(G [B, n, D] on the GPU, f for Krum / trimmed mean / ALIE, f for Bulyan)."""
    rng = np.random.default_rng(SHAPES.index(shape_id))
    if shape_id == "tf32_padded":                # 7 x 10 x 79,510, ld 79,520: split TF32
        buf = torch.from_numpy(hetero(rng, 7, 10, 79_520)).cuda()
        return buf[:, :, :79_510], 2, 1
    if shape_id == "simt_unpadded":              # 5 x 10 x 79,510: misaligned pitch, SIMT
        return torch.from_numpy(hetero(rng, 5, 10, 79_510)).cuda(), 2, 1
    if shape_id == "sym_box56":                  # 4 x 51 x 40,960: symmetric bf16x2, box 56
        return torch.from_numpy(hetero(rng, 4, 51, 40_960)).cuda(), 12, 12
    if shape_id == "sym_box104":                 # 3 x 100 x 40,960: box 104
        return torch.from_numpy(hetero(rng, 3, 100, 40_960)).cuda(), 24, 24
    if shape_id == "tf32_box128":                # 3 x 128 x 8,192: split TF32, box 128
        return torch.from_numpy(hetero(rng, 3, 128, 8_192)).cuda(), 31, 31
    if shape_id == "bf16_clients":               # 4 x 51 x 8,192 bf16
        return torch.from_numpy(hetero(rng, 4, 51, 8_192)).cuda().bfloat16(), 12, 12
    if shape_id == "batch_of_one":
        buf = torch.from_numpy(hetero(rng, 1, 10, 79_520)).cuda()
        return buf[:, :, :79_510], 2, 1
    if shape_id == "large_grid":                 # 1,024 x 10 x 4,096: per-problem counters
        return torch.from_numpy(hetero(rng, 1024, 10, 4_096)).cuda(), 2, 1
    if shape_id == "strided_batch":              # big[::2]: batch stride of two problems
        big = torch.from_numpy(hetero(rng, 8, 10, 4_096)).cuda()
        return big[::2], 2, 1
    raise KeyError(shape_id)


SHAPES = ["tf32_padded", "simt_unpadded", "sym_box56", "sym_box104", "tf32_box128", "bf16_clients", "batch_of_one",
          "large_grid", "strided_batch"]


def same_bits(a, b):
    a, b = a.contiguous(), b.contiguous()
    return a.shape == b.shape and a.dtype == b.dtype and torch.equal(a.view(torch.uint8), b.view(torch.uint8))


def batch_tables(api, G):
    """The n x n float64 tables the last batched Krum / Bulyan call left at the start of its workspace."""
    _, _, _, dev, _ = api
    B, n, _ = G.shape
    ws = dev.Workspace.get(G.device, "batched", 0)
    return ws[:B * n * n * 8].view(torch.float64).view(B, n, n).clone()


def check_column_rules(api, G, f):
    bt, D, M, dev, _ = api
    B, n, _ = G.shape
    tm, mean = bt.trimmed_mean(G, n, f), bt.no_defense(G, n, f)
    for b in range(B):
        assert same_bits(tm[b], D.trimmed_mean(G[b], n, f)), b
        assert same_bits(mean[b], D.no_defense(G[b], n, f)), b
    # ALIE on rows 0..f-1 of every problem, written back in place, against the single call on a copy of each problem
    Gb = torch.empty_strided(G.shape, G.stride(), dtype=G.dtype, device=G.device).copy_(G)   # same batch stride
    crafted, mu, sigma = bt.alie_rows(Gb, f, 1.5)
    for b in range(B):
        _, mu1, sigma1 = dev.alie(G[b, :f], 1.5, None, alias_mean=False)
        one = G[b].clone()
        crafted1 = M.DriftAttack(1.5).attack_rows(one, f)
        assert same_bits(mu[b], mu1) and same_bits(sigma[b], sigma1) and same_bits(crafted[b], crafted1), b
        assert same_bits(Gb[b], one), b


@pytest.mark.parametrize("shape_id", SHAPES)
def test_batch_matches_single_calls(api, splits, shape_id):
    bt, D, M, dev, _ = api
    G, f, fb = make(shape_id)
    B, n, _ = G.shape
    splits(SPLITS)
    idx = bt.krum(G, n, f, return_index=True)
    tables = batch_tables(api, G)
    rows = bt.krum(G, n, f)
    out, sel = bt.bulyan(G, n, fb, return_selection=True)
    idx_h, sel_h = idx.cpu().tolist(), sel.cpu()
    for b in range(B):
        assert same_bits(tables[b], dev.sqdist_partial(G[b])), b
        assert idx_h[b] == D.krum(G[b], n, f, return_index=True), b
        assert same_bits(rows[b], G[b, idx_h[b]])
        out1, sel1 = D.bulyan(G[b], n, fb, return_selection=True)
        assert same_bits(sel_h[b], sel1.cpu()) and same_bits(out[b], out1), b
    check_column_rules(api, G, f)
    assert set(bt.defend) == {"Krum", "Bulyan", "TrimmedMean", "NoDefense"}


@pytest.mark.parametrize("shape_id", SHAPES)
def test_column_rules_without_split_override(api, splits, shape_id):
    G, f, _ = make(shape_id)
    splits(None)
    check_column_rules(api, G, f)


@pytest.mark.parametrize("shape_id", SHAPES)
def test_selections_match_c_oracle(api, shape_id):
    bt = api[0]
    from oracle import c_oracle as co
    G, f, fb = make(shape_id)
    B, n, _ = G.shape
    idx = bt.krum(G, n, f, return_index=True).cpu().tolist()
    _, sel = bt.bulyan(G, n, fb, return_selection=True)
    sel = sel.cpu().tolist()
    for b in range(min(B, 3)):
        Gh = G[b].float().cpu().numpy()
        table = np.sqrt(co.pairwise_sqdist(Gh))
        want, margin = co.krum_select(table, n, f, with_margin=True)
        assert idx[b] == want or margin <= MARGIN, (b, idx[b], want, margin)
        want_sel, margins = co.bulyan_select(table, n, fb, with_margins=True)
        first_close = next((i for i, m in enumerate(margins) if 0.0 < m <= MARGIN), len(margins))
        assert sel[b][:first_close] == want_sel[:first_close], b


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_alie_rows_select_user_1(api, dtype):
    """ALIE makes rows 0..f-1 of every problem one vector; exact ties go to user 1 ([1, 0, 2, ...])."""
    bt = api[0]
    rng = np.random.default_rng(11)
    B, n, d, f = 6, 80, 40_960, 19
    G = 5.0 * hetero(rng, B, n, d)
    G[:, :f] = 0.002 * G[:, f:f + 1]
    Gd = torch.from_numpy(G).cuda().to(dtype)
    bt.alie_rows(Gd, f, 1.5)
    assert all(torch.equal(Gd[:, i], Gd[:, 0]) for i in range(1, f))
    assert bt.krum(Gd, n, f, return_index=True).cpu().tolist() == [1] * B


def test_failed_bulyan_round_in_one_problem(api):
    bt, D, _, dev, nat = api
    B, n, d, f = 3, 40, 1000, 9
    rng = np.random.default_rng(3)
    G = hetero(rng, B, n, d)
    G[1] = 0.0
    G[1, np.arange(n), np.arange(n)] = 1e30                   # problem 1: no eligible user from some round on
    Gd = torch.from_numpy(G).cuda()
    with pytest.raises(KeyError) as e:
        bt.bulyan(Gd, n, f, return_selection=True)
    assert e.value.args == (-1,)
    # through the C ABI: problem 1's row holds -1 from the failed round on, the others equal their single calls
    theta = n - 2 * f
    out = torch.empty((B, d), dtype=torch.float32, device="cuda")
    sel = torch.empty((B, theta), dtype=torch.int32, device="cuda")
    L = nat.lib()
    ws = dev.Workspace.get(Gd.device, "batched", L.afl_batched_workspace_bytes(b"Bulyan", B, n, d, nat.AFL_F32))
    nat.check(L.afl_defend_batched(b"Bulyan", Gd.data_ptr(), B, n * d, n, d, d, nat.AFL_F32, n, f, out.data_ptr(), None,
                                   sel.data_ptr(), ws.data_ptr(), ws.numel(), torch.cuda.current_stream().cuda_stream))
    want = dev.bulyan_select(dev.sqdist_to_dist(dev.sqdist_partial(Gd[1])), n, f).cpu()
    assert int(want[-1]) < 0
    assert same_bits(sel[1].cpu(), want)
    first_bad = int((want < 0).int().argmax())
    assert (sel[1, first_bad:] == -1).all()
    for b in (0, 2):
        out1, sel1 = D.bulyan(Gd[b], n, f, return_selection=True)
        assert same_bits(sel[b].cpu(), sel1.cpu()) and same_bits(out[b], out1), b
