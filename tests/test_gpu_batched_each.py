"""Per-problem batched aggregation (batched.py with one corrupted_count / num_std per problem,
afl_defend_batched_each, afl_alie_batched_each) on an H100 (-m gpu).  Problem b's result must be, bit for bit,
the single device call's on G[b] with its own f_b (and z_b): Krum's index, Bulyan's selection (then -2 padding)
and output, the trimmed mean, the mean and ALIE's statistics and written rows.  A uniform count vector must give
what the scalar batched call gives, and the distance tables must equal the scalar call's (split count pinned).
Selections are also held to the C oracle wherever its top-1 / top-2 margin exceeds 1e-5.
"""
import os

import numpy as np
import pytest

from test_gpu_batched import MARGIN, SHAPES, SPLITS, hetero, make, same_bits

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def api():
    if not torch.cuda.is_available():
        pytest.skip("no GPU")
    from attacking_federate_learning_b200 import batched, defences, malicious, _device, _native
    _native.lib()
    return batched, defences, malicious, _device, _native


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


def cycle(B, hi):
    """f_b = b mod (hi + 1): every valid value 0..hi, one per problem in turn."""
    return [b % (hi + 1) for b in range(B)]


def tables_at(api, G, rule, each):
    """The float64 d2 tables the last batched Krum / Bulyan call left in its workspace (after the parameter table)."""
    _, _, _, dev, nat = api
    B, n, D = G.shape
    L = nat.lib()
    code = nat.AFL_F32 if G.dtype == torch.float32 else nat.AFL_BF16
    off = 0
    if each:
        off = L.afl_batched_each_workspace_bytes(rule, B, n, D, code) - L.afl_batched_workspace_bytes(rule, B, n, D, code)
    ws = dev.Workspace.get(G.device, "batched", 0)
    return ws[off:off + B * n * n * 8].view(torch.float64).view(B, n, n).clone()


@pytest.mark.parametrize("shape_id", SHAPES)
def test_each_matches_single_calls(api, splits, shape_id):
    bt, D, _, dev, _ = api
    G, _, _ = make(shape_id)
    B, n, _ = G.shape
    fk, fb, ft = cycle(B, (n - 1) // 2), cycle(B, (n - 3) // 4), cycle(B, n + 1)   # Krum, Bulyan, trimmed mean (past n: slices)
    splits(SPLITS)
    idx = bt.krum(G, n, np.array(fk), return_index=True)
    tables = tables_at(api, G, b"Krum", True)
    bt.krum(G, n, fk[0], return_index=True)
    assert same_bits(tables, tables_at(api, G, b"Krum", False))
    out, sel = bt.bulyan(G, n, fb, return_selection=True)
    assert same_bits(tables_at(api, G, b"Bulyan", True), tables)
    tm, mean = bt.trimmed_mean(G, n, tuple(ft)), bt.no_defense(G, n, torch.tensor(ft))
    theta_max = n - 2 * min(fb)
    assert sel.shape == (B, theta_max)
    idx_h, sel_h = idx.cpu().tolist(), sel.cpu()
    for b in range(B):
        assert idx_h[b] == D.krum(G[b], n, fk[b], return_index=True), b
        theta = n - 2 * fb[b]
        out1, sel1 = D.bulyan(G[b], n, fb[b], return_selection=True)
        assert same_bits(sel_h[b, :theta], sel1.cpu()) and same_bits(out[b], out1), b
        assert (sel_h[b, theta:] == -2).all(), b
        assert same_bits(tm[b], D.trimmed_mean(G[b], n, ft[b])), b
        assert same_bits(mean[b], D.no_defense(G[b], n, ft[b])), b
    rows = bt.krum(G, n, fk)
    assert same_bits(rows, G[torch.arange(B, device=G.device), idx.long()])


@pytest.mark.parametrize("shape_id", SHAPES)
def test_uniform_counts_equal_scalar_call(api, shape_id):
    bt = api[0]
    G, f, fb = make(shape_id)
    B, n, _ = G.shape
    assert same_bits(bt.krum(G, n, [f] * B, return_index=True), bt.krum(G, n, f, return_index=True))
    o1, s1 = bt.bulyan(G, n, np.full(B, fb), return_selection=True)
    o0, s0 = bt.bulyan(G, n, fb, return_selection=True)
    assert same_bits(o1, o0) and same_bits(s1, s0)
    assert same_bits(bt.trimmed_mean(G, n, [f] * B), bt.trimmed_mean(G, n, f))
    assert same_bits(bt.no_defense(G, n, [f] * B), bt.no_defense(G, n, f))
    Ga, Gb = G.clone(), G.clone()
    each, scalar = bt.alie_rows(Ga, [f] * B, [1.5] * B), bt.alie_rows(Gb, f, 1.5)
    assert all(same_bits(x, y) for x, y in zip(each, scalar)) and same_bits(Ga, Gb)


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_alie_each_matches_attack_rows(api, dtype):
    bt, _, M, dev, _ = api
    rng = np.random.default_rng(5)
    fs = [0, 1, 2, 10, 3, 0, 5, 10, 4]
    zs = [1.5, 0.0, 0.5, 2.0, 0.0, 0.0, 3.0, 0.25, -1.0]
    B, n, d = len(fs), 10, 4_099                                   # d not a multiple of 4: the scalar column path too
    G = torch.from_numpy(hetero(rng, B, n, d)).cuda().to(dtype)
    Gb = G.clone()
    crafted, mu, sigma = bt.alie_rows(Gb, fs, np.array(zs))
    for b in range(B):
        f, z = fs[b], zs[b]
        if f == 0:
            assert torch.isnan(mu[b]).all() and torch.isnan(sigma[b]).all() and torch.isnan(crafted[b]).all(), b
            assert same_bits(Gb[b], G[b]), b
            continue
        c1, mu1, sigma1 = dev.alie(G[b, :f], z, None, alias_mean=False)
        assert same_bits(mu[b], mu1) and same_bits(sigma[b], sigma1) and same_bits(crafted[b], c1), b
        one = G[b].clone()
        got = M.DriftAttack(z).attack_rows(one, f)
        if z == 0:
            assert got is None and same_bits(crafted[b], mu[b]), b
        else:
            assert same_bits(crafted[b], got), b
        assert same_bits(Gb[b], one), b
        if z == 0:
            assert same_bits(Gb[b], G[b]), b


def test_alie_each_then_krum_selects_user_1(api):
    """Per problem, rows 0..f_b-1 start tiny and become one crafted vector: Krum's tie goes to user 1 for f_b >= 2."""
    bt, D = api[0], api[1]
    rng = np.random.default_rng(11)
    fs = [19, 2, 1, 0, 10, 19]
    B, n, d = len(fs), 80, 40_960
    G = 5.0 * hetero(rng, B, n, d)
    for b, f in enumerate(fs):
        G[b, :f] = 0.002 * G[b, f]
    for dtype in (torch.float32, torch.bfloat16):
        Gd = torch.from_numpy(G).cuda().to(dtype)
        bt.alie_rows(Gd, fs, 1.5)
        idx = bt.krum(Gd, n, fs, return_index=True).cpu().tolist()
        for b, f in enumerate(fs):
            assert all(torch.equal(Gd[b, i], Gd[b, 0]) for i in range(1, f)), b
            assert idx[b] == (1 if f >= 2 else D.krum(Gd[b], n, f, return_index=True)), (b, idx[b])


def test_failed_bulyan_round_in_one_problem(api):
    bt, D, _, dev, _ = api
    B, n, d = 3, 40, 1000
    fs = [9, 5, 2]                                            # theta_max = 36; problem 1 has 30 rounds
    rng = np.random.default_rng(3)
    G = hetero(rng, B, n, d)
    G[1] = 0.0
    G[1, np.arange(n), np.arange(n)] = 1e30                   # problem 1: no eligible user from some round on
    Gd = torch.from_numpy(G).cuda()
    with pytest.raises(KeyError) as e:
        bt.bulyan(Gd, n, fs, return_selection=True)
    assert e.value.args == (-1,)
    # through the C ABI: problem 1's row holds -1 from the failed round on, then -2; the others equal their single calls
    _, _, _, _, nat = api
    L = nat.lib()
    theta_max = n - 2 * min(fs)
    out = torch.empty((B, d), dtype=torch.float32, device="cuda")
    sel = torch.empty((B, theta_max), dtype=torch.int32, device="cuda")
    ws = dev.Workspace.get(Gd.device, "batched", L.afl_batched_each_workspace_bytes(b"Bulyan", B, n, d, nat.AFL_F32))
    c_fs = np.array(fs, np.int32)
    nat.check(L.afl_defend_batched_each(b"Bulyan", Gd.data_ptr(), B, n * d, n, d, d, nat.AFL_F32, n, c_fs.ctypes.data,
                                        out.data_ptr(), None, sel.data_ptr(), ws.data_ptr(), ws.numel(),
                                        torch.cuda.current_stream().cuda_stream))
    theta1 = n - 2 * fs[1]
    want = dev.bulyan_select(dev.sqdist_to_dist(dev.sqdist_partial(Gd[1])), n, fs[1]).cpu()
    assert int(want[-1]) < 0
    row = sel[1].cpu()
    assert same_bits(row[:theta1], want)
    first_bad = int((want < 0).int().argmax())
    assert (row[first_bad:theta1] == -1).all() and (row[theta1:] == -2).all()
    for b in (0, 2):
        out1, sel1 = D.bulyan(Gd[b], n, fs[b], return_selection=True)
        theta = n - 2 * fs[b]
        assert same_bits(sel[b, :theta].cpu(), sel1.cpu()) and same_bits(out[b], out1), b
        assert (sel[b, theta:] == -2).all(), b


def test_counts_on_the_device_are_refused(api):
    bt = api[0]
    G = torch.zeros((2, 10, 64), device="cuda")
    with pytest.raises(TypeError):
        bt.krum(G, 10, torch.tensor([1, 2], device="cuda"))
    with pytest.raises(TypeError):
        bt.alie_rows(G, [1, 2], torch.tensor([0.5, 1.0], device="cuda"))
    with pytest.raises(ValueError):
        bt.trimmed_mean(G, 10, [1, 2, 3])
    with pytest.raises(AssertionError, match="problem 1"):
        bt.bulyan(G, 10, [1, 2])


@pytest.mark.parametrize("shape_id", SHAPES)
def test_each_selections_match_c_oracle(api, shape_id):
    bt = api[0]
    from oracle import c_oracle as co
    G, _, _ = make(shape_id)
    B, n, _ = G.shape
    fk, fb = cycle(B, (n - 1) // 2), cycle(B, (n - 3) // 4)
    idx = bt.krum(G, n, fk, return_index=True).cpu().tolist()
    _, sel = bt.bulyan(G, n, fb, return_selection=True)
    sel = sel.cpu().tolist()
    for b in range(min(B, 3)):
        Gh = G[b].float().cpu().numpy()
        table = np.sqrt(co.pairwise_sqdist(Gh))
        want, margin = co.krum_select(table, n, fk[b], with_margin=True)
        assert idx[b] == want or margin <= MARGIN, (b, idx[b], want, margin)
        want_sel, margins = co.bulyan_select(table, n, fb[b], with_margins=True)
        first_close = next((i for i, m in enumerate(margins) if 0.0 < m <= MARGIN), len(margins))
        assert sel[b][:first_close] == want_sel[:first_close], b
