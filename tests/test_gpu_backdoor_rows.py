"""The backdoor attack on device-resident client matrices (-m gpu): BackdoorAttack.attack_rows and
batched.backdoor_rows (C ABI afl_backdoor_start_batched / afl_backdoor_finish_batched).

attack_rows must give, bit for bit, what BackdoorAttack.attack gives on the same rows (the statistics kernel, then
torch's element-wise fp32 arithmetic and afl_alie_band), and the golden fixtures minted from the reference's
backdoor.py must hold against the NumPy oracle evaluated on the device's own statistics.  Problem b of a batch must
be the single call on G[b] with its own f_b, z_b, lr_b and w_b; f_b = 0 and z_b = 0 problems are left alone and never
reach the training.  The training stand-in is the golden one, p * 0.9 + 0.01.
"""
import os

import numpy as np
import pytest

from oracle import ref_numpy as orc
from test_gpu_batched import SPLITS, same_bits

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

DTYPES = {"f32": torch.float32, "bf16": torch.bfloat16, "f16": torch.float16}


@pytest.fixture(scope="module")
def api():
    if not torch.cuda.is_available():
        pytest.skip("no GPU")
    from attacking_federate_learning_b200 import batched, defences, malicious, _native
    _native.lib()
    return malicious, batched, defences


def fake(p):                                   # make_golden_backdoor.py's stand-in for backdoor.py:108
    if isinstance(p, torch.Tensor):
        return p * 0.9 + 0.01
    return (p * np.float32(0.9) + np.float32(0.01)).astype(np.float32)


class User:
    def __init__(self, g, w, lr):
        self.grads, self.original_params, self.learning_rate = g, w, lr


def matrix(rng, n, d, ld, dtype, specials=True):
    """[n, d] client rows in an [n, ld] buffer whose padding holds 7.0; NaN and +-inf entries when asked."""
    X = (rng.standard_normal((n, d)) * np.exp(0.25 * rng.standard_normal((n, 1)))).astype(np.float32)
    if specials:
        X[0, 1] = np.nan
        X[n - 1, 2] = np.inf
        X[0, 3] = -np.inf
        X[:, 5] = np.float32(3e4)                # a constant column: sigma = 0
    buf = torch.full((n, ld), 7.0, dtype=dtype, device="cuda")
    buf[:, :d] = torch.from_numpy(X).cuda().to(dtype)
    return buf, buf[:, :d]


def vec(rng, d):
    return torch.from_numpy(rng.standard_normal(d).astype(np.float32)).cuda()


# ------------------------------------------------------------------ 1. attack_rows == attack, bit for bit
@pytest.mark.parametrize("dt", list(DTYPES))
@pytest.mark.parametrize("d", [8, 257, 1000, 4099])
def test_attack_rows_matches_attack(api, dt, d):
    M, *_ = api
    dtype = DTYPES[dt]
    rng = np.random.default_rng(d)
    for f in (1, 2, 5, 24):
        n = f + 3
        for z in (0.0, 0.25, 1.5, -1.0):
            for lr in (0.1, 1e-3, 0.0):
                case = (f, z, lr)
                buf, G = matrix(rng, n, d, d + 5, dtype)
                w = vec(rng, d)
                before = buf.clone()
                users = [User(G[i].clone(), w, lr) for i in range(f)]
                ref = M.BackdoorAttack(z, fake)
                ref.attack(users)
                att = M.BackdoorAttack(z, fake)
                got = att.attack_rows(G, f, w, lr)
                assert same_bits(att.grads_mean, ref.grads_mean) and same_bits(att.grads_stdev, ref.grads_stdev), case
                assert same_bits(buf[f:], before[f:]) and same_bits(buf[:, d:], before[:, d:]), case
                if z == 0:
                    assert got is None and same_bits(buf, before), case
                    continue
                assert same_bits(got, users[0].grads), case
                assert same_bits(G[:f], got.to(dtype).expand(f, d)), case


# ------------------------------------------------------------------ 2. the reference's fixtures
@pytest.mark.parametrize("nm", ["f5_d300", "f24_d2051"])
def test_golden_backdoor_attack_rows(api, golden_backdoor, nm):
    M, *_ = api
    g = golden_backdoor
    z, lr = float(g[f"attack_{nm}/z"]), float(g[f"attack_{nm}/lr"])
    rows, params = g[f"attack_{nm}/rows"], g[f"attack_{nm}/params"]
    f, d = rows.shape
    for ld in (d, d + 3):
        buf = torch.zeros((f, ld), dtype=torch.float32)
        buf[:, :d] = torch.from_numpy(rows)
        G = buf.cuda()[:, :d]
        att = M.BackdoorAttack(z, fake)
        got = att.attack_rows(G, f, torch.from_numpy(params).cuda(), lr).cpu().numpy()
        mu, sigma = att.grads_mean.cpu().numpy(), att.grads_stdev.cpu().numpy()
        np.testing.assert_allclose(sigma, g[f"attack_{nm}/stdev"], rtol=1e-5, atol=1e-7)
        np.testing.assert_allclose(mu, g[f"attack_{nm}/mean"], rtol=1e-5, atol=1e-6)
        want = orc.backdoor_attack_grads(mu.copy(), sigma.copy(), params, lr, z, fake)
        assert np.array_equal(got.view(np.uint32), want.view(np.uint32))
        assert np.array_equal(G.cpu().numpy().view(np.uint32), np.broadcast_to(want, (f, d)).view(np.uint32))
        np.testing.assert_allclose(got, g[f"attack_{nm}/grads0"], rtol=1e-5, atol=2e-5)


# ------------------------------------------------------------------ 3. a batch == its problems one by one
@pytest.mark.parametrize("dt", ["f32", "bf16"])
@pytest.mark.parametrize("shared_w", [True, False], ids=["shared_w", "own_w"])
def test_batch_matches_single_calls(api, dt, shared_w):
    M, bt, _ = api
    dtype = DTYPES[dt]
    rng = np.random.default_rng(11)
    fs = [3, 0, 9, 1, 4, 2, 5, 9]
    zs = [1.5, 1.0, 0.0, -1.0, 0.25, 1.5, 0.5, 2.0]
    lrs = [0.1, 0.2, 0.1, 1e-3, 0.0, 0.05, 0.1, 0.3]
    B, n, d, ld = len(fs), 9, 1000, 1003
    buf = torch.stack([matrix(rng, n, d, ld, dtype, specials=b % 2 == 0)[0] for b in range(B)])
    G = buf[:, :, :d]
    W = vec(rng, d) if shared_w else torch.stack([vec(rng, d) for _ in range(B)])
    before = buf.clone()
    calls = []

    def train(initial, problems):
        calls.append((initial.clone(), problems))
        return fake(initial)
    crafted, mu, sigma = bt.backdoor_rows(G, fs, zs, W, lrs, train)
    active = [b for b in range(B) if fs[b] > 0 and zs[b] != 0]
    assert len(calls) == 1 and calls[0][1] == active and calls[0][0].shape == (len(active), d)
    assert crafted.shape == mu.shape == sigma.shape == (B, d) and crafted.dtype == torch.float32
    assert same_bits(buf[:, :, d:], before[:, :, d:])
    for b in range(B):
        if fs[b] == 0:
            assert bool(crafted[b].isnan().all() and mu[b].isnan().all() and sigma[b].isnan().all()), b
            assert same_bits(buf[b], before[b]), b
            continue
        single_init = []
        att = M.BackdoorAttack(zs[b], lambda p: (single_init.append(p.clone()), fake(p))[1])
        Gb = before[b, :, :d].clone()
        got = att.attack_rows(Gb, fs[b], W if shared_w else W[b], lrs[b])
        assert same_bits(mu[b], att.grads_mean) and same_bits(sigma[b], att.grads_stdev), b
        assert same_bits(G[b], Gb), b
        if zs[b] == 0:
            assert got is None and not single_init and same_bits(crafted[b], mu[b]), b
        else:
            assert same_bits(crafted[b], got), b
            assert same_bits(calls[0][0][active.index(b)], single_init[0]), b


def test_uniform_values_and_no_active_problem(api):
    M, bt, _ = api
    rng = np.random.default_rng(5)
    B, n, d = 4, 6, 300
    G = torch.stack([matrix(rng, n, d, d, torch.float32, specials=False)[1] for _ in range(B)])
    w = vec(rng, d)
    G2 = G.clone()
    got = bt.backdoor_rows(G, 2, 1.5, w, 0.1, lambda x, p: fake(x))
    want = bt.backdoor_rows(G2, [2] * B, np.full(B, 1.5), w, torch.full((B,), 0.1, dtype=torch.float64),
                            lambda x, p: fake(x))
    assert all(same_bits(a, b) for a, b in zip(got, want)) and same_bits(G, G2)

    def never(x, p):
        raise AssertionError("the training was called without an attacking problem")
    G3 = G.clone()
    crafted, mu, _ = bt.backdoor_rows(G3, [0, 2, 3, 0], [1.0, 0.0, 0.0, 2.0], w, 0.1, never)
    assert same_bits(G3, G) and same_bits(crafted[1:3], mu[1:3])


def test_python_errors(api):
    M, bt, _ = api
    B, n, d = 2, 5, 16
    G = torch.randn((B, n, d), device="cuda")
    before = G.clone()
    w = torch.zeros(d, device="cuda")
    ok = lambda x, p: fake(x)                                                       # noqa: E731
    with pytest.raises(TypeError, match="host"):
        bt.backdoor_rows(G, torch.tensor([1, 2], device="cuda"), 1.5, w, 0.1, ok)
    with pytest.raises(TypeError, match="host"):
        bt.backdoor_rows(G, 2, 1.5, w, torch.tensor([0.1, 0.2], device="cuda"), ok)
    with pytest.raises(ValueError, match="one value per problem"):
        bt.backdoor_rows(G, [1, 2, 3], 1.5, w, 0.1, ok)
    with pytest.raises(ValueError, match="one value per problem"):
        bt.backdoor_rows(G, 2, [1.5], w, 0.1, ok)
    with pytest.raises(ValueError, match="problem 1"):                            # f_b > n
        bt.backdoor_rows(G, [1, n + 1], 1.5, w, 0.1, ok)
    for bad_w in (torch.zeros(d - 1, device="cuda"), torch.zeros((B + 1, d), device="cuda"),
                  torch.zeros(d, dtype=torch.float64, device="cuda")):
        with pytest.raises(ValueError, match="original_params"):
            bt.backdoor_rows(G, 2, 1.5, bad_w, 0.1, ok)
    for bad in (lambda x, p: x[:, :-1], lambda x, p: x.double(), lambda x, p: x.cpu(), lambda x, p: x.cpu().numpy(),
                lambda x, p: x[:1]):
        with pytest.raises(ValueError, match="train_malicious_network"):
            bt.backdoor_rows(G, 2, 1.5, w, 0.1, bad)
    with pytest.raises(ValueError, match="train_malicious_network"):           # the single form's training returns [D]
        M.BackdoorAttack(1.5, lambda p: p.cpu().numpy()).attack_rows(G[0], 2, w, 0.1)
    assert same_bits(G, before)                                                  # nothing written before the finish


# ------------------------------------------------------------------ 4. a short sweep == the same steps per problem
def test_backdoor_sweep_matches_loop(api):
    M, bt, D = api
    saved = os.environ.get("AFL_GRAM_SPLITS")
    os.environ["AFL_GRAM_SPLITS"] = SPLITS                      # the batch and the single calls split d alike
    try:
        rng = np.random.default_rng(3)
        fs = [0, 2, 5, 2, 5, 3]
        zs = [1.5, 1.5, 0.5, 0.0, 1.0, -0.5]
        B, n, d, lr = len(fs), 23, 2051, 0.1
        G = torch.stack([matrix(rng, n, d, d, torch.float32, specials=False)[1] for _ in range(B)])
        w = vec(rng, d)
        loop = G.clone()
        bt.backdoor_rows(G, fs, zs, w, lr, lambda x, p: fake(x))
        kidx = bt.krum(G, n, fs, return_index=True)
        out, sel = bt.bulyan(G, n, fs, return_selection=True)
        mk = bt.attack_metrics(G, fs, krum_index=kidx)
        mb = bt.attack_metrics(G, fs, aggregated=out, selection=sel)
        kidx_h, sel_h = kidx.cpu().tolist(), sel.cpu()
        for b in range(B):
            Gb = loop[b].clone()
            M.BackdoorAttack(zs[b], fake).attack_rows(Gb, fs[b], w, lr)
            assert same_bits(Gb, G[b]), b
            k = D.krum(Gb, n, fs[b], return_index=True)
            assert kidx_h[b] == k, b
            ob, sb = D.bulyan(Gb, n, fs[b], return_selection=True)
            theta = n - 2 * fs[b]
            assert same_bits(sel_h[b, :theta], sb.cpu()) and same_bits(out[b], ob), b
            k1 = bt.attack_metrics(Gb[None], fs[b], krum_index=torch.tensor([k], dtype=torch.int32, device="cuda"))
            b1 = bt.attack_metrics(Gb[None], fs[b], aggregated=ob[None], selection=sb[None])
            assert same_bits(mk["rel_deviation"][b:b + 1], k1["rel_deviation"]), b
            assert bool(mk["krum_success"][b]) == bool(k1["krum_success"][0]), b
            assert same_bits(mb["rel_deviation"][b:b + 1], b1["rel_deviation"]), b
            assert same_bits(mb["bulyan_malicious_fraction"][b:b + 1], b1["bulyan_malicious_fraction"]), b
    finally:
        if saved is None:
            os.environ.pop("AFL_GRAM_SPLITS", None)
        else:
            os.environ["AFL_GRAM_SPLITS"] = saved


# ------------------------------------------------------------------ 5. the harness's -b experiment
@pytest.mark.parametrize("backdoor", ["pattern", 1])
def test_harness_backdoor(api, tmp_path, monkeypatch, backdoor):
    M, *_ = api
    from attacking_federate_learning_b200 import harness
    seen = []
    original = M.BackdoorAttack.attack_rows

    def checked(self, users_grads, f, w, lr):
        crafted = original(self, users_grads, f, w, lr)
        zs = self.num_std * self.grads_stdev
        lo, hi = self.grads_mean - zs, self.grads_mean + zs
        ok = crafted.isnan() | ((crafted >= lo) & (crafted <= hi))
        seen.append(bool(ok.all()) and same_bits(users_grads[:f], crafted.expand(f, -1)))
        return crafted
    monkeypatch.setattr(M.BackdoorAttack, "attack_rows", checked)
    acc, epochs, csv = harness.main(0.2, 1.0, "Krum", users_count=10, epochs=3, out_dir=str(tmp_path), train_size=2000,
                                    test_size=400, test_step=1, backdoor=backdoor)
    assert seen == [True] * 3 and epochs == [0, 1, 2]
    assert os.path.exists(csv) and f"backdoor-{backdoor}_" in os.path.basename(csv) and "alpha_4" in csv
    assert np.loadtxt(csv, delimiter=",").shape == (3,)
