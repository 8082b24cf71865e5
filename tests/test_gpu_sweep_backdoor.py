"""The backdoor sweep on an H100 (sweep.py, csrc/backdoor_train.cu, the _dev backdoor crafting).

1. The trainer kernel against harness.BackdoorTrainer.train (fp32 autograd) and a float64 restatement of it, for a
   pattern set of whole minibatches, one with a tail minibatch, and a one-sample set, from several initial vectors.
2. An initial vector that already scores 100 % comes back bit for bit.
3. Problems with f = 0, z = 0 or a set status leave sentinel-filled outputs alone.
4. A problem's result is the same bits alone and inside a mixed batch.
5. A NaN initial sets AFL_ERR_NAN_DIST_LOSS (alpha > 0) or AFL_ERR_NAN_LOSS (alpha = 0) for that problem only.
6. DeviceRound.backdoor_start / backdoor_finish equal batched.backdoor_rows bit for bit.
7. The backdoor test against BackdoorTrainer.test('POST').
8. Sweeps: captured equals eager; drift experiments are not moved by backdoor experiments in their batch; a NaN-loss
   experiment fails alone.
9. End to end against harness.main(..., backdoor='pattern' and 1).
"""
import os
import re

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

D = 79_510
SPLITS = "4"
# Trained vectors: ||k - r64|| / ||r64 - initial|| for the kernel k against the float64 restatement r64 must be within
# FACTOR times the same figure for fp32 autograd (BackdoorTrainer.train), plus FLOOR.  Both are fp32 trainings of 50
# dependent SGD steps whose sums run in different orders, so their distances to the float64 trajectory are of one
# size; a wrong term (a missing weight decay, MSE or 1/m factor, a wrong row) moves the result by O(1) of the step.
FACTOR, FLOOR = 4.0, 1e-6


@pytest.fixture(scope="module")
def env():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    import __graft_entry__ as g
    g.build()
    from attacking_federate_learning_b200 import _native, batched, harness, sweep
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    return _native, batched, harness, sweep


@pytest.fixture
def pinned_splits():
    saved = os.environ.get("AFL_GRAM_SPLITS")
    os.environ["AFL_GRAM_SPLITS"] = SPLITS
    yield
    if saved is None:
        os.environ.pop("AFL_GRAM_SPLITS", None)
    else:
        os.environ["AFL_GRAM_SPLITS"] = saved


def setup(harness, seed, n_train):
    (x, y), _, net = harness.experiment_setup(seed, n_train, 10, "cuda")
    layout = harness.ParamLayout(net.parameters())
    return x, y, layout, layout.flatten(list(net.parameters()))


def dev(v, dtype):
    return torch.as_tensor(np.asarray(v), dtype=dtype, device="cuda")


def run_trainer(nat, initial, sets, index, f=None, z=None, status=None, alpha=4.0, epochs=5, out=None):
    B = initial.shape[0]
    xs, ys, lens = sets
    f = dev([1] * B if f is None else f, torch.int32)
    z = dev([1.0] * B if z is None else z, torch.float64)
    status = dev([0] * B, torch.int32) if status is None else status
    out = torch.full_like(initial, -7.25) if out is None else out
    index = dev(index, torch.int32)                 # every array the kernel reads stays alive until it has run
    nat.check(nat.lib().afl_mnist_backdoor_train(initial.data_ptr(), out.data_ptr(), B, D, xs.data_ptr(), ys.data_ptr(),
                                                 xs.shape[0], xs.shape[1], lens.data_ptr(), index.data_ptr(),
                                                 f.data_ptr(), z.data_ptr(), status.data_ptr(), alpha, epochs, 200,
                                                 torch.cuda.current_stream().cuda_stream))
    torch.cuda.current_stream().synchronize()
    return out, status


def train64(harness, layout, x, y, initial, alpha=4.0, epochs=5):
    """BackdoorTrainer.train in float64 (same loop, fresh optimiser per minibatch)."""
    import torch.nn.functional as F
    net = harness.MnistNet().to("cuda", torch.float64)
    params = list(net.parameters())
    layout.row_into_parameters(initial.double(), params)
    p0 = [p.detach().clone() for p in params]
    x = x.double()
    for _ in range(epochs):
        for lo in range(0, len(x), 200):
            opt = torch.optim.SGD(params, lr=0.1, momentum=0.9, weight_decay=0.0001)
            opt.zero_grad()
            loss = F.nll_loss(net(x[lo:lo + 200]), y[lo:lo + 200])
            if alpha > 0:
                loss = loss + alpha * sum(F.mse_loss(p, q) for p, q in zip(params, p0))
            loss.backward()
            opt.step()
    return layout.flatten(params, out=torch.empty(D, dtype=torch.float64, device="cuda"))


def noise_initials(w, k, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return torch.stack([w + 0.02 * i * torch.randn(D, device="cuda", generator=g) for i in range(k)]).contiguous()


@pytest.mark.parametrize("bd, n_train", [("pattern", 2000), ("pattern", 5000), (1, 2000)])
def test_trainer_against_backdoor_trainer_and_float64(env, bd, n_train):
    nat, _, harness, sweep = env
    x, y, layout, w = setup(harness, 3, n_train)
    sets = sweep.backdoor_sets([(bd, x, y, 3)])
    n = int(sets[2][0])
    assert n == {"pattern": {2000: 2000, 5000: 2500}, 1: {2000: 1}}[bd][n_train]
    initials = noise_initials(w, 3, 11)
    got, status = run_trainer(nat, initials, sets, [0] * 3)
    assert status.cpu().tolist() == [0, 0, 0]
    for b in range(3):
        tr = harness.BackdoorTrainer(bd, 4, 5, layout, x, y, "cuda", lambda *a, **k: None, 3)
        a32 = tr.train(initials[b].clone())
        r64 = train64(harness, layout, tr.x, tr.y, initials[b])
        scale = torch.linalg.norm(r64 - initials[b].double())
        assert scale > 1e-3                                                     # it trained
        e_k = float(torch.linalg.norm(got[b].double() - r64) / scale)
        e_a = float(torch.linalg.norm(a32.double() - r64) / scale)
        assert e_k <= FACTOR * e_a + FLOOR, (bd, n_train, b, e_k, e_a)


def test_early_exit_returns_initial_bit_for_bit(env):
    nat, _, harness, sweep = env
    x, y, layout, w = setup(harness, 0, 2000)
    sets = sweep.backdoor_sets([("pattern", x, y, 0)])
    init = w.clone()
    init[D - 10] = 1e4                                                          # fc2.bias[0]: every row says 0
    tr = harness.BackdoorTrainer("pattern", 4, 5, layout, x, y, "cuda", lambda *a, **k: None, 0)
    assert tr.train(init) is init
    got, status = run_trainer(nat, init[None].contiguous(), sets, [0])
    assert int(status[0]) == 0
    assert torch.equal(got[0].view(torch.int32), init.view(torch.int32))


def test_inactive_problems_are_left_alone_and_batches_do_not_matter(env):
    nat, _, harness, sweep = env
    x, y, layout, w = setup(harness, 1, 2000)
    x2, y2, _, _ = setup(harness, 2, 5000)
    sets = sweep.backdoor_sets([("pattern", x, y, 1), (2, x, y, 1), ("pattern", x2, y2, 2)])
    inits = noise_initials(w, 6, 5)
    st = dev([0, 0, 0, 0, nat.AFL_ERR_PRECONDITION, 0], torch.int32)
    got, status = run_trainer(nat, inits, sets, [0, 2, 1, 0, 1, 2], f=[2, 0, 1, 3, 2, 1], z=[1.0, 1.0, 0.0, 1.5, 1.0, 0.5],
                              status=st)
    assert status.cpu().tolist() == [0, 0, 0, 0, nat.AFL_ERR_PRECONDITION, 0]
    sentinel = torch.full((D,), -7.25, device="cuda")
    for b in (1, 2, 4):                                                         # f = 0, z = 0, a set status
        assert torch.equal(got[b].view(torch.int32), sentinel.view(torch.int32)), b
    for b, s in ((0, 0), (3, 0), (5, 2)):                                       # alone: the same bits
        alone, _ = run_trainer(nat, inits[b:b + 1].contiguous(), sets, [s])
        assert torch.equal(alone[0].view(torch.int32), got[b].view(torch.int32)), b
        assert not torch.equal(got[b], inits[b])


@pytest.mark.parametrize("alpha, code", [(4.0, "AFL_ERR_NAN_DIST_LOSS"), (0.0, "AFL_ERR_NAN_LOSS")])
def test_nan_initial_flags_its_problem_only(env, alpha, code):
    nat, _, harness, sweep = env
    x, y, layout, w = setup(harness, 0, 2000)
    k = next(k for k in (1, 2, 3) if int(harness.backdoor_set(k, x, y)[1][0]) != 0)   # NaN logits predict class 0
    sets = sweep.backdoor_sets([("pattern", x, y, 0), (k, x, y, 0)])
    inits = noise_initials(w, 3, 9)
    inits[1, D - 3] = float("nan")
    got, status = run_trainer(nat, inits, sets, [0, 1, 0], alpha=alpha)
    assert status.cpu().tolist() == [0, getattr(nat, code), 0]
    for b in (0, 2):
        alone, _ = run_trainer(nat, inits[b:b + 1].contiguous(), sets, [0], alpha=alpha)
        assert torch.equal(alone[0].view(torch.int32), got[b].view(torch.int32))


def test_dev_crafting_equals_backdoor_rows(env):
    nat, batched, _, _ = env
    g = torch.Generator(device="cuda").manual_seed(4)
    B, N, d = 6, 9, 4099
    G = torch.randn((B, N, d + 29), device="cuda", generator=g)[:, :, :d]
    w = torch.randn((B, d), device="cuda", generator=g)
    fs, zs, lrs = [0, 1, 3, 9, 2, 4], [1.0, 1.5, 0.0, 0.5, 2.0, -1.0], [0.1, 0.05, 0.1, 0.2, 1e-3, 0.1]
    G1, G2 = G.clone(), G.clone()

    def stand_in(initial, problems=None):
        return initial * 0.9 + 0.01
    crafted, mu, sigma = batched.backdoor_rows(G1, fs, zs, w, lrs, stand_in)
    rnd = batched.DeviceRound(G2, rules=())
    rnd.f.copy_(dev(fs, torch.int32)); rnd.z.copy_(dev(zs, torch.float64)); rnd.lr.copy_(dev(lrs, torch.float64))
    mu2, sigma2, initial = rnd.backdoor_start(w)
    crafted2 = rnd.backdoor_finish(stand_in(initial))
    for a, b in ((crafted, crafted2), (mu, mu2), (sigma, sigma2), (G1, G2)):
        assert torch.equal(a.contiguous().view(torch.int32), b.contiguous().view(torch.int32))
    assert rnd.status.cpu().tolist() == [0] * B
    rnd.f.copy_(dev([0, 1, 10, -1, 2, 4], torch.int32))                        # f_b > N and f_b < 0 are flagged
    rnd.backdoor_start(w)
    assert rnd.status.cpu().tolist() == [0, 0, nat.AFL_ERR_BAD_ARG, nat.AFL_ERR_BAD_ARG, 0, 0]


def test_backdoor_test_against_post(env):
    nat, _, harness, sweep = env
    x, y, layout, w = setup(harness, 2, 5000)
    specs = [("pattern", x, y, 2), (3, x, y, 2)]
    sets = sweep.backdoor_sets(specs)
    Wt = noise_initials(w, 4, 1)
    trained, _ = run_trainer(nat, Wt[:2].contiguous(), sets, [0, 1], epochs=1)
    Wt[2:] = trained
    index = [0, 1, 0, 1]
    loss = torch.full((3, 4), -1.0, dtype=torch.float64, device="cuda")
    correct = torch.full((3, 4), -1, dtype=torch.int32, device="cuda")
    xs, ys, lens = sets
    index_d, slot = dev(index, torch.int32), dev([1], torch.int32)
    nat.check(nat.lib().afl_mnist_backdoor_test(Wt.data_ptr(), 4, D, xs.data_ptr(), ys.data_ptr(), 2, xs.shape[1],
                                                lens.data_ptr(), index_d.data_ptr(), 200, slot.data_ptr(), 3,
                                                loss.data_ptr(), correct.data_ptr(),
                                                torch.cuda.current_stream().cuda_stream))
    assert (loss[[0, 2]] == -1.0).all() and (correct[[0, 2]] == -1).all()
    for b in range(4):
        tr = harness.BackdoorTrainer(specs[index[b]][0], 4, 5, layout, x, y, "cuda", lambda *a, **k: None, 2)
        layout.row_into_parameters(Wt[b], list(tr.net.parameters()))
        acc = tr.test("POST", to_print=False)
        n = len(tr.x)
        assert 100. * int(correct[1, b]) / n == acc, b
        want = 0.0
        with torch.no_grad():
            for lo in range(0, n, 200):
                want += torch.nn.functional.nll_loss(tr.net(tr.x[lo:lo + 200]), tr.y[lo:lo + 200]).item()
        assert abs(float(loss[1, b]) - want) <= 1e-5 * max(1.0, abs(want)), (b, float(loss[1, b]), want)


def small_sweep(sweep, exps, epochs, capture, **kw):
    kw = dict(dict(learning_rate=0.1, batch_size=83, train_size=2000, test_size=500, test_step=2), **kw)
    return sweep.Sweep(exps, epochs, capture=capture, **kw)


MIXED = [("NoDefense", 0.24, 1.0, 10, 0, "pattern"), ("TrimmedMean", 0.24, 1.5, 10, 0), ("Krum", 0.1, 1.0, 10, 1, 1),
         ("TrimmedMean", 0.24, 0.5, 10, 1, "pattern"), ("NoDefense", 0.1, 1.0, 10, 1)]


def bits(t):
    return t.contiguous().view(torch.int32).cpu()


def test_captured_epochs_equal_eager(env, pinned_splits):
    _, _, _, sweep = env
    runs = []
    for capture in (False, True):
        sw = small_sweep(sweep, MIXED, 5, capture)
        for e in range(5):
            sw.step(e)
        runs.append((sw, sw.results()))
    (a, ra), (b, rb) = runs
    for t in ("W", "V", "loss_sum", "correct", "bd_loss_sum", "bd_correct", "bd_mal"):
        assert torch.equal(bits(getattr(a, t)), bits(getattr(b, t))), t
    assert [r["backdoor_accuracies"] for r in ra if "backdoor_accuracies" in r] == \
        [r["backdoor_accuracies"] for r in rb if "backdoor_accuracies" in r]
    assert all(r["error"] is None for r in ra + rb)
    assert a.order == b.order == [1, 4, 2, 3, 0]                                # drift by rule, then backdoor by rule
    assert (a.bd_correct.cpu() >= 0).all() and a.n_backdoor == 3


def test_drift_experiments_keep_their_bits_beside_backdoor_ones(env, pinned_splits):
    _, _, _, sweep = env
    drift = [e for e in MIXED if len(e) == 5]
    sw_a, sw_b = small_sweep(sweep, MIXED, 4, True), small_sweep(sweep, drift, 4, True)
    for e in range(4):
        sw_a.step(e)
        sw_b.step(e)
    ra, rb = sw_a.results(), sw_b.results()
    for i, e in enumerate(drift):
        pa, pb = sw_a.order.index(MIXED.index(e)), sw_b.order.index(i)
        assert torch.equal(bits(sw_a.W[pa]), bits(sw_b.W[pb])), e
        assert ra[MIXED.index(e)]["accuracies"] == rb[i]["accuracies"]
        assert "backdoor_accuracies" not in rb[i]


def test_nan_loss_experiment_fails_alone(env, pinned_splits):
    _, _, harness, sweep = env
    (x, y), _, _ = harness.experiment_setup(0, 2000, 10, "cpu")
    k = next(k for k in (1, 2, 3) if int(harness.backdoor_set(k, x, y)[1][0]) != 0)
    failing = ("NoDefense", 0.24, 1.0, 10, 0, k)
    others = [("NoDefense", 0.24, 1.0, 10, 1, "pattern"), ("TrimmedMean", 0.24, 1.5, 10, 0),
              ("TrimmedMean", 0.24, 0.5, 10, 0, 2)]
    runs = []
    for exps in ([failing] + others, others):
        sw = small_sweep(sweep, exps, 4, True)
        sw.step(0)
        if len(exps) > len(others):
            sw.W[sw.order.index(0)] = float("nan")
        for e in range(1, 4):
            sw.step(e)
        runs.append((sw, sw.results()))
    (a, ra), (b, rb) = runs
    assert type(ra[0]["error"]) is Exception and "Got nan" in str(ra[0]["error"])
    for i in range(len(others)):
        assert ra[i + 1]["error"] is None and rb[i]["error"] is None
        pa, pb = a.order.index(i + 1), b.order.index(i)
        assert torch.equal(bits(a.W[pa]), bits(b.W[pb])), others[i]
        assert ra[i + 1]["accuracies"] == rb[i]["accuracies"]
        assert ra[i + 1].get("backdoor_accuracies") == rb[i].get("backdoor_accuracies")


# The first epoch's weight step of the sweep against harness.main's: ||dW_sweep - dW_h|| / ||dW_h||.  The client
# gradients and the malicious training sum in other orders (fp32), and the crafted rows are clipped to mu +/- z sigma,
# so the steps agree to a few fp32 ulps of accumulated error; 1e-3 is far below a wrong term, which is O(1).
STEP_BOUND = 1e-3


@pytest.mark.parametrize("bd", ["pattern", 1])
def test_end_to_end_against_harness_main(env, tmp_path, monkeypatch, bd):
    _, _, harness, sweep = env
    kw = dict(learning_rate=0.1, batch_size=128, train_size=4000, test_size=1000)
    e = ("NoDefense", 0.24, 1.0, 10, 0, bd)
    sw = sweep.Sweep([e], 1, **kw)
    w0 = sw.W[0].clone()
    sw.step(0)
    seen = []
    orig = harness.AggregationServer.defend

    def defend(self, *a, **k):
        out = orig(self, *a, **k)
        seen.append(self.current_weights.clone())
        return out
    monkeypatch.setattr(harness.AggregationServer, "defend", defend)
    log = str(tmp_path / "log.txt")
    harness.main(e[1], e[2], e[0], users_count=e[3], epochs=1, out_dir=str(tmp_path / "h1"), seed=0, output=log,
                 backdoor=bd, **kw)
    monkeypatch.undo()
    step_h, step_s = seen[0] - w0, sw.W[0] - w0
    err = float(torch.linalg.norm((step_s - step_h).double()) / torch.linalg.norm(step_h.double()))
    assert err <= STEP_BOUND, err
    # a longer run: accuracies, backdoor accuracies and the CSV
    res = sweep.run([e], 6, out_dir=str(tmp_path / "sweep"), **kw)[0]
    log = str(tmp_path / "log6.txt")
    acc, epochs, csv = harness.main(e[1], e[2], e[0], users_count=e[3], epochs=6, out_dir=str(tmp_path / "h"), seed=0,
                                    output=log, backdoor=bd, **kw)
    assert res["error"] is None and epochs == res["accuracies_epochs"] == [0, 5]
    assert np.max(np.abs(np.array(acc) - res["accuracies"])) <= 1.0, (acc, res["accuracies"])
    post = [float(m) for m in re.findall(r"\[POST\] Average loss: [^,]+, Accuracy: \d+/\d+ \(([\d.]+)%\)",
                                         open(log).read())]
    assert len(post) == 2
    assert abs(post[0] - res["backdoor_accuracies"][0]) <= 1.0, (post, res["backdoor_accuracies"])
    assert abs(post[1] - res["backdoor_accuracies"][1]) <= 10.0, (post, res["backdoor_accuracies"])
    assert os.path.basename(res["csv"]) == os.path.basename(csv)[:-4] + "_seed_0.csv"
    want, got = open(csv).read().splitlines(), open(res["csv"]).read().splitlines()
    assert len(got) == len(want) == 2
    assert all(len(g) == len(w) and g.endswith(w[-4:]) for g, w in zip(got, want))   # np.savetxt's %.18e
    summary = open(tmp_path / "sweep" / "logs" / sweep.SUMMARY).read().splitlines()
    assert summary[0].split(",") == sweep.summary_header(True)
    assert summary[1].startswith(f"NoDefense,0.24,1.0,10,0,{bd},") and summary[1].endswith(",ok")
