"""The CIFAR10 backdoor sweep on an H100 (sweep.py with dataset='CIFAR10' and cifar10_backdoor=True,
csrc/cifar_backdoor.cu), with TF32 off.

1. The trainer kernel against harness.BackdoorTrainer.train (fp32 autograd) and a float64 restatement of it, for a
   pattern set of whole minibatches, one with a tail minibatch, and a one-sample set.
2. One step at alpha = 0 and m <= 128: the step's gradient row is afl_cifar10_client_grads' on the same rows bit for
   bit, and the update is formed from it with the documented roundings.
3. An initial vector that already scores 100 % comes back bit for bit.
4. Problems with f = 0, z = 0 or a set status leave sentinel-filled outputs alone.
5. A problem's result is the same bits alone and inside a mixed batch.
6. A NaN initial sets AFL_ERR_NAN_DIST_LOSS (alpha > 0) or AFL_ERR_NAN_LOSS (alpha = 0) for that problem only.
7. The backdoor test against BackdoorTrainer.test('POST'), with out-of-range slots and sets.
8. Sweeps: captured equals eager; CIFAR10 drift experiments are not moved by backdoor experiments in their batch; a
   NaN-loss experiment fails alone.
9. The first weight step against harness.main(dataset='CIFAR10', backdoor='pattern' and 1), on synthetic data and on
   generated CIFAR10 files through data_dir.
"""
import os

import numpy as np
import pytest
import torch

from test_data_files import write_cifar10

pytestmark = pytest.mark.gpu

D = 117_706
SPLITS = "4"
# Trained vectors: ||k - r64|| / ||r64 - initial|| for the kernel k against the float64 restatement r64 must be within
# FACTOR times the same figure for fp32 autograd (BackdoorTrainer.train), plus FLOOR: both are fp32 trainings of
# dependent SGD steps whose sums run in different orders, so their distances to the float64 trajectory are of one size,
# while a wrong term (a missing weight decay, MSE or 1/m factor, a wrong row) moves the result by O(1) of the step.
FACTOR, FLOOR = 4.0, 1e-6


@pytest.fixture(scope="module")
def env():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    import __graft_entry__ as g
    g.build()
    from attacking_federate_learning_b200 import _native, harness, sweep
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    return _native, harness, sweep


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
    (x, y), _, net = harness.experiment_setup(seed, n_train, 10, "cuda", "CIFAR10")
    layout = harness.ParamLayout(net.parameters())
    return x, y, layout, layout.flatten(list(net.parameters()))


def dev(v, dtype):
    return torch.as_tensor(np.asarray(v), dtype=dtype, device="cuda")


def run_trainer(nat, initial, sets, index, f=None, z=None, status=None, alpha=4.0, epochs=2, out=None, m=200):
    """The trainer on initial [B, D]; returns (out, status, the gradient workspace as [B, D] floats)."""
    B = initial.shape[0]
    xs, ys, lens = sets
    f = dev([1] * B if f is None else f, torch.int32)
    z = dev([1.0] * B if z is None else z, torch.float64)
    status = dev([0] * B, torch.int32) if status is None else status
    out = torch.full_like(initial, -7.25) if out is None else out
    index = dev(index, torch.int32)                 # every array the kernel reads stays alive until it has run
    L = nat.lib()
    ws = torch.empty(L.afl_cifar10_backdoor_train_workspace_bytes(B) // 4, dtype=torch.float32, device="cuda")
    nat.check(L.afl_cifar10_backdoor_train(initial.data_ptr(), out.data_ptr(), B, D, xs.data_ptr(), ys.data_ptr(),
                                           xs.shape[0], xs.shape[1], lens.data_ptr(), index.data_ptr(), f.data_ptr(),
                                           z.data_ptr(), status.data_ptr(), alpha, epochs, m, ws.data_ptr(),
                                           ws.numel() * 4, torch.cuda.current_stream().cuda_stream))
    torch.cuda.current_stream().synchronize()
    return out, status, ws.view(B, D)


def train64(harness, layout, x, y, initial, alpha=4.0, epochs=2):
    """BackdoorTrainer.train in float64 (same loop, fresh optimiser per minibatch)."""
    import torch.nn.functional as F
    net = harness.Cifar10Net().to("cuda", torch.float64)
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
    return torch.stack([w + 0.01 * i * torch.randn(D, device="cuda", generator=g) for i in range(k)]).contiguous()


def quiet(*a, **k):
    pass


@pytest.mark.parametrize("bd, n_train", [("pattern", 2000), ("pattern", 5000), (1, 2000)])
def test_trainer_against_backdoor_trainer_and_float64(env, bd, n_train):
    nat, harness, sweep = env
    x, y, layout, w = setup(harness, 3, n_train)
    sets = sweep.backdoor_sets([(bd, x, y, 3)])
    n = int(sets[2][0])
    assert n == {"pattern": {2000: 2000, 5000: 2500}, 1: {2000: 1}}[bd][n_train]
    initials = noise_initials(w, 2, 11)
    got, status, _ = run_trainer(nat, initials, sets, [0] * 2)
    assert status.cpu().tolist() == [0, 0]
    for b in range(2):
        tr = harness.BackdoorTrainer(bd, 4, 2, layout, x, y, "cuda", quiet, 3, dataset="CIFAR10")
        a32 = tr.train(initials[b].clone())
        r64 = train64(harness, layout, tr.x, tr.y, initials[b])
        scale = torch.linalg.norm(r64 - initials[b].double())
        assert scale > 1e-3                                                     # it trained
        e_k = float(torch.linalg.norm(got[b].double() - r64) / scale)
        e_a = float(torch.linalg.norm(a32.double() - r64) / scale)
        print(f"trainer {bd} {n_train} problem {b}: kernel {e_k:.3e}, fp32 autograd {e_a:.3e}")
        assert e_k <= FACTOR * e_a + FLOOR, (bd, n_train, b, e_k, e_a)


@pytest.mark.parametrize("m", [100, 128])
def test_one_step_gradient_is_the_client_gradient_bit_for_bit(env, m):
    nat, harness, sweep = env
    x, y, layout, w = setup(harness, 4, 2000)
    xs, ys, _ = sweep.backdoor_sets([("pattern", x, y, 4)])
    xs, ys = xs[:, :m].contiguous(), ys[:, :m].contiguous()                     # one minibatch of m rows
    init = noise_initials(w, 2, 3)[1:].contiguous()
    got, status, g = run_trainer(nat, init, (xs, ys, dev([m], torch.int32)), [0], alpha=0.0, epochs=1, m=m)
    assert int(status[0]) == 0 and not torch.equal(got[0], init[0])
    # client 0 of one client, its shard the m rows, epoch 0: the same rows in the same order
    G = torch.full((1, 1, D), 7.0, device="cuda")
    zero, one = dev([0], torch.int32), dev([1], torch.int32)
    nat.check(nat.lib().afl_cifar10_client_grads(init.data_ptr(), 1, D, xs.data_ptr(), ys.data_ptr(), 1, m,
                                                 zero.data_ptr(), one.data_ptr(), 1, m, zero.data_ptr(),
                                                 G.data_ptr(), G.stride(0),
                                                 G.stride(1), torch.cuda.current_stream().cuda_stream))
    torch.cuda.synchronize()
    assert torch.equal(g[0].view(torch.int32), G[0, 0].view(torch.int32))
    # p - 0.1 (g + 1e-4 p) with the kernel's two fused multiply-adds, each rounded once to fp32: the products of two
    # fp32 values are exact in the 64-bit significand of long double, and a long double sum lands on an fp32 midpoint
    # only with probability ~2^-40
    if np.finfo(np.longdouble).nmant < 63:
        pytest.skip("no 64-bit long double significand on this host")
    ld = np.longdouble
    p, gg = init[0].cpu().numpy(), g[0].cpu().numpy()
    dp = (ld(np.float32(1e-4)) * p.astype(ld) + gg.astype(ld)).astype(np.float32)
    want = (ld(np.float32(-0.1)) * dp.astype(ld) + p.astype(ld)).astype(np.float32)
    assert np.array_equal(got[0].cpu().numpy().view(np.int32), want.view(np.int32))


def test_early_exit_returns_initial_bit_for_bit(env):
    nat, harness, sweep = env
    x, y, layout, w = setup(harness, 0, 2000)
    sets = sweep.backdoor_sets([("pattern", x, y, 0)])
    init = w.clone()
    init[D - 10] = 1e4                                                          # fc3.bias[0]: every row says 0
    tr = harness.BackdoorTrainer("pattern", 4, 2, layout, x, y, "cuda", quiet, 0, dataset="CIFAR10")
    assert tr.train(init) is init
    got, status, _ = run_trainer(nat, init[None].contiguous(), sets, [0])
    assert int(status[0]) == 0
    assert torch.equal(got[0].view(torch.int32), init.view(torch.int32))


def test_inactive_problems_are_left_alone_and_batches_do_not_matter(env):
    nat, harness, sweep = env
    x, y, layout, w = setup(harness, 1, 2000)
    x2, y2, _, _ = setup(harness, 2, 5000)
    sets = sweep.backdoor_sets([("pattern", x, y, 1), (2, x, y, 1), ("pattern", x2, y2, 2)])
    inits = noise_initials(w, 6, 5)
    st = dev([0, 0, 0, 0, nat.AFL_ERR_PRECONDITION, 0], torch.int32)
    got, status, _ = run_trainer(nat, inits, sets, [0, 2, 1, 0, 1, 2], f=[2, 0, 1, 3, 2, 1],
                                 z=[1.0, 1.0, 0.0, 1.5, 1.0, 0.5], status=st, epochs=1)
    assert status.cpu().tolist() == [0, 0, 0, 0, nat.AFL_ERR_PRECONDITION, 0]
    sentinel = torch.full((D,), -7.25, device="cuda")
    for b in (1, 2, 4):                                                         # f = 0, z = 0, a set status
        assert torch.equal(got[b].view(torch.int32), sentinel.view(torch.int32)), b
    for b, s in ((0, 0), (3, 0), (5, 2)):                                       # alone: the same bits
        alone, _, _ = run_trainer(nat, inits[b:b + 1].contiguous(), sets, [s], epochs=1)
        assert torch.equal(alone[0].view(torch.int32), got[b].view(torch.int32)), b
        assert not torch.equal(got[b], inits[b])
    bad, status, _ = run_trainer(nat, inits[:2].contiguous(), sets, [3, -1], epochs=1)   # set index out of range
    assert status.cpu().tolist() == [nat.AFL_ERR_BAD_ARG] * 2


@pytest.mark.parametrize("alpha, code", [(4.0, "AFL_ERR_NAN_DIST_LOSS"), (0.0, "AFL_ERR_NAN_LOSS")])
def test_nan_initial_flags_its_problem_only(env, alpha, code):
    nat, harness, sweep = env
    x, y, layout, w = setup(harness, 0, 2000)
    k = next(k for k in (1, 2, 3) if int(harness.backdoor_set(k, x, y)[1][0]) != 0)   # NaN logits predict class 0
    sets = sweep.backdoor_sets([("pattern", x, y, 0), (k, x, y, 0)])
    inits = noise_initials(w, 3, 9)
    inits[1, D - 3] = float("nan")
    got, status, _ = run_trainer(nat, inits, sets, [0, 1, 0], alpha=alpha, epochs=1)
    assert status.cpu().tolist() == [0, getattr(nat, code), 0]
    for b in (0, 2):
        alone, _, _ = run_trainer(nat, inits[b:b + 1].contiguous(), sets, [0], alpha=alpha, epochs=1)
        assert torch.equal(alone[0].view(torch.int32), got[b].view(torch.int32))


def backdoor_test(nat, W, sets, index, m, slot, n_slots, loss, correct):
    xs, ys, lens = sets
    B = W.shape[0]
    L = nat.lib()
    ws = torch.empty(L.afl_cifar10_backdoor_test_workspace_bytes(B, xs.shape[1], m), dtype=torch.uint8, device="cuda")
    index_d, slot_d = dev(index, torch.int32), dev([slot], torch.int32)
    nat.check(L.afl_cifar10_backdoor_test(W.data_ptr(), B, D, xs.data_ptr(), ys.data_ptr(), xs.shape[0], xs.shape[1],
                                          lens.data_ptr(), index_d.data_ptr(), m, slot_d.data_ptr(), n_slots,
                                          loss.data_ptr(), correct.data_ptr(), ws.data_ptr(), ws.numel(),
                                          torch.cuda.current_stream().cuda_stream))
    torch.cuda.synchronize()


@pytest.mark.parametrize("m", [200, 64])
def test_backdoor_test_against_post(env, m):
    nat, harness, sweep = env
    x, y, layout, w = setup(harness, 2, 5000)
    specs = [("pattern", x, y, 2), (3, x, y, 2)]
    sets = sweep.backdoor_sets(specs)
    Wt = noise_initials(w, 5, 1)
    trained, _, _ = run_trainer(nat, Wt[:2].contiguous(), sets, [0, 1], epochs=1)
    Wt[2:4] = trained
    index = [0, 1, 0, 1, 2]                                                     # problem 4: a set index out of range
    loss = torch.full((3, 5), -1.0, dtype=torch.float64, device="cuda")
    correct = torch.full((3, 5), -1, dtype=torch.int32, device="cuda")
    backdoor_test(nat, Wt, sets, index, m, 1, 3, loss, correct)
    assert (loss[[0, 2]] == -1.0).all() and (correct[[0, 2]] == -1).all()
    assert float(loss[1, 4]) == -1.0 and int(correct[1, 4]) == -1
    for slot in (-1, 3):                                                        # slots out of range write nothing
        backdoor_test(nat, Wt, sets, index, m, slot, 3, loss, correct)
    assert (loss[[0, 2]] == -1.0).all() and (correct[[0, 2]] == -1).all()
    for b in range(4):
        tr = harness.BackdoorTrainer(specs[index[b]][0], 4, 5, layout, x, y, "cuda", quiet, 2, dataset="CIFAR10")
        tr.batch_size = m                                                       # the same set, tested in m-row batches
        layout.row_into_parameters(Wt[b], list(tr.net.parameters()))
        acc = tr.test("POST", to_print=False)
        n = len(tr.x)
        assert 100. * int(correct[1, b]) / n == acc, b
        want = 0.0
        with torch.no_grad():
            for lo in range(0, n, m):
                want += torch.nn.functional.nll_loss(tr.net(tr.x[lo:lo + m]), tr.y[lo:lo + m]).item()
        assert abs(float(loss[1, b]) - want) <= 1e-5 * max(1.0, abs(want)), (b, float(loss[1, b]), want)


def small_sweep(sweep, exps, epochs, capture, **kw):
    kw = dict(dict(learning_rate=0.1, batch_size=83, train_size=2000, test_size=500, test_step=2, mal_epochs=2,
                   fading_rate=2000, dataset="CIFAR10", cifar10_backdoor=True), **kw)
    return sweep.Sweep(exps, epochs, capture=capture, **kw)


MIXED = [("NoDefense", 0.24, 1.0, 10, 0, "pattern"), ("TrimmedMean", 0.24, 1.5, 10, 0), ("Krum", 0.1, 1.0, 10, 1, 1),
         ("TrimmedMean", 0.24, 0.5, 10, 1, "pattern"), ("NoDefense", 0.1, 1.0, 10, 1)]


def bits(t):
    return t.contiguous().view(torch.int32).cpu()


def test_captured_epochs_equal_eager(env, pinned_splits):
    _, _, sweep = env
    runs = []
    for capture in (False, True):
        sw = small_sweep(sweep, MIXED, 4, capture)
        for e in range(4):
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
    assert a.bd_x.shape[2:] == (3, 32, 32)


def test_drift_experiments_keep_their_bits_beside_backdoor_ones(env, pinned_splits):
    _, _, sweep = env
    drift = [e for e in MIXED if len(e) == 5]
    sw_a, sw_b = small_sweep(sweep, MIXED, 3, True), small_sweep(sweep, drift, 3, True)
    for e in range(3):
        sw_a.step(e)
        sw_b.step(e)
    ra, rb = sw_a.results(), sw_b.results()
    for i, e in enumerate(drift):
        pa, pb = sw_a.order.index(MIXED.index(e)), sw_b.order.index(i)
        assert torch.equal(bits(sw_a.W[pa]), bits(sw_b.W[pb])), e
        assert ra[MIXED.index(e)]["accuracies"] == rb[i]["accuracies"]
        assert "backdoor_accuracies" not in rb[i]


def test_nan_loss_experiment_fails_alone(env, pinned_splits):
    _, harness, sweep = env
    (x, y), _, _ = harness.experiment_setup(0, 2000, 10, "cpu", "CIFAR10")
    k = next(k for k in (1, 2, 3) if int(harness.backdoor_set(k, x, y)[1][0]) != 0)
    failing = ("NoDefense", 0.24, 1.0, 10, 0, k)
    others = [("NoDefense", 0.24, 1.0, 10, 1, "pattern"), ("TrimmedMean", 0.24, 1.5, 10, 0),
              ("TrimmedMean", 0.24, 0.5, 10, 0, 2)]
    runs = []
    for exps in ([failing] + others, others):
        sw = small_sweep(sweep, exps, 3, True, alpha=0)                        # no dist loss: the NLL check fires
        sw.step(0)
        if len(exps) > len(others):
            sw.W[sw.order.index(0)] = float("nan")
        for e in range(1, 3):
            sw.step(e)
        runs.append((sw, sw.results()))
    (a, ra), (b, rb) = runs
    assert type(ra[0]["error"]) is Exception and str(ra[0]["error"]).endswith(": Got nan loss")
    for i in range(len(others)):
        assert ra[i + 1]["error"] is None and rb[i]["error"] is None
        pa, pb = a.order.index(i + 1), b.order.index(i)
        assert torch.equal(bits(a.W[pa]), bits(b.W[pb])), others[i]
        assert ra[i + 1]["accuracies"] == rb[i]["accuracies"]
        assert ra[i + 1].get("backdoor_accuracies") == rb[i].get("backdoor_accuracies")


# The first epoch's weight step of the sweep against harness.main's: ||dW_sweep - dW_h|| / ||dW_h||.  The client
# gradients and the malicious training sum in other orders (fp32), and the crafted rows are clipped to mu +/- z sigma,
# so the steps agree to accumulated fp32 rounding; 1e-3 is far below a wrong term, which is O(1).
STEP_BOUND = 1e-3


@pytest.fixture(scope="module")
def cifar_root(tmp_path_factory):
    return write_cifar10(tmp_path_factory.mktemp("data") / "cifar10_data", per_batch=400, n_test=300, seed=2)


@pytest.mark.parametrize("bd", ["pattern", 1])
@pytest.mark.parametrize("files", [False, True])
def test_first_weight_step_against_harness_main(env, cifar_root, tmp_path, monkeypatch, bd, files):
    _, harness, sweep = env
    from attacking_federate_learning_b200.server import AggregationServer
    seen = {}

    class Recording(AggregationServer):
        def __init__(self, *a, initial_weights=None, **k):
            super().__init__(*a, initial_weights=initial_weights, **k)
            seen['w0'] = initial_weights.clone()

        def defend(self, *a, **k):
            super().defend(*a, **k)
            seen.setdefault('w1', self.current_weights.clone())
    e = ("NoDefense", 0.24, 1.0, 10, 0, bd)
    kw = dict(learning_rate=0.1, batch_size=83, fading_rate=2000, dataset="CIFAR10")
    kw.update(dict(data_dir=cifar_root) if files else dict(train_size=2000, test_size=500))
    monkeypatch.setattr(harness, 'AggregationServer', Recording)
    harness.main(e[1], e[2], e[0], users_count=e[3], epochs=1, seed=e[4], backdoor=bd, out_dir=str(tmp_path),
                 output=str(tmp_path / 'log.txt'), **kw)
    monkeypatch.undo()
    sw = sweep.Sweep([e], 1, capture=False, cifar10_backdoor=True, **kw)
    assert torch.equal(sw.W[0], seen['w0'])                               # the same initial weights
    sw.step(0)
    assert sw.results()[0]["error"] is None
    step = seen['w1'].double() - seen['w0'].double()
    rel = float(((sw.W[0].double() - seen['w0'].double()) - step).norm() / step.norm())
    print(f"first weight step CIFAR10 {e} files={files}: relative difference {rel:.3e}")
    assert rel <= STEP_BOUND, rel
