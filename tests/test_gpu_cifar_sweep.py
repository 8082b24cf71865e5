"""The CIFAR10 training sweep on an H100 (sweep.py with dataset='CIFAR10', csrc/cifar_grad.cu).

1. Client gradients against float64 autograd of harness.Cifar10Net per tensor: each tensor's distance to float64
   within 4x fp32 autograd's plus a small floor, at every chunk boundary of m (1 ... 128), on shard-tail batches, at
   1024 clients (1- and 2-row shards, n = train_size), with rows_b = 0 and pitch sentinels.
2. MaxPool ties (windows of exact zeros, exact ties of positive values in both pools: the gradient takes the first
   maximum) and non-finite weights (NaN/inf positions equal fp32 autograd's entry for entry).
3. A client's gradient is bit-identical whatever B, N and the other problems are.
4. Evaluation against harness.main's test loop, first-maximum ties, out-of-range sets and slots.
5. sweep.run(dataset='CIFAR10'): captured equals eager, a failed Bulyan experiment leaves the others alone, an
   N = 1000 problem beside N = 10 ones, the first weight step against harness.main, and learnability.
"""
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

D = 117_706
LD = 117_728
SPLITS = "4"
# tensors in ParamLayout order
SLICES = {"conv1.w": (0, 432), "conv1.b": (432, 448), "conv2.w": (448, 16_832), "conv2.b": (16_832, 16_896),
          "fc1.w": (16_896, 41_472), "fc1.b": (41_472, 41_856), "fc2.w": (41_856, 115_584),
          "fc2.b": (115_584, 115_776), "fc3.w": (115_776, 117_696), "fc3.b": (117_696, D)}
# Per tensor: ||g - g64|| <= 4 ||g32 - g64|| + FLOOR ||g64||.  The kernel's sums run in another order than cuDNN's;
# the longest is conv1's weight gradient, 49 cells then up to 128 rows, whose fp32 error bound is (49 + 128) u ~ 1e-5
# relative to the sum of |terms|.
FLOOR = 1e-5


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


_DATA = {}


def data(harness, seed, n_train=2000, n_test=500):
    key = (seed, n_train, n_test)
    if key not in _DATA:
        (xtr, ytr), (xte, yte), net = harness.experiment_setup(seed, n_train, n_test, "cuda", "CIFAR10")
        _DATA[key] = (xtr, ytr, xte, yte, harness.ParamLayout(net.parameters()).flatten(list(net.parameters())))
    return _DATA[key]


def i32(v):
    return torch.as_tensor(np.asarray(v, np.int32), device="cuda")


def client_grads(nat, W, x, y, data_index, rows, n, m, epoch, G):
    """W [B, D]; x [n_sets, n_train, 3, 32, 32]; G [B, n, ld] fp32 (written in place)."""
    nat.check(nat.lib().afl_cifar10_client_grads(W.data_ptr(), W.shape[0], D, x.data_ptr(), y.data_ptr(), x.shape[0],
                                                 x.shape[1], data_index.data_ptr(), rows.data_ptr(), n, m,
                                                 epoch.data_ptr(), G.data_ptr(), G.stride(0), G.stride(1),
                                                 torch.cuda.current_stream().cuda_stream))


def autograd(harness, w, xb, yb, dtype):
    net = harness.Cifar10Net().to("cuda", dtype)
    layout = harness.ParamLayout(net.parameters())
    layout.row_into_parameters(w.to(dtype), list(net.parameters()))
    net.zero_grad()
    torch.nn.NLLLoss()(net(xb.to(dtype)), yb).backward()
    return torch.cat([p.grad.flatten().to(torch.float64) for p in net.parameters()])


def minibatch_rows(sweep, n_train, n, u, m, epoch):
    lo, hi = sweep.minibatch(n_train, n, u, m, epoch)
    return torch.arange(u + n * lo, u + n * hi, n, device="cuda")


def check_against_autograd(harness, got, W, xb, yb):
    g32 = autograd(harness, W, xb, yb, torch.float32)
    g64 = autograd(harness, W, xb, yb, torch.float64)
    got = got.double()
    for name, (a, b) in SLICES.items():
        ref = g64[a:b]
        err, err32 = float((got[a:b] - ref).norm()), float((g32[a:b] - ref).norm())
        assert err <= 4 * err32 + FLOOR * float(ref.norm()), (name, err, err32, float(ref.norm()))


def perturbed(w, seed, scale=0.01):
    return (w + scale * torch.randn(D, device="cuda", generator=torch.Generator("cuda").manual_seed(seed))).contiguous()


# every chunk count ceil(m / 16) at its boundaries, and the harness default
CHUNK_EDGES = [1, 15, 16, 17, 32, 33, 48, 49, 64, 65, 83, 97, 112, 113, 127, 128]


@pytest.mark.parametrize("m, n, epoch, u", [(m, 10, 0, 0) for m in CHUNK_EDGES] +
                         [(83, 10, 2, 9), (128, 10, 1, 7), (83, 7, 3, 6), (16, 7, 17, 6)])
def test_gradient_against_float64_autograd(env, m, n, epoch, u):
    """(83, 7, 3, 6): shard length 285 (2000 rows, 7 users), positions 249..284, a 36-row tail batch; (16, 7, 17, 6):
    positions 272..284, a 13-row tail."""
    nat, harness, sweep = env
    xtr, ytr, _, _, w = data(harness, 1)
    W = perturbed(w, m)
    G = torch.full((1, n, LD), 7.0, device="cuda")
    client_grads(nat, W[None], xtr[None], ytr[None], i32([0]), i32([n]), n, m, i32([epoch]), G)
    idx = minibatch_rows(sweep, len(xtr), n, u, m, epoch)
    check_against_autograd(harness, G[0, u, :D], W, xtr[idx], ytr[idx])
    assert bool((G[0, :, D:] == 7.0).all())


@pytest.mark.parametrize("n_train, m", [(1024, 83), (2048, 83), (2048, 1)])
def test_1024_clients_with_one_and_two_row_shards(env, n_train, m):
    nat, harness, sweep = env
    xtr, ytr, _, _, w = data(harness, 2, n_train=n_train, n_test=16)
    n = 1024
    G = torch.full((1, n, LD), -5.0, device="cuda")
    client_grads(nat, w[None].contiguous(), xtr[None], ytr[None], i32([0]), i32([n]), n, m, i32([1]), G)
    assert bool(torch.isfinite(G[0, :, :D]).all()) and bool((G[0, :, D:] == -5.0).all())
    for u in (0, 511, 1023):
        idx = minibatch_rows(sweep, n_train, n, u, m, 1)
        assert len(idx) == (n_train // n if m > 1 else 1)
        check_against_autograd(harness, G[0, u, :D], w, xtr[idx], ytr[idx])


def test_rows_zero_and_pitch_sentinels(env):
    nat, harness, sweep = env
    xtr, ytr, _, _, w = data(harness, 3)
    W = torch.stack([w, perturbed(w, 1), perturbed(w, 2)]).contiguous()
    rows, N = [10, 0, 5], 10
    G = torch.full((3, N, LD + 32), -3.0, device="cuda")
    client_grads(nat, W, xtr[None], ytr[None], i32([0, 0, 0]), i32(rows), N, 83, i32([2]), G)
    torch.cuda.synchronize()
    for b, nb in enumerate(rows):
        assert bool((G[b, nb:] == -3.0).all()), b                             # rows u >= n_b untouched
        assert bool((G[b, :, D:] == -3.0).all()), b                           # pitch columns untouched
        assert bool(torch.isfinite(G[b, :nb, :D]).all()), b
    idx = minibatch_rows(sweep, len(xtr), 5, 4, 83, 2)
    check_against_autograd(harness, G[2, 4, :D], W[2], xtr[idx], ytr[idx])


def test_batch_composition_does_not_change_a_gradient(env):
    nat, harness, _ = env
    x0, y0, _, _, w0 = data(harness, 3)
    x1, y1, _, _, w1 = data(harness, 4)
    X, Y = torch.stack([x0, x1]), torch.stack([y0, y1])
    G1 = torch.full((1, 10, LD), -3.0, device="cuda")
    client_grads(nat, w1[None].contiguous(), X, Y, i32([1]), i32([10]), 10, 83, i32([4]), G1)
    B, N = 9, 40
    W = torch.full((B, D), float("nan"), device="cuda")
    W[6], W[2] = w1, w0
    rows = [((b * 7) % N) + 1 for b in range(B)]
    rows[6], rows[2] = 10, 40
    sets = [b % 2 for b in range(B)]
    sets[6], sets[2] = 1, 0
    G = torch.full((B, N, LD), -3.0, device="cuda")
    client_grads(nat, W, X, Y, i32(sets), i32(rows), N, 83, i32([4]), G)
    torch.cuda.synchronize()
    assert torch.equal(G[6, :10, :D].view(torch.int32), G1[0, :, :D].view(torch.int32))
    G2 = torch.full((1, 40, LD), -3.0, device="cuda")
    client_grads(nat, w0[None].contiguous(), X, Y, i32([0]), i32([40]), 40, 83, i32([4]), G2)
    assert torch.equal(G[2, :, :D].view(torch.int32), G2[0, :, :D].view(torch.int32))
    for b in range(B):
        assert bool((G[b, rows[b]:] == -3.0).all()), b


def test_maxpool_ties_take_the_first_maximum(env):
    """conv1 filter 3 at zero weight and bias -1: every pool1 window of channel 3 is exact zeros.  Filter 5 at zero
    weight and bias 1: every window of channel 5 ties at 1.0, so its gradient goes to each window's first position.
    conv2 filter 7 at zero weight and bias 0.5: every pool2 window of channel 7 ties the same way."""
    nat, harness, sweep = env
    xtr, ytr, _, _, w = data(harness, 5)
    W = w.clone()
    W[3 * 27:4 * 27], W[432 + 3] = 0.0, -1.0
    W[5 * 27:6 * 27], W[432 + 5] = 0.0, 1.0
    W[448 + 7 * 256:448 + 8 * 256], W[16_832 + 7] = 0.0, 0.5
    G = torch.zeros((1, 10, LD), device="cuda")
    client_grads(nat, W[None], xtr[None], ytr[None], i32([0]), i32([10]), 10, 83, i32([0]), G)
    idx = minibatch_rows(sweep, len(xtr), 10, 3, 83, 0)
    got = G[0, 3, :D]
    check_against_autograd(harness, got, W, xtr[idx], ytr[idx])
    g64 = autograd(harness, W, xtr[idx], ytr[idx], torch.float64)
    assert bool((got[3 * 27:4 * 27] == 0).all()) and float(got[432 + 3]) == 0.0
    # channel 5 and conv2 channel 7 carry a gradient, and it is float64's (the first-maximum routing)
    for a, b in ((5 * 27, 6 * 27), (448 + 7 * 256, 448 + 8 * 256)):
        ref = g64[a:b]
        assert float(ref.norm()) > 0
        assert float((got[a:b].double() - ref).norm()) <= 1e-4 * float(ref.norm()), (a, b)


NONFINITE = {
    "nan_conv1_filter": lambda W: W[2 * 27:3 * 27].fill_(float("nan")),
    "inf_conv2_weight": lambda W: W.__setitem__(448 + 5 * 256 + 3 * 16 + 6, float("inf")),
    "nan_fc1_row": lambda W: W[16_896 + 17 * 64:16_896 + 18 * 64].fill_(float("nan")),
    "inf_fc3_bias": lambda W: W.__setitem__(117_696 + 4, float("inf")),
}


@pytest.mark.parametrize("case", list(NONFINITE))
def test_non_finite_weights_match_fp32_autograd(env, case):
    nat, harness, sweep = env
    xtr, ytr, _, _, w = data(harness, 6)
    W = w.clone()
    NONFINITE[case](W)
    G = torch.zeros((1, 10, LD), device="cuda")
    client_grads(nat, W[None], xtr[None], ytr[None], i32([0]), i32([10]), 10, 83, i32([1]), G)
    idx = minibatch_rows(sweep, len(xtr), 10, 2, 83, 1)
    got = G[0, 2, :D].double()
    g32 = autograd(harness, W, xtr[idx], ytr[idx], torch.float32)
    for name, (a, b) in SLICES.items():
        for pred in (torch.isnan, torch.isposinf, torch.isneginf):
            assert torch.equal(pred(got[a:b]), pred(g32[a:b])), (case, name, pred.__name__,
                                                                 int(pred(got[a:b]).sum()), int(pred(g32[a:b]).sum()))
        fin = torch.isfinite(g32[a:b])
        if fin.any():
            ref = g32[a:b][fin]
            assert float((got[a:b][fin] - ref).norm()) <= 1e-4 * float(ref.norm()) + 1e-30, (case, name)


@pytest.mark.parametrize("m, n_test", [(16, 497), (83, 499), (128, 513)])
def test_evaluation_against_the_harness_test_loop(env, m, n_test):
    """Last test batch of one row; problem 1 has an exact tie of its two top classes; a set index out of range
    writes nothing, and neither does a slot out of range."""
    nat, harness, _ = env
    _, _, xte, yte, w = data(harness, 7, n_test=n_test)
    w_tie = w.clone()
    w_tie[115_776 + 5 * 192:115_776 + 6 * 192] = w_tie[115_776 + 2 * 192:115_776 + 3 * 192]
    w_tie[117_696 + 2] = w_tie[117_696 + 5] = 50.0                      # classes 2 and 5 tie at the top
    Ws = torch.stack([perturbed(w, 9, 0.02), w_tie, w, w]).contiguous()
    L = nat.lib()
    ws = torch.empty(L.afl_cifar10_evaluate_workspace_bytes(4, n_test, m), dtype=torch.uint8, device="cuda")
    loss = torch.full((3, 4), -1.0, dtype=torch.float64, device="cuda")
    correct = torch.full((3, 4), -1, dtype=torch.int32, device="cuda")
    sets = i32([0, 0, -1, 1])                                           # n_sets = 1: problems 2 and 3 are out of range

    def run(slot):
        nat.check(L.afl_cifar10_evaluate(Ws.data_ptr(), 4, D, xte[None].data_ptr(), yte[None].data_ptr(), 1, n_test,
                                         sets.data_ptr(), m, slot.data_ptr(), 3, loss.data_ptr(), correct.data_ptr(),
                                         ws.data_ptr(), ws.numel(), torch.cuda.current_stream().cuda_stream))
        torch.cuda.synchronize()
    run(i32([3]))
    run(i32([-1]))
    assert bool((loss == -1).all()) and bool((correct == -1).all())
    run(i32([1]))
    assert bool((loss[[0, 2]] == -1).all()) and bool((correct[[0, 2]] == -1).all())   # only slot 1 is written
    assert bool((loss[1, 2:] == -1).all()) and bool((correct[1, 2:] == -1).all())
    for b in range(2):
        net = harness.Cifar10Net().cuda()
        harness.ParamLayout(net.parameters()).row_into_parameters(Ws[b], list(net.parameters()))
        crit = torch.nn.NLLLoss()
        want_loss, want_correct = 0.0, 0
        with torch.no_grad():
            for lo in range(0, n_test, m):                                    # harness.main's test loop
                out = net(xte[lo:lo + m])
                want_loss += crit(out, yte[lo:lo + m]).item()
                want_correct += int(out.max(1)[1].eq(yte[lo:lo + m]).sum())
            lp = net.double()(xte.double())
            top2 = lp.topk(2, dim=1).values
        if b == 1:
            assert want_correct == int((yte == 2).sum())                    # the first maximum: class 2
            assert int(correct[1, b]) == want_correct
        else:
            close = int(((top2[:, 0] - top2[:, 1]).abs() < 1e-4 * lp.abs().max(1).values.clamp(min=1)).sum())
            assert abs(int(correct[1, b]) - want_correct) <= close, (int(correct[1, b]), want_correct, close)
        assert float(loss[1, b]) == pytest.approx(want_loss, rel=1e-5)


def sweep_experiments():
    return [("Krum", 0.1, 1.0, 10, 0), ("TrimmedMean", 0.24, 0.5, 12, 1), ("Bulyan", 0.1, 1.5, 10, 0),
            ("NoDefense", 0.24, 2.0, 7, 1), ("Krum", 0.24, 3.0, 12, 0), ("NoDefense", 0.1, 0.0, 12, 0)]


def small_sweep(sweep, exps, epochs=6, capture=False):
    return sweep.Sweep(exps, epochs, batch_size=83, train_size=2000, test_size=500, test_step=5, capture=capture,
                       dataset="CIFAR10")


def test_captured_epochs_equal_eager_epochs(env, pinned_splits):
    _, _, sweep = env
    runs = []
    for capture in (False, True):
        sw = small_sweep(sweep, sweep_experiments(), epochs=7, capture=capture)
        for e in range(7):
            sw.step(e)
        torch.cuda.synchronize()
        runs.append(sw)
    a, b = runs
    assert a.D == D and a.x_train.shape[2:] == (3, 32, 32)
    for t in ("W", "V", "correct", "loss_sum", "epoch_counter", "test_slot"):
        x, y = getattr(a, t), getattr(b, t)
        assert torch.equal(x.view(torch.uint8), y.view(torch.uint8)), t
    assert int(b.epoch_counter) == 7 and int(b.test_slot) == 3
    assert not a.status().any()
    assert [r["accuracies"] for r in a.results()] == [r["accuracies"] for r in b.results()]


def test_failed_bulyan_experiment_leaves_the_others_alone(env, pinned_splits):
    _, _, sweep = env
    failing = ("Bulyan", 0.1, 1.0, 10, 0)
    others = [("Bulyan", 0.1, 1.5, 12, 1), ("TrimmedMean", 0.24, 1.0, 10, 0), ("Krum", 0.1, 0.5, 10, 1)]
    runs = []
    for exps in ([failing] + others, others):
        sw = small_sweep(sweep, exps, epochs=4, capture=True)
        sw.step(0)
        if len(exps) > len(others):
            sw.W[sw.order.index(0)] = float("nan")                          # every distance NaN: no eligible user
        for e in range(1, 4):
            sw.step(e)
        runs.append((sw, sw.results()))
    (a, ra), (b, rb) = runs
    assert isinstance(ra[0]["error"], KeyError) and ra[0]["error"].args == (-1,)
    for i in range(len(others)):
        assert ra[i + 1]["error"] is None and rb[i]["error"] is None
        pa, pb = a.order.index(i + 1), b.order.index(i)
        assert torch.equal(a.W[pa].view(torch.int32), b.W[pb].view(torch.int32)), others[i]
        assert ra[i + 1]["accuracies"] == rb[i]["accuracies"]


def test_n1000_problem_beside_n10_ones(env):
    """At 2000 training rows the N = 1000 clients hold two-row shards; its trajectory equals the one it has alone."""
    _, _, sweep = env
    big = ("TrimmedMean", 0.24, 0.5, 1000, 1)
    exps = [("NoDefense", 0.1, 1.0, 10, 0), big, ("TrimmedMean", 0.1, 1.5, 10, 1)]
    runs = []
    for grid in (exps, [big]):
        sw = small_sweep(sweep, grid, epochs=3, capture=True)
        for e in range(3):
            sw.step(e)
        runs.append((sw, sw.results()))
    (a, ra), (b, rb) = runs
    assert all(r["error"] is None for r in ra)
    assert a.N == 1000 and bool(torch.isfinite(a.W).all())
    assert torch.equal(a.W[a.order.index(1)].view(torch.int32), b.W[0].view(torch.int32))
    assert ra[1]["accuracies"] == rb[0]["accuracies"]


def harness_epoch0_weights(harness, malicious, e, batch_size, train_size, test_size):
    """harness.main's setup and its first epoch body (main.py:64-71) on CIFAR10: the weights before and after it."""
    from attacking_federate_learning_b200.server import AggregationServer
    defense, mal_prop, num_std, n, seed = e
    f = int(mal_prop * n)
    (xtr, ytr), _, net = harness.experiment_setup(seed, train_size, test_size, "cuda", "CIFAR10")
    layout = harness.ParamLayout(net.parameters())
    w0 = layout.flatten(list(net.parameters()))
    srv = AggregationServer(n, layout.dim, mal_prop, 0.1, 0.9, device="cuda", initial_weights=w0)
    users = [harness.Client(u, u < f, xtr[u::n], ytr[u::n], batch_size, layout, "cuda", "CIFAR10") for u in range(n)]
    for u in users:
        u.step(srv.current_weights, 0.1, srv.users_grads[u.user_id])
    malicious.DriftAttack(num_std).attack_rows(srv.users_grads, f)
    srv.defend(defense, 0)
    return w0, srv.current_weights


def test_first_weight_step_against_harness_main(env, tmp_path):
    _, harness, sweep = env
    from attacking_federate_learning_b200 import malicious
    exps = [("TrimmedMean", 0.24, 1.5, 10, 0), ("NoDefense", 0.24, 1.5, 10, 0), ("NoDefense", 0.0, 0.0, 10, 1)]
    kw = dict(batch_size=83, train_size=4000, test_size=500)
    sw = sweep.Sweep(exps, 1, capture=False, dataset="CIFAR10", **kw)
    sw.step(0)
    for i, e in enumerate(sw.experiments):
        w0, w = harness_epoch0_weights(harness, malicious, e, **kw)
        step = w.double() - w0.double()
        rel = float(((sw.W[i].double() - w0.double()) - step).norm() / step.norm())
        assert rel < 1e-3, (e, rel)
    # and the log files harness.main would write, named as it names them
    res = sweep.run(exps[:1], 2, out_dir=str(tmp_path), dataset="CIFAR10", **kw)
    assert os.path.basename(res[0]["csv"]).startswith("SYNTH-CIFAR10_stdev_1.5_TrimmedMean")


def test_learnability_at_the_harness_defaults(env, tmp_path):
    """synthetic_cifar_problem's docstring: NoDefense at the harness defaults reaches a best test accuracy of at
    least 40 % within 100 epochs for seeds 0 and 1."""
    _, _, sweep = env
    exps = [("NoDefense", 0.0, 0.0, 10, 0), ("NoDefense", 0.0, 0.0, 10, 1)]
    res = sweep.run(exps, 100, out_dir=str(tmp_path), dataset="CIFAR10", fading_rate=2000)
    for r in res:
        assert r["error"] is None
        assert max(r["accuracies"]) >= 40.0, (r["experiment"], r["accuracies"])
