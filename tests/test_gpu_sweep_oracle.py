"""The training-sweep kernels against float64 autograd and exact oracles where test_gpu_sweep.py and
test_gpu_sweep_backdoor.py do not reach (csrc/client_grad.cu, csrc/backdoor_train.cu, sweep.py).

1. Client gradients on shard-tail batches that leave whole 16-row groups empty (mb = 1 and mb = 16 (RT - 1) + 1), at
   1024 clients (2-row and 1-row shards) and at n = train_size (1-row shards), with rows_b = 0 and pitch sentinels,
   and at device epochs near 2^31; against float64 autograd per tensor and per fc1 hidden unit.
2. Partially non-finite weights (a NaN fc1 row or bias, an infinite fc1 weight, a NaN fc2 weight, an infinite fc2
   bias): the NaN and +-inf positions of fp32 autograd (harness.Client.step) entry by entry, the finite entries within
   the bound of float64 autograd, and the evaluation's correct count and NaN loss as harness.main's test loop gives.
3. The evaluation at every tile instance RT = 1 .. 8 with a one-row last batch, two data sets, out-of-range set
   indices and slots; exact ties go to the first maximum.
4. The backdoor trainer at alpha in {0, 0.5}, m in {1, 64, 200} and tails of 1, 31, 32, 33 and 199 rows against a
   float64 restatement; mal_epochs = 0; the backdoor test at m in {1, 64, 200} and its out-of-range guards.
5. Sweeps with N in {200, 1000} beside N = 10: captured epochs equal eager ones; a NaN fc1 row injected into one
   experiment gives harness.main's accuracy and leaves the other experiments' bits alone.
"""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from test_gpu_sweep import BOUND, SLICES, bad_fc1_units, i32, pinned_splits, sweep_experiments_large  # noqa: F401
from test_gpu_sweep_backdoor import FACTOR, FLOOR

pytestmark = pytest.mark.gpu

D, IN, HID = 79_510, 784, 100
LD = 79_520


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


def train_data(harness, seed, n_train):
    (x, y), _, net = harness.experiment_setup(seed, n_train, 10, "cuda")
    return x, y, harness.ParamLayout(net.parameters()).flatten(list(net.parameters()))


def eval_data(harness, seed, n_test):
    _, (x, y), net = harness.experiment_setup(seed, 10, n_test, "cuda")
    return x, y, harness.ParamLayout(net.parameters()).flatten(list(net.parameters()))


def noisy(w, seed, scale=0.01):
    return (w + scale * torch.randn(D, device="cuda", generator=torch.Generator("cuda").manual_seed(seed))).contiguous()


def client_grads(nat, W, x, y, data_index, rows, n, m, epoch, G):
    """W [B, D], x [n_sets, n_train, 784], G [B, N, ld] (written in place); synchronises."""
    nat.check(nat.lib().afl_mnist_client_grads(W.data_ptr(), W.shape[0], D, x.data_ptr(), y.data_ptr(), x.shape[0],
                                               x.shape[1], data_index.data_ptr(), rows.data_ptr(), n, m,
                                               epoch.data_ptr(), G.data_ptr(), G.stride(0), G.stride(1),
                                               torch.cuda.current_stream().cuda_stream))
    torch.cuda.synchronize()


def autograd(harness, w, xb, yb):
    """(fp32 autograd, float64 autograd) of NLLLoss(mean) through harness.MnistNet at the fp32 weights w."""
    out = []
    for dtype in (torch.float32, torch.float64):
        net = harness.MnistNet().to("cuda", dtype)
        layout = harness.ParamLayout(net.parameters())
        layout.row_into_parameters(w.to(dtype), list(net.parameters()))
        net.zero_grad()
        torch.nn.NLLLoss()(net(xb.to(dtype)), yb).backward()
        out.append(torch.cat([p.grad.reshape(-1) for p in net.parameters()]))
    return out[0], out[1]


def shard_rows(sweep, n_train, n, u, m, epoch):
    lo, hi = sweep.minibatch(n_train, n, u, m, epoch)
    return torch.arange(u + n * lo, u + n * hi, n, device="cuda")


def check_gradient(got, g32, g64, what):
    """NaN, +inf and -inf where fp32 autograd has them; the finite entries within BOUND of float64 autograd per tensor
    and per fc1 unit."""
    for f in (torch.isnan, torch.isposinf, torch.isneginf):
        a, b = f(got), f(g32)
        assert torch.equal(a, b), (what, f.__name__, int(a.sum()), int(b.sum()), int((a != b).sum()))
    fin = torch.isfinite(got)
    assert bool(torch.isfinite(g64[fin]).all()), what
    diff = torch.where(fin, got.double() - g64, 0.0)
    ref = torch.where(fin, g64, 0.0)
    for (a, b), name in zip(SLICES, ("fc1.weight", "fc1.bias", "fc2.weight", "fc2.bias")):
        e, r = float(diff[a:b].norm()), float(ref[a:b].norm())
        assert e <= BOUND * r, (what, name, e, r)
    bad = bad_fc1_units(diff, ref)
    assert not bad, (what, bad)


# ---------------------------------------------------------------------------------------------------------- gradients

@pytest.mark.parametrize("m, L, mb", [(128, 129, 1), (128, 241, 113), (40, 41, 1), (40, 73, 33)])
def test_tail_batches_with_empty_row_groups(env, m, L, mb):
    """Every client of n = 10 has an L-row shard (n_train = 10 L); epoch 1 takes the tail of mb rows."""
    nat, _, harness, sweep = env
    n, n_train = 10, 10 * L
    x, y, w = train_data(harness, 6, n_train)
    W = noisy(w, m + L)
    G = torch.full((1, n, LD), -3.0, device="cuda")
    client_grads(nat, W[None], x[None], y[None], i32([0]), i32([n]), n, m, i32([1]), G)
    for u in (0, 4, n - 1):
        idx = shard_rows(sweep, n_train, n, u, m, 1)
        assert len(idx) == mb
        g32, g64 = autograd(harness, W, x[idx], y[idx])
        check_gradient(G[0, u, :D], g32, g64, (m, L, u))
    assert bool(torch.isfinite(G[0, :, :D]).all())
    assert bool((G[0, :, D:] == -3.0).all())


def test_1024_clients_with_two_and_one_row_shards(env):
    """n = 1024 of 2000 rows: clients u < 976 hold 2 rows, the others 1.  Problem 1 has no client, problem 2 has 700,
    so rows u >= n_b and the pitch columns keep their sentinel."""
    nat, _, harness, sweep = env
    n_train, N, m = 2000, 1024, 83
    x, y, w = train_data(harness, 7, n_train)
    W = torch.stack([noisy(w, 1), noisy(w, 2), noisy(w, 3)]).contiguous()
    rows = [N, 0, 700]
    G = torch.full((3, N, LD), -3.0, device="cuda")
    client_grads(nat, W, x[None], y[None], i32([0, 0, 0]), i32(rows), N, m, i32([0]), G)
    for u in (0, 1, 975, 976, 977, 1023):
        idx = shard_rows(sweep, n_train, N, u, m, 0)
        assert len(idx) == (2 if u < 976 else 1), u
        g32, g64 = autograd(harness, W[0], x[idx], y[idx])
        check_gradient(G[0, u, :D], g32, g64, u)
    for u in (0, 699):
        idx = shard_rows(sweep, n_train, 700, u, m, 0)
        g32, g64 = autograd(harness, W[2], x[idx], y[idx])
        check_gradient(G[2, u, :D], g32, g64, (700, u))
    for b, n in enumerate(rows):
        assert bool(torch.isfinite(G[b, :n, :D]).all()), b
        assert bool((G[b, n:] == -3.0).all()), b
        assert bool((G[b, :, D:] == -3.0).all()), b


@pytest.mark.parametrize("m", [1, 83])
def test_one_row_shards_at_n_equal_train_size(env, m):
    nat, _, harness, sweep = env
    n = n_train = 1000
    x, y, w = train_data(harness, 8, n_train)
    W = noisy(w, m)
    G = torch.full((1, n, LD), -3.0, device="cuda")
    client_grads(nat, W[None], x[None], y[None], i32([0]), i32([n]), n, m, i32([5]), G)
    for u in (0, 499, 999):
        idx = shard_rows(sweep, n_train, n, u, m, 5)
        assert idx.tolist() == [u]
        g32, g64 = autograd(harness, W, x[idx], y[idx])
        check_gradient(G[0, u, :D], g32, g64, u)
    assert bool(torch.isfinite(G[0, :, :D]).all())
    assert bool((G[0, :, D:] == -3.0).all())


@pytest.mark.parametrize("m, epoch", [(83, 2**31 - 1), (83, 10**6 + 7), (64, 2**31 - 1), (64, 10**6 + 7)])
def test_large_device_epoch(env, m, epoch):
    """n = 10 of 2000 rows: every shard has L = 200 rows, so epoch e takes batch e mod ceil(200 / m) everywhere."""
    nat, _, harness, sweep = env
    n, n_train = 10, 2000
    x, y, w = train_data(harness, 9, n_train)
    W = noisy(w, epoch % 1000)
    q = (200 + m - 1) // m
    G, Gr = (torch.full((1, n, LD), -3.0, device="cuda") for _ in range(2))
    client_grads(nat, W[None], x[None], y[None], i32([0]), i32([n]), n, m, i32([epoch]), G)
    client_grads(nat, W[None], x[None], y[None], i32([0]), i32([n]), n, m, i32([epoch % q]), Gr)
    assert torch.equal(G.view(torch.int32), Gr.view(torch.int32))
    for u in (0, n - 1):
        assert sweep.minibatch(n_train, n, u, m, epoch) == sweep.minibatch(n_train, n, u, m, epoch % q)
        idx = shard_rows(sweep, n_train, n, u, m, epoch)
        g32, g64 = autograd(harness, W, x[idx], y[idx])
        check_gradient(G[0, u, :D], g32, g64, u)


def poison(w, case):
    """experiment_setup weights with one non-finite entry or row."""
    w = w.clone()
    if case == "fc1_row_nan":
        w[98 * IN:99 * IN] = float("nan")                   # a unit of the fc1 weight gradient's c = 3 path
    elif case == "fc1_bias_nan":
        w[78_400 + 3] = float("nan")
    elif case == "fc1_weight_inf":
        w[40 * IN + 300] = float("inf")                     # +inf or 0 activations: the inputs have no zeros
    elif case == "fc2_weight_nan":
        w[78_500 + 4 * HID + 10] = float("nan")
    elif case == "fc2_bias_inf":
        w[79_500 + 6] = float("inf")
    return w


NONFINITE = ["fc1_row_nan", "fc1_bias_nan", "fc1_weight_inf", "fc2_weight_nan", "fc2_bias_inf"]


@pytest.mark.parametrize("case", NONFINITE)
def test_nonfinite_weights_gradient(env, case):
    nat, _, harness, sweep = env
    n, n_train, m = 10, 2000, 83
    x, y, w = train_data(harness, 0, n_train)
    W = poison(w, case)
    G = torch.full((1, n, LD), -3.0, device="cuda")
    client_grads(nat, W[None], x[None], y[None], i32([0]), i32([n]), n, m, i32([0]), G)
    for u in (0, 5, n - 1):
        idx = shard_rows(sweep, n_train, n, u, m, 0)
        g32, g64 = autograd(harness, W, x[idx], y[idx])
        got = G[0, u, :D]
        check_gradient(got, g32, g64, (case, u))
        assert bool(torch.isnan(got).any()), (case, u)
        c = harness.Client(u, False, x[u::n], y[u::n], m, harness.ParamLayout(harness.MnistNet().parameters()), "cuda")
        row = torch.empty(D, device="cuda")
        c.step(W, 0.1, row)                                  # the harness's client is fp32 autograd
        assert torch.equal(torch.isnan(row), torch.isnan(got)), (case, u)
        if case == "fc1_weight_inf":                         # +inf activations on some rows, 0 on the others
            assert bool((x[idx, 300] > 0).any()) and bool((x[idx, 300] < 0).any())
    assert bool((G[0, :, D:] == -3.0).all())


# --------------------------------------------------------------------------------------------------------- evaluation

def evaluate(nat, W, X, Y, sets, m, slot, loss, correct):
    """afl_mnist_evaluate into the tables loss [n_slots, B] and correct [n_slots, B]; synchronises."""
    L = nat.lib()
    B, n_test = W.shape[0], X.shape[1]
    ws = torch.empty(L.afl_mnist_evaluate_workspace_bytes(B, n_test, m), dtype=torch.uint8, device="cuda")
    sets, slot = i32(sets), i32([slot])
    nat.check(L.afl_mnist_evaluate(W.data_ptr(), B, D, X.data_ptr(), Y.data_ptr(), X.shape[0], n_test,
                                   sets.data_ptr(), m, slot.data_ptr(), loss.shape[0], loss.data_ptr(),
                                   correct.data_ptr(), ws.data_ptr(), ws.numel(), torch.cuda.current_stream().cuda_stream))
    torch.cuda.synchronize()


def harness_test_loop(harness, w, xte, yte, m):
    """harness.main's test loop at the weights w: (loss sum, correct count, rows whose float64 top-2 margin is too
    close to call)."""
    net = harness.MnistNet().cuda()
    harness.ParamLayout(net.parameters()).row_into_parameters(w, list(net.parameters()))
    crit = torch.nn.NLLLoss()
    loss, correct = 0.0, 0
    with torch.no_grad():
        for lo in range(0, len(xte), m):
            out = net(xte[lo:lo + m])
            loss += crit(out, yte[lo:lo + m]).item()
            correct += int(out.max(1)[1].eq(yte[lo:lo + m]).sum())
        lp = net.double()(xte.double())
        top2 = lp.topk(2, dim=1).values
        margin = (top2[:, 0] - top2[:, 1]).abs()
    close = int((margin < 1e-4 * lp.abs().max(1).values.clamp(min=1)).sum())       # NaN rows are never close
    return loss, correct, close


def table(B, fill=-1):
    return (torch.full((3, B), float(fill), dtype=torch.float64, device="cuda"),
            torch.full((3, B), fill, dtype=torch.int32, device="cuda"))


@pytest.mark.parametrize("m", [16, 17, 32, 33, 48, 49, 64, 65, 80, 81, 96, 97, 112, 113, 127, 128])
def test_evaluation_every_tile_instance(env, m):
    """n_test = q m + 1: the last batch has one row.  Problems 4 and 5 name no set; slots -1 and 3 write nothing."""
    nat, _, harness, _ = env
    n_test = m * ((300 + m - 1) // m) + 1
    x0, y0, w0 = eval_data(harness, 0, n_test)
    x1, y1, w1 = eval_data(harness, 1, n_test)
    X, Y = torch.stack([x0, x1]).contiguous(), torch.stack([y0, y1]).contiguous()
    sets = [0, 1, 1, 0, 2, -1]
    W = torch.stack([noisy(w0, m, 0.0), noisy(w1, m), noisy(w1, m + 1, 0.03), noisy(w0, m + 2, 0.05),
                     w0, w1]).contiguous()
    loss, correct = table(6)
    evaluate(nat, W, X, Y, sets, m, 1, loss, correct)
    assert bool((loss[[0, 2]] == -1).all()) and bool((correct[[0, 2]] == -1).all())
    assert bool((loss[1, 4:] == -1).all()) and bool((correct[1, 4:] == -1).all())
    for b in range(4):
        want_loss, want_correct, close = harness_test_loop(harness, W[b], X[sets[b]], Y[sets[b]], m)
        assert abs(int(correct[1, b]) - want_correct) <= close, (b, int(correct[1, b]), want_correct, close)
        assert float(loss[1, b]) == pytest.approx(want_loss, rel=1e-5), b
    before = loss.clone(), correct.clone()
    for slot in (-1, 3):
        evaluate(nat, W, X, Y, sets, m, slot, loss, correct)
        assert torch.equal(loss, before[0]) and torch.equal(correct, before[1]), slot


@pytest.mark.parametrize("m", [1, 83])
def test_evaluation_exact_tie_takes_the_first_maximum(env, m):
    nat, _, harness, _ = env
    xte, yte, w = eval_data(harness, 2, 500)
    w = w.clone()
    w[78_500:79_500] = 0.0                                   # fc2.weight = 0: every row's logits are fc2.bias
    w[79_500:] = 0.0
    w[79_500 + 3] = w[79_500 + 7] = 0.75
    loss, correct = table(1)
    evaluate(nat, w[None].contiguous(), xte[None], yte[None], [0], m, 0, loss, correct)
    want_loss, want_correct, _ = harness_test_loop(harness, w, xte, yte, m)
    assert int(correct[0, 0]) == want_correct == int((yte == 3).sum())
    assert float(loss[0, 0]) == pytest.approx(want_loss, rel=1e-5)


@pytest.mark.parametrize("case", NONFINITE)
def test_nonfinite_weights_evaluation(env, case):
    nat, _, harness, _ = env
    m = 83
    xte, yte, w = eval_data(harness, 0, 500)
    W = torch.stack([poison(w, case), w]).contiguous()
    loss, correct = table(2)
    evaluate(nat, W, xte[None], yte[None], [0, 0], m, 2, loss, correct)
    for b in range(2):
        want_loss, want_correct, close = harness_test_loop(harness, W[b], xte, yte, m)
        got = int(correct[2, b])
        assert abs(got - want_correct) <= close, (case, b, got, want_correct, close)
        assert np.isnan(float(loss[2, b])) == np.isnan(want_loss), (case, b, float(loss[2, b]), want_loss)
        if not np.isnan(want_loss):
            assert float(loss[2, b]) == pytest.approx(want_loss, rel=1e-5)
    if case in ("fc1_row_nan", "fc1_bias_nan", "fc2_weight_nan"):  # NaN log-probabilities everywhere: class 0
        assert int(correct[2, 0]) == int((yte == 0).sum())


# --------------------------------------------------------------------------------------------------- backdoor trainer

def run_trainer(nat, initial, sets, index, m, alpha, epochs):
    B = initial.shape[0]
    xs, ys, lens = sets
    f, z = i32([1] * B), torch.ones(B, dtype=torch.float64, device="cuda")
    status = i32([0] * B)
    out = torch.full_like(initial, -7.25)
    index = i32(index)
    nat.check(nat.lib().afl_mnist_backdoor_train(initial.data_ptr(), out.data_ptr(), B, D, xs.data_ptr(), ys.data_ptr(),
                                                 xs.shape[0], xs.shape[1], lens.data_ptr(), index.data_ptr(),
                                                 f.data_ptr(), z.data_ptr(), status.data_ptr(), alpha, epochs, m,
                                                 torch.cuda.current_stream().cuda_stream))
    torch.cuda.synchronize()
    return out, status


def train64(harness, layout, x, y, initial, alpha, epochs, m):
    """BackdoorTrainer.train in float64 with minibatches of m rows (a fresh optimiser per minibatch)."""
    net = harness.MnistNet().to("cuda", torch.float64)
    params = list(net.parameters())
    layout.row_into_parameters(initial.double(), params)
    p0 = [p.detach().clone() for p in params]
    x = x.double()
    for _ in range(epochs):
        for lo in range(0, len(x), m):
            opt = torch.optim.SGD(params, lr=0.1, momentum=0.9, weight_decay=0.0001)
            opt.zero_grad()
            loss = F.nll_loss(net(x[lo:lo + m]), y[lo:lo + m])
            if alpha > 0:
                loss = loss + alpha * sum(F.mse_loss(p, q) for p, q in zip(params, p0))
            loss.backward()
            opt.step()
    return torch.cat([p.detach().reshape(-1) for p in params])


def cut_set(harness, seed, n):
    """The first n rows of the pattern set of a 2000-row training set, as the trainer's (x, y, len) and the rows."""
    x, y, w = train_data(harness, seed, 2000)
    bx, by = harness.backdoor_set("pattern", x, y, seed)
    bx, by = bx[:n].contiguous(), by[:n].contiguous()
    return (bx[None].contiguous(), by[None].contiguous(), i32([n])), bx, by, w, x, y


@pytest.mark.parametrize("alpha, m, n", [(0.0, 1, 7), (0.5, 1, 5), (0.0, 64, 129), (0.5, 64, 95), (0.0, 64, 96),
                                         (0.5, 64, 97), (0.5, 200, 201), (0.0, 200, 399), (0.5, 200, 200)])
def test_trainer_against_float64_at_every_tail(env, alpha, m, n):
    """Tails of n mod m rows: 1, 31, 32, 33, 199 and a whole batch; m = 1 on a short set."""
    nat, _, harness, _ = env
    epochs = 2 if m == 1 else 3
    sets, bx, by, w, x, y = cut_set(harness, 4, n)
    layout = harness.ParamLayout(harness.MnistNet().parameters())
    g = torch.Generator(device="cuda").manual_seed(n)
    initials = torch.stack([w, w + 0.03 * torch.randn(D, device="cuda", generator=g)]).contiguous()
    got, status = run_trainer(nat, initials, sets, [0, 0], m, alpha, epochs)
    assert status.cpu().tolist() == [0, 0]
    for b in range(2):
        tr = harness.BackdoorTrainer("pattern", alpha, epochs, layout, x, y, "cuda", lambda *a, **k: None, 4, m)
        tr.x, tr.y = bx, by
        init = initials[b].clone()
        a32 = tr.train(init)
        assert a32 is not init                                                  # not 100 % before: it trains
        r64 = train64(harness, layout, bx, by, initials[b], alpha, epochs, m)
        scale = torch.linalg.norm(r64 - initials[b].double())
        assert scale > 1e-4
        e_k = float(torch.linalg.norm(got[b].double() - r64) / scale)
        e_a = float(torch.linalg.norm(a32.double() - r64) / scale)
        assert e_k <= FACTOR * e_a + FLOOR, (alpha, m, n, b, e_k, e_a)


@pytest.mark.parametrize("alpha, m", [(4.0, 200), (0.0, 1), (0.5, 64)])
def test_trainer_zero_epochs_returns_initial(env, alpha, m):
    nat, _, harness, _ = env
    sets, _, _, w, _, _ = cut_set(harness, 5, 233)
    initials = torch.stack([w, noisy(w, 3, 0.05)]).contiguous()
    got, status = run_trainer(nat, initials, sets, [0, 0], m, alpha, 0)
    assert status.cpu().tolist() == [0, 0]
    assert torch.equal(got.view(torch.int32), initials.view(torch.int32))


@pytest.mark.parametrize("m", [1, 64, 200])
def test_backdoor_test_against_post_and_its_guards(env, m):
    """Problems 0..2 on a 233-row set; problem 3's set is longer than max_len, problems 4 and 5 name no set; slots -1
    and 3 write nothing."""
    nat, _, harness, _ = env
    n = 233
    (xs, ys, _), bx, by, w, x, y = cut_set(harness, 2, n)
    layout = harness.ParamLayout(harness.MnistNet().parameters())
    trained, _ = run_trainer(nat, torch.stack([w, noisy(w, 4, 0.02)]).contiguous(), (xs, ys, i32([n])), [0, 0],
                             200, 4.0, 1)
    W = torch.stack([w, trained[0], trained[1], w, w, w]).contiguous()
    X, Y = torch.cat([xs, xs]).contiguous(), torch.cat([ys, ys]).contiguous()
    lens, index = i32([n, n + 1]), i32([0, 0, 0, 1, 2, -1])
    loss, correct = table(6)

    def call(slot):
        sl = i32([slot])
        nat.check(nat.lib().afl_mnist_backdoor_test(W.data_ptr(), 6, D, X.data_ptr(), Y.data_ptr(), 2, n,
                                                    lens.data_ptr(), index.data_ptr(), m, sl.data_ptr(), 3,
                                                    loss.data_ptr(), correct.data_ptr(),
                                                    torch.cuda.current_stream().cuda_stream))
        torch.cuda.synchronize()
    call(1)
    assert bool((loss[[0, 2]] == -1).all()) and bool((correct[[0, 2]] == -1).all())
    assert bool((loss[1, 3:] == -1).all()) and bool((correct[1, 3:] == -1).all())
    for b in range(3):
        tr = harness.BackdoorTrainer("pattern", 4, 5, layout, x, y, "cuda", lambda *a, **k: None, 2, m)
        tr.x, tr.y = bx, by
        layout.row_into_parameters(W[b], list(tr.net.parameters()))
        assert 100. * int(correct[1, b]) / n == tr.test("POST", to_print=False), b
        want = 0.0
        with torch.no_grad():
            for lo in range(0, n, m):
                want += F.nll_loss(tr.net(bx[lo:lo + m]), by[lo:lo + m]).item()
        assert abs(float(loss[1, b]) - want) <= 1e-5 * max(1.0, abs(want)), (b, float(loss[1, b]), want)
    before = loss.clone(), correct.clone()
    for slot in (-1, 3):
        call(slot)
        assert torch.equal(loss, before[0]) and torch.equal(correct, before[1]), slot


# ------------------------------------------------------------------------------------------------------------- sweeps

def test_large_grid_captured_epochs_equal_eager(env, pinned_splits):
    _, _, _, sweep = env
    runs = []
    for capture in (False, True):
        sw = sweep.Sweep(sweep_experiments_large(), 3, batch_size=83, train_size=2000, test_size=500, test_step=2,
                         capture=capture)
        assert sw.N == 1000
        for e in range(3):
            sw.step(e)
        torch.cuda.synchronize()
        runs.append(sw)
    a, b = runs
    for t in ("W", "V", "correct", "loss_sum", "epoch_counter", "test_slot"):
        assert torch.equal(getattr(a, t).view(torch.uint8), getattr(b, t).view(torch.uint8)), t
    assert not a.status().any() and not b.status().any()
    assert bool(torch.isfinite(a.W).all())


def test_nan_unit_in_one_experiment(env, pinned_splits):
    """One fc1 row of experiment 0 (NoDefense) set to NaN after epoch 0: its recorded accuracy is harness.main's test
    loop on its final weights, and the other experiments keep their bits."""
    _, _, harness, sweep = env
    exps = [("NoDefense", 0.24, 1.0, 10, 0), ("TrimmedMean", 0.24, 1.0, 10, 0), ("NoDefense", 0.1, 1.5, 12, 1),
            ("Krum", 0.1, 0.5, 10, 1)]
    runs = []
    for inject in (True, False):
        sw = sweep.Sweep(exps, 3, batch_size=83, train_size=2000, test_size=500, test_step=1, capture=True)
        sw.step(0)
        if inject:
            i = sw.order.index(0)
            sw.W[i, 37 * IN:38 * IN] = float("nan")
        for e in range(1, 3):
            sw.step(e)
        torch.cuda.synchronize()
        runs.append(sw)
    a, b = runs
    i = a.order.index(0)
    xte, yte = a.x_test[int(a.data_index[i])], a.y_test[int(a.data_index[i])]
    _, want_correct, close = harness_test_loop(harness, a.W[i], xte, yte, 83)
    assert abs(int(a.correct[2, i]) - want_correct) <= close, (int(a.correct[2, i]), want_correct, close)
    assert np.isnan(float(a.loss_sum[2, i]))
    assert int(a.correct[1, i]) == int(a.correct[2, i]) == int((yte == 0).sum())  # NaN log-probabilities: class 0
    for k in range(1, len(exps)):
        pa, pb = a.order.index(k), b.order.index(k)
        assert torch.equal(a.W[pa].view(torch.int32), b.W[pb].view(torch.int32)), exps[k]
        assert torch.equal(a.correct[:, pa], b.correct[:, pb]), exps[k]
        assert torch.equal(a.loss_sum[:, pa].view(torch.int64), b.loss_sum[:, pb].view(torch.int64)), exps[k]
