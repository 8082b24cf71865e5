"""The training sweep on an H100 (sweep.py, csrc/client_grad.cu).

1. Client gradients against float64 autograd of harness.MnistNet on the same fp32 weights and rows, at m in
   {1, 7, 83, 128} and on a shard-tail batch, and against fp32 torch autograd (harness.Client.step), within one
   per-tensor bound; zero pre-activations get a zero derivative.
2. A client's gradient is bit-identical at B = 1 and inside a large ragged batch whose other problems hold NaN
   weights; pitch columns and rows past n_b keep a sentinel.
3. Evaluation against harness.main's test loop on the same weights.
4. The epoch chain after the kernel (ALIE, every rule, the momentum step) equals the host-parameter batched calls, at
   N <= 12 and on a grid with N = 200 and 1000.
5. Captured epochs equal eager epochs bit for bit.
6. End to end against harness.main; a failing Bulyan experiment leaves the others' bits alone.
"""
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

D, IN = 79_510, 784
SPLITS = "4"
# Per-tensor bound ||g - g64|| / ||g64||.  Each gradient entry is a product of fp32 dot products of at most K = 784
# terms (fc1), then sums over at most 128 rows; the worst-case relative error of a K-term fp32 dot product is
# gamma_K = K u / (1 - K u) ~ 4.7e-5 (u = 2^-24) relative to the sum of |terms|, and the backward adds gamma_128 and
# the softmax's few ulps.  Rounding errors are not all of one sign, so the norm-wise error is far below the sum of the
# worst cases; 1e-4 sits above the worst case of the forward alone and stays five orders of magnitude below an error
# that changes the training (a wrong row, a wrong sign or a missing 1/m term is O(1)).
BOUND = 1e-4


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


def data(harness, seed, n_train=2000, n_test=500):
    (xtr, ytr), (xte, yte), net = harness.experiment_setup(seed, n_train, n_test, "cuda")
    w = harness.ParamLayout(net.parameters()).flatten(list(net.parameters()))
    return xtr, ytr, xte, yte, w


def i32(v):
    return torch.as_tensor(np.asarray(v, np.int32), device="cuda")


def client_grads(nat, W, x, y, data_index, rows, n, m, epoch, G):
    """G: [B, n, ld] fp32 (written in place)."""
    nat.check(nat.lib().afl_mnist_client_grads(W.data_ptr(), W.shape[0], D, x.data_ptr(), y.data_ptr(), x.shape[0],
                                               x.shape[1], data_index.data_ptr(), rows.data_ptr(), n, m,
                                               epoch.data_ptr(), G.data_ptr(), G.stride(0), G.stride(1),
                                               torch.cuda.current_stream().cuda_stream))


def autograd(harness, w, xb, yb, dtype):
    net = harness.MnistNet().to("cuda", dtype)
    layout = harness.ParamLayout(net.parameters())
    layout.row_into_parameters(w.to(dtype), list(net.parameters()))
    net.zero_grad()
    torch.nn.NLLLoss()(net(xb.to(dtype)), yb).backward()
    return layout.flatten([p.grad.to(torch.float32) for p in net.parameters()]), \
        layout.flatten([p.grad.double() for p in net.parameters()], out=torch.empty(D, dtype=torch.float64, device="cuda"))


SLICES = [(0, 78_400), (78_400, 78_500), (78_500, 79_500), (79_500, D)]          # fc1.w, fc1.b, fc2.w, fc2.b
# fc1 is also checked per hidden unit, against BOUND * max(||ref_j||, UNIT_FLOOR * ||ref_fc1||), so that an error
# confined to a few units (the weight gradient's units 96..99 take a path of their own) cannot hide in the tensor norm.
UNIT_FLOOR = 1e-2


def rel_errors(g, ref):
    return [float((g[a:b].double() - ref[a:b]).norm() / ref[a:b].norm()) for a, b in SLICES]


def bad_fc1_units(diff, ref):
    """The hidden units whose fc1 error norm exceeds the per-unit bound (diff = g - ref, both float64 [D])."""
    e = diff[:78_400].view(100, IN).norm(dim=1)
    allow = BOUND * torch.maximum(ref[:78_400].view(100, IN).norm(dim=1), UNIT_FLOOR * ref[:78_400].norm())
    return (e > allow).nonzero().flatten().tolist()


# every tile instance RT = ceil(m / 16) at each row-group boundary, for the first and the last client
ROW_GROUP_EDGES = [16, 17, 32, 33, 48, 49, 64, 65, 80, 81, 96, 97, 112, 113, 127, 128]


@pytest.mark.parametrize("m, n, epoch, u", [(1, 10, 3, 4), (7, 10, 5, 9), (83, 10, 0, 0), (83, 10, 2, 3),
                                            (128, 10, 1, 7), (83, 7, 3, 6)] +
                         [(m, 10, e, u) for m in ROW_GROUP_EDGES for e, u in ((0, 0), (3, 9))])
def test_gradient_against_float64_and_fp32_autograd(env, m, n, epoch, u):
    """(83, 7, 3, 6): shard length 285 (2000 rows, 7 users), positions 249..284, a 36-row tail batch.  fc1 is also
    checked per hidden unit (units 96..99 take a path of their own in the weight gradient)."""
    nat, _, harness, sweep = env
    xtr, ytr, _, _, w = data(harness, 1)
    W = (w + 0.01 * torch.randn(D, device="cuda", generator=torch.Generator("cuda").manual_seed(m))).contiguous()
    G = torch.full((1, n, 79_520), 7.0, device="cuda")
    client_grads(nat, W[None], xtr[None], ytr[None], i32([0]), i32([n]), n, m, i32([epoch]), G)
    lo, hi = sweep.minibatch(len(xtr), n, u, m, epoch)
    if (m, n) == (83, 7):
        assert (lo, hi) == (249, 285)
    idx = torch.arange(u + n * lo, u + n * hi, n, device="cuda")
    g32, _ = autograd(harness, W, xtr[idx], ytr[idx], torch.float32)
    _, g64 = autograd(harness, W, xtr[idx], ytr[idx], torch.float64)
    got = G[0, u, :D]
    assert all(e < BOUND for e in rel_errors(got, g64)), rel_errors(got, g64)
    assert all(e < BOUND for e in rel_errors(g32, g64)), rel_errors(g32, g64)        # torch's fp32 sits inside too
    assert all(e < 2 * BOUND for e in rel_errors(got, g32.double()))
    assert not bad_fc1_units(got.double() - g64, g64)
    # the client through the harness itself
    c = harness.Client(u, False, xtr[u::n], ytr[u::n], m, harness.ParamLayout(harness.MnistNet().parameters()), "cuda")
    for _ in range(epoch):
        c.pos = c.pos + m if c.pos + m < len(c.x) else 0
    row = torch.empty(D, device="cuda")
    c.step(W, 0.1, row)
    assert torch.equal(row, g32)


def test_zero_preactivations_get_a_zero_derivative(env):
    nat, _, harness, sweep = env
    xtr, ytr, _, _, w = data(harness, 2)
    W = w.clone()
    dead = [0, 17, 99]
    for j in dead:
        W[j * IN:(j + 1) * IN] = 0.0
        W[78_400 + j] = 0.0
    G = torch.zeros((1, 10, 79_520), device="cuda")
    client_grads(nat, W[None], xtr[None], ytr[None], i32([0]), i32([10]), 10, 83, i32([0]), G)
    g = G[0, 3, :D]
    lo, hi = sweep.minibatch(len(xtr), 10, 3, 83, 0)
    g32, g64 = autograd(harness, W, xtr[3 + 10 * lo:3 + 10 * hi:10], ytr[3 + 10 * lo:3 + 10 * hi:10], torch.float32)
    for j in dead:
        assert torch.equal(g[j * IN:(j + 1) * IN], torch.zeros(IN, device="cuda"))
        assert float(g[78_400 + j]) == 0.0 and float(g32[78_400 + j]) == 0.0
        assert torch.equal(g32[j * IN:(j + 1) * IN], torch.zeros(IN, device="cuda"))
    assert float(g.abs().sum()) > 0


def test_batch_composition_does_not_change_a_gradient(env):
    nat, _, harness, _ = env
    x0, y0, _, _, w0 = data(harness, 3)
    x1, y1, _, _, w1 = data(harness, 4)
    X, Y = torch.stack([x0, x1]), torch.stack([y0, y1])
    ld = 79_552
    # alone: problem (set 1, n = 10)
    G1 = torch.full((1, 10, ld), -3.0, device="cuda")
    client_grads(nat, w1[None].contiguous(), X, Y, i32([1]), i32([10]), 10, 83, i32([4]), G1)
    # inside B = 37 with N = 130: ragged rows, NaN weights elsewhere, problem 21 is the one above
    B, N = 37, 130
    W = torch.full((B, D), float("nan"), device="cuda")
    W[21] = w1
    W[5] = w0
    rows = [((b * 7) % N) + 1 for b in range(B)]
    rows[21], rows[5] = 10, 130
    sets = [b % 2 for b in range(B)]
    sets[21], sets[5] = 1, 0
    G = torch.full((B, N, ld), -3.0, device="cuda")
    client_grads(nat, W, X, Y, i32(sets), i32(rows), N, 83, i32([4]), G)
    torch.cuda.synchronize()
    assert torch.equal(G[21, :10, :D].view(torch.int32), G1[0, :, :D].view(torch.int32))
    sentinel = torch.tensor(-3.0, device="cuda")
    for b in range(B):
        assert bool((G[b, rows[b]:] == sentinel).all()), b                   # rows u >= n_b untouched
        assert bool((G[b, :, D:] == sentinel).all()), b                      # pitch columns untouched
    assert bool(torch.isfinite(G[5, :130, :D]).all())
    G5 = torch.full((1, 130, ld), -3.0, device="cuda")
    client_grads(nat, w0[None].contiguous(), X, Y, i32([0]), i32([130]), 130, 83, i32([4]), G5)
    assert torch.equal(G[5, :, :D].view(torch.int32), G5[0, :, :D].view(torch.int32))


@pytest.mark.parametrize("m", [83, 128])
def test_evaluation_against_the_harness_test_loop(env, m):
    nat, _, harness, _ = env
    n_test = 1000
    _, _, xte, yte, w = data(harness, 5, n_test=n_test)
    Ws = torch.stack([w, w + 0.02 * torch.randn(D, device="cuda")]).contiguous()
    L = nat.lib()
    ws = torch.empty(L.afl_mnist_evaluate_workspace_bytes(2, n_test, m), dtype=torch.uint8, device="cuda")
    loss = torch.full((3, 2), -1.0, dtype=torch.float64, device="cuda")
    correct = torch.full((3, 2), -1, dtype=torch.int32, device="cuda")
    sets, slot = i32([0, 0]), i32([1])                 # held until the kernels have read them
    nat.check(L.afl_mnist_evaluate(Ws.data_ptr(), 2, D, xte[None].data_ptr(), yte[None].data_ptr(), 1, n_test,
                                   sets.data_ptr(), m, slot.data_ptr(), 3, loss.data_ptr(),
                                   correct.data_ptr(), ws.data_ptr(), ws.numel(), torch.cuda.current_stream().cuda_stream))
    assert bool((loss[[0, 2]] == -1).all()) and bool((correct[[0, 2]] == -1).all())     # only slot 1 is written
    for b in range(2):
        net = harness.MnistNet().cuda()
        harness.ParamLayout(net.parameters()).row_into_parameters(Ws[b], list(net.parameters()))
        crit = torch.nn.NLLLoss()
        want_loss, want_correct = 0.0, 0
        with torch.no_grad():
            for lo in range(0, n_test, m):                                    # harness.main's test loop
                out = net(xte[lo:lo + m])
                want_loss += crit(out, yte[lo:lo + m]).item()
                want_correct += int(out.max(1)[1].eq(yte[lo:lo + m]).sum())
            net64 = net.double()
            lp = net64(xte.double())
            top2 = lp.topk(2, dim=1).values
            margin = (top2[:, 0] - top2[:, 1]).abs()
        # a logit is a 784-term then a 100-term fp32 dot product: |error| <= ~1e-4 relative to the logit scale here
        close = int((margin < 1e-4 * lp.abs().max(1).values.clamp(min=1)).sum())
        assert abs(int(correct[1, b]) - want_correct) <= close, (int(correct[1, b]), want_correct, close)
        assert float(loss[1, b]) == pytest.approx(want_loss, rel=1e-5)


def sweep_experiments():
    return [("Krum", 0.1, 1.0, 10, 0), ("TrimmedMean", 0.24, 0.5, 12, 1), ("Bulyan", 0.1, 1.5, 10, 0),
            ("NoDefense", 0.24, 2.0, 7, 1), ("Krum", 0.24, 3.0, 12, 0), ("TrimmedMean", 0.0, 1.0, 10, 0),
            ("Bulyan", 0.0, 0.25, 7, 1), ("NoDefense", 0.1, 0.0, 12, 0)]


def small_sweep(sweep, exps, epochs=6, capture=False):
    return sweep.Sweep(exps, epochs, batch_size=83, train_size=2000, test_size=500, test_step=5, capture=capture)


def sweep_experiments_large():
    """N = 200 and 1000 beside N = 10: every DeviceRound takes the large path; at 2000 training rows the N = 1000
    clients hold two-row shards."""
    return [("Krum", 0.1, 1.0, 200, 0), ("TrimmedMean", 0.24, 0.5, 1000, 1), ("Bulyan", 0.1, 1.5, 200, 0),
            ("NoDefense", 0.24, 2.0, 1000, 0), ("Krum", 0.24, 3.0, 10, 1), ("Bulyan", 0.0, 0.25, 10, 0),
            ("TrimmedMean", 0.1, 1.0, 10, 0), ("NoDefense", 0.1, 0.0, 200, 1)]


def test_epoch_chain_equals_host_parameter_calls(env, pinned_splits):
    nat, bt, harness, sweep = env
    from attacking_federate_learning_b200._device import momentum_step
    for grid in (sweep_experiments(), sweep_experiments_large()):
        sw = small_sweep(sweep, grid)
        for _ in range(2):                                                   # a second epoch on moved weights
            sw.client_grads()
            G0, W0, V0 = sw._storage.clone(), sw.W.clone(), sw.V.clone()
            sw.aggregate()
            sw.epoch_counter.add_(1)
            for r, (sl, _) in sw.rounds.items():
                exps = sw.experiments[sl]
                fs = [e.corrupted_count for e in exps]
                zs = [e.num_std for e in exps]
                rows = [e.users_count for e in exps]
                G = G0[sl, :, :D]
                bt.alie_rows(G, fs, zs)
                agg = bt.defend[r](G, None, fs, rows=rows)
                W, V = W0[sl].contiguous(), V0[sl].contiguous()
                momentum_step(W, V, agg.float().contiguous(), 0.9, 0.1)
                for b, n in enumerate(rows):
                    assert torch.equal(G[b, :n].view(torch.int32), sw.G[sl][b, :n].view(torch.int32)), (r, b)
                assert torch.equal(W.view(torch.int32), sw.W[sl].view(torch.int32)), r
                assert torch.equal(V.view(torch.int32), sw.V[sl].view(torch.int32)), r
            del G0, W0, V0
        assert not sw.status().any()
        del sw


def test_captured_epochs_equal_eager_epochs(env, pinned_splits):
    _, _, _, sweep = env
    runs = []
    for capture in (False, True):
        sw = small_sweep(sweep, sweep_experiments(), epochs=7, capture=capture)
        for e in range(7):
            sw.step(e)
        torch.cuda.synchronize()
        runs.append(sw)
    a, b = runs
    assert a.n_tests == 3
    for t in ("W", "V", "correct", "loss_sum", "epoch_counter", "test_slot"):
        x, y = getattr(a, t), getattr(b, t)
        assert torch.equal(x.view(torch.uint8), y.view(torch.uint8)), t
    assert int(b.epoch_counter) == 7 and int(b.test_slot) == 3
    assert [r["accuracies"] for r in a.results()] == [r["accuracies"] for r in b.results()]


def test_end_to_end_against_harness_main(env, tmp_path):
    _, _, harness, sweep = env
    kw = dict(learning_rate=0.1, batch_size=128, train_size=6000, test_size=1500)
    exps = [("NoDefense", 0.24, 1.5, 10, 0), ("TrimmedMean", 0.24, 1.5, 10, 0), ("NoDefense", 0.1, 1.0, 10, 3)]
    res = sweep.run(exps, 16, out_dir=str(tmp_path / "sweep"), **kw)
    for r, e in zip(res, exps):
        assert r["error"] is None and r["experiment"] == sweep.Experiment(*e)
        acc, epochs, csv = harness.main(e[1], e[2], e[0], users_count=e[3], epochs=16, out_dir=str(tmp_path / "h"),
                                        seed=e[4], output=str(tmp_path / "log.txt"), **kw)
        assert epochs == r["accuracies_epochs"] == [0, 5, 10, 15]
        # the trajectories part in the last bits (fp32 sums in another order) and stay within a point of accuracy
        assert np.max(np.abs(np.array(acc) - r["accuracies"])) <= 1.0, (acc, r["accuracies"])
        assert os.path.basename(r["csv"]) == os.path.basename(csv)[:-4] + f"_seed_{e[4]}.csv"
        want = open(csv).read().splitlines()
        got = open(r["csv"]).read().splitlines()
        assert len(got) == len(want) == 4
        assert all(len(g) == len(w) and g.endswith(w[-4:]) for g, w in zip(got, want))   # np.savetxt's %.18e
        if e[0] == "NoDefense":
            assert r["accuracies"][-1] > r["accuracies"][0] + 20.0           # it learns
    summary = open(tmp_path / "sweep" / "logs" / sweep.SUMMARY).read().splitlines()
    assert summary[0].split(",") == ["defense", "mal_prop", "num_std", "users_count", "seed", "max_accuracy",
                                     "final_accuracy", "status"]
    assert len(summary) == 4 and all(s.endswith(",ok") for s in summary[1:])


def test_failed_bulyan_experiment_leaves_the_others_alone(env, pinned_splits, tmp_path):
    _, _, _, sweep = env
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
