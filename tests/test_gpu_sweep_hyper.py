"""Per-experiment learning rates and batch sizes on an H100 (the _each entry points, afl_momentum_step_batched and
sweep.Sweep with 8-tuple experiments).

1. Client gradients, both nets: one batch mixing m in {1, 15, 16, 17, 48, 64, 80, 83, 112, 127, 128} (every MnistNet RT
   instance and both sides of a 16-row chunk boundary), on training sets of different lengths and on shard-tail
   minibatches, equals the scalar _sets call at each problem's m bit for bit; a problem whose m lies outside
   [1, max_m] keeps its sentinel rows.
2. Evaluation, both nets: per-problem test batch sizes on a test set that is not a multiple of them equal the scalar
   call at each m bit for bit; a slot out of range, or an m outside [min_m, max_m], writes nothing.
3. The batched momentum step equals afl_momentum_step at each row's learning rate bit for bit.
4. A mixed lr x c sweep (MNIST drift and backdoor, CIFAR10 drift, CIFAR10 backdoor) gives every experiment the bits of
   a sweep of its own (lr, c); captured runs equal eager ones; the first weight step is harness.main's at that lr and
   batch size.
"""
import os

import pytest
import torch

pytestmark = pytest.mark.gpu

D = {"mnist": 79_510, "cifar10": 117_706}
DATASET = {"mnist": "MNIST", "cifar10": "CIFAR10"}
SPLITS = "4"
MS = [1, 15, 16, 17, 48, 64, 80, 83, 112, 127, 128]


@pytest.fixture(scope="module")
def env():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    import __graft_entry__ as g
    g.build()
    from attacking_federate_learning_b200 import _native, harness, sweep
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


def i32(v):
    return torch.tensor(v, dtype=torch.int32, device="cuda")


def bits(t):
    return t.contiguous().view(torch.int32).cpu()


def stream():
    return torch.cuda.current_stream().cuda_stream


_DATA = {}


def data(harness, net, n_train=2000, n_test=500):
    """Two training sets (the second 7 rows shorter, as padded sampler lengths differ), one test set and B weights."""
    if net not in _DATA:
        (xtr, ytr), (xte, yte), model = harness.experiment_setup(3, n_train, n_test, "cuda", DATASET[net])
        w = harness.ParamLayout(model.parameters()).flatten(list(model.parameters()))
        x = torch.stack([xtr, xtr.flip(0)]).contiguous()
        y = torch.stack([ytr, ytr.flip(0)]).contiguous()
        g = torch.Generator("cuda").manual_seed(11)
        W = (w + 0.01 * torch.randn((len(MS), w.numel()), device="cuda", generator=g)).contiguous()
        _DATA[net] = (x, y, i32([n_train, n_train - 7]), xte[None].contiguous(), yte[None].contiguous(), W)
    return _DATA[net]


def grads(nat, net, W, x, y, set_len, sets, rows, n, m, epoch, G, max_m=None):
    """The _sets call at scalar m (max_m None), else the _each call with m a device array."""
    L = nat.lib()
    head = (W.data_ptr(), W.shape[0], D[net], x.data_ptr(), y.data_ptr(), x.shape[0], x.shape[1], set_len.data_ptr(),
            sets.data_ptr(), rows.data_ptr(), n)
    tail = (epoch.data_ptr(), G.data_ptr(), G.stride(0), G.stride(1), stream())
    if max_m is None:
        nat.check(getattr(L, f"afl_{net}_client_grads_sets")(*head, m, *tail))
    else:
        nat.check(getattr(L, f"afl_{net}_client_grads_each")(*head, m.data_ptr(), max_m, *tail))


@pytest.mark.parametrize("net", ["mnist", "cifar10"])
@pytest.mark.parametrize("epoch", [2, 3])
def test_client_grads_each_equal_the_scalar_call(env, net, epoch):
    """7 clients on sets of 2000 and 1993 rows (shards of 284-286 rows): at epoch 2 m = 112, 127 and 128 take a
    shard-tail minibatch, at epoch 3 m = 80 and 83 do."""
    nat, harness, _ = env
    x, y, set_len, _, _, W = data(harness, net)
    B, n, d = len(MS), 7, D[net]
    ld = (d + 31) // 32 * 32
    sets, rows, ep = i32([b % 2 for b in range(B)]), i32([n] * B), i32([epoch])
    got = torch.full((B, n, ld), 7.0, device="cuda")
    grads(nat, net, W, x, y, set_len, sets, rows, n, i32(MS), ep, got, max_m=128)
    want = torch.full((B, n, ld), 7.0, device="cuda")
    for m in MS:
        grads(nat, net, W, x, y, set_len, sets, rows, n, m, ep, want)
        b = MS.index(m)
        assert torch.equal(bits(got[b]), bits(want[b])), m
    # max_m = 64 (MnistNet's RT = 4 instance): problems with m in [1, 64] are the same bits, the others keep sentinels
    again = torch.full((B, n, ld), 7.0, device="cuda")
    grads(nat, net, W, x, y, set_len, sets, rows, n, i32(MS), ep, again, max_m=64)
    for b, m in enumerate(MS):
        if m <= 64:
            assert torch.equal(bits(again[b]), bits(got[b])), m
        else:
            assert bool((again[b] == 7.0).all()), m
    # m = 0 and a negative m are out of range too
    bad = torch.full((B, n, ld), 7.0, device="cuda")
    grads(nat, net, W, x, y, set_len, sets, rows, n, i32([0, -3] + MS[2:]), ep, bad, max_m=128)
    assert bool((bad[:2] == 7.0).all())
    assert torch.equal(bits(bad[2:]), bits(got[2:]))


def evaluate(nat, net, W, xte, yte, sets, m, slot, n_slots, loss, correct, n_test, min_m=None, max_m=None):
    L = nat.lib()
    ws_m = m if min_m is None else min_m
    ws = torch.empty(getattr(L, f"afl_{net}_evaluate_workspace_bytes")(W.shape[0], n_test, ws_m), dtype=torch.uint8,
                     device="cuda")
    head = (W.data_ptr(), W.shape[0], D[net], xte.data_ptr(), yte.data_ptr(), 1, n_test, sets.data_ptr())
    tail = (slot.data_ptr(), n_slots, loss.data_ptr(), correct.data_ptr(), ws.data_ptr(), ws.numel(), stream())
    if min_m is None:
        nat.check(getattr(L, f"afl_{net}_evaluate")(*head, m, *tail))
    else:
        nat.check(getattr(L, f"afl_{net}_evaluate_each")(*head, m.data_ptr(), min_m, max_m, *tail))
    torch.cuda.synchronize()                      # ws is freed on return


@pytest.mark.parametrize("net", ["mnist", "cifar10"])
def test_evaluate_each_equals_the_scalar_call(env, net):
    nat, harness, _ = env
    _, _, _, xte, yte, W = data(harness, net)
    B, n_test = len(MS), 500
    sets, slot = i32([0] * B), i32([1])
    loss = torch.full((3, B), -1.0, dtype=torch.float64, device="cuda")
    correct = torch.full((3, B), -1, dtype=torch.int32, device="cuda")
    evaluate(nat, net, W, xte, yte, sets, i32(MS), slot, 3, loss, correct, n_test, min_m=1, max_m=128)
    assert bool((loss[[0, 2]] == -1).all()) and bool((correct[[0, 2]] == -1).all())
    for b, m in enumerate(MS):
        wl = torch.full((3, B), -1.0, dtype=torch.float64, device="cuda")
        wc = torch.full((3, B), -1, dtype=torch.int32, device="cuda")
        evaluate(nat, net, W, xte, yte, sets, m, slot, 3, wl, wc, n_test)
        assert float(loss[1, b]) == float(wl[1, b]) and int(correct[1, b]) == int(wc[1, b]), m
    # [min_m, max_m] = [16, 83]: the other problems, and a slot out of range, write nothing
    l2 = torch.full((3, B), -1.0, dtype=torch.float64, device="cuda")
    c2 = torch.full((3, B), -1, dtype=torch.int32, device="cuda")
    evaluate(nat, net, W, xte, yte, sets, i32(MS), slot, 3, l2, c2, n_test, min_m=16, max_m=83)
    for b, m in enumerate(MS):
        if 16 <= m <= 83:
            assert float(l2[1, b]) == float(loss[1, b]) and int(c2[1, b]) == int(correct[1, b]), m
        else:
            assert float(l2[1, b]) == -1 and int(c2[1, b]) == -1, m
    l3 = torch.full((3, B), -1.0, dtype=torch.float64, device="cuda")
    c3 = torch.full((3, B), -1, dtype=torch.int32, device="cuda")
    evaluate(nat, net, W, xte, yte, sets, i32(MS), i32([3]), 3, l3, c3, n_test, min_m=1, max_m=128)
    assert bool((l3 == -1).all()) and bool((c3 == -1).all())


def test_momentum_step_batched_equals_the_scalar_step(env):
    nat, _, _ = env
    from attacking_federate_learning_b200 import _device
    lrs = [0.05, 0.1, 0.2, 0.3, 1e-3]
    B, d = len(lrs), D["mnist"]
    g = torch.Generator("cuda").manual_seed(5)
    w, v, gr = (torch.randn((B, d), device="cuda", generator=g) for _ in range(3))
    w2, v2 = w.clone(), v.clone()
    _device.momentum_step_batched(w, v, gr, 0.9, torch.tensor(lrs, dtype=torch.float32, device="cuda"))
    for b, lr in enumerate(lrs):
        _device.momentum_step(w2[b], v2[b], gr[b], 0.9, lr)
    assert torch.equal(bits(w), bits(w2)) and torch.equal(bits(v), bits(v2))


def run_sweep(sweep, exps, epochs, capture=True, **kw):
    kw = dict(dict(learning_rate=0.1, batch_size=83, train_size=2000, test_size=500, test_step=2), **kw)
    sw = sweep.Sweep(exps, epochs, capture=capture, **kw)
    for e in range(epochs):
        sw.step(e)
    return sw, sw.results()


def assert_alone(sweep, exps, epochs, **kw):
    """Each experiment of a mixed run against a sweep of its own (lr, c), as the short tuple."""
    mixed, res = run_sweep(sweep, exps, epochs, **kw)
    for i, e in enumerate(exps):
        short = tuple(sweep.Experiment(*e[:6]))                          # the 5- or 6-tuple
        own = dict(learning_rate=e[6], batch_size=e[7]) if len(e) == 8 else {}
        alone, ra = run_sweep(sweep, [short], epochs, **dict(kw, **own))
        p = mixed.order.index(i)
        assert res[i]["error"] is None and ra[0]["error"] is None, exps[i]
        assert torch.equal(bits(mixed.W[p]), bits(alone.W[0])), exps[i]
        assert torch.equal(bits(mixed.V[p]), bits(alone.V[0])), exps[i]
        for k in ("accuracies", "losses", "backdoor_accuracies", "backdoor_losses"):
            assert res[i].get(k) == ra[0].get(k), (exps[i], k)


def test_mnist_mixed_sweep_equals_each_experiment_alone(env, pinned_splits):
    _, _, sweep = env
    exps = [("Krum", 0.1, 1.0, 10, 0, False, 0.05, 32), ("TrimmedMean", 0.24, 1.5, 10, 1, False, 0.2, 128),
            ("NoDefense", 0.24, 1.0, 10, 0, "pattern", 0.05, 83), ("TrimmedMean", 0.24, 0.5, 10, 1, 1, 0.2, 17),
            ("Bulyan", 0.0, 0.25, 10, 1, False, 0.1, 1), ("NoDefense", 0.1, 1.0, 10, 0)]
    assert_alone(sweep, exps, 4)


def test_cifar10_mixed_sweep_equals_each_experiment_alone(env, pinned_splits):
    _, _, sweep = env
    exps = [("Krum", 0.1, 1.0, 10, 0, False, 0.05, 32), ("NoDefense", 0.24, 1.0, 10, 1, False, 0.2, 128),
            ("TrimmedMean", 0.24, 1.5, 10, 0)]
    assert_alone(sweep, exps, 3, dataset="CIFAR10", fading_rate=2000)


def test_cifar10_backdoor_mixed_sweep_equals_each_experiment_alone(env, pinned_splits):
    _, _, sweep = env
    exps = [("NoDefense", 0.24, 1.0, 10, 0, "pattern", 0.05, 32), ("NoDefense", 0.24, 1.0, 10, 0, False, 0.2, 83)]
    assert_alone(sweep, exps, 2, dataset="CIFAR10", fading_rate=2000, cifar10_backdoor=True)


def test_captured_mixed_sweep_equals_eager(env, pinned_splits):
    _, _, sweep = env
    exps = [("Krum", 0.1, 1.0, 10, 0, False, 0.05, 32), ("NoDefense", 0.24, 1.0, 10, 0, "pattern", 0.2, 128),
            ("TrimmedMean", 0.24, 1.5, 10, 1), ("TrimmedMean", 0.24, 0.5, 10, 1, 2, 0.1, 64)]
    (a, ra), (b, rb) = (run_sweep(sweep, exps, 5, capture=c) for c in (False, True))
    for t in ("W", "V", "loss_sum", "correct", "bd_loss_sum", "bd_correct", "bd_mal"):
        assert torch.equal(bits(getattr(a, t)), bits(getattr(b, t))), t
    for k in ("accuracies", "losses", "backdoor_accuracies", "backdoor_losses"):
        assert [r.get(k) for r in ra] == [r.get(k) for r in rb], k
    assert a.m.tolist() == [32, 83, 64, 128] and a.lr.tolist() == pytest.approx([0.05, 0.1, 0.1, 0.2])


@pytest.mark.parametrize("e", [("NoDefense", 0.24, 1.0, 10, 0, False, 0.05, 32),
                               ("TrimmedMean", 0.24, 1.5, 10, 0, False, 0.2, 128)])
def test_first_weight_step_against_harness_main(env, e, monkeypatch, tmp_path):
    """The sweep's first weight step, in a batch with other (lr, c), against harness.main(learning_rate=lr,
    batch_size=c)'s: ||dW_sweep - dW_h|| / ||dW_h|| <= 1e-3 (the client gradients sum in another fp32 order)."""
    _, harness, sweep = env
    other = ("NoDefense", 0.1, 1.0, 10, 0, False, 0.1, 83)
    kw = dict(train_size=4000, test_size=1000)
    sw = sweep.Sweep([e, other], 1, **kw)
    p = sw.order.index(0)
    w0 = sw.W[p].clone()
    sw.step(0)
    seen = []
    orig = harness.AggregationServer.defend

    def defend(self, *a, **k):
        out = orig(self, *a, **k)
        seen.append(self.current_weights.clone())
        return out
    monkeypatch.setattr(harness.AggregationServer, "defend", defend)
    harness.main(e[1], e[2], e[0], users_count=e[3], epochs=1, out_dir=str(tmp_path), seed=e[4],
                 output=str(tmp_path / "log.txt"), learning_rate=e[6], batch_size=e[7], **kw)
    monkeypatch.undo()
    step_h, step_s = seen[0] - w0, sw.W[p] - w0
    err = float(torch.linalg.norm((step_s - step_h).double()) / torch.linalg.norm(step_h.double()))
    assert err <= 1e-3, err


def test_run_writes_per_experiment_names_and_columns(env, tmp_path):
    _, _, sweep = env
    exps = [("NoDefense", 0.1, 1.0, 10, 0, False, 0.05, 32), ("NoDefense", 0.1, 1.0, 10, 0, False, 0.05, 64),
            ("NoDefense", 0.1, 1.0, 10, 0)]
    res = sweep.run(exps, 2, train_size=2000, test_size=500, out_dir=str(tmp_path))
    names = [os.path.basename(r["csv"]) for r in res]
    assert len(set(names)) == 3 and "_batch_32_seed_0" in names[0] and "_batch_64_seed_0" in names[1]
    assert "_batch_" not in names[2] and "_lr_0.05_" in names[0] and "_lr_0.1_" in names[2]
    rows = open(os.path.join(tmp_path, "logs", sweep.SUMMARY)).read().splitlines()
    assert rows[0].split(",") == sweep.summary_header(False, True)
    assert [r.split(",")[5:7] for r in rows[1:]] == [["0.05", "32"], ["0.05", "64"], ["0.1", "83"]]
