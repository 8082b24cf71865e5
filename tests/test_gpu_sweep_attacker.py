"""Per-experiment backdoor α and malicious epochs on an H100 (afl_*_backdoor_train_each and sweep.Sweep with 10-tuple
experiments), for MnistNet and Cifar10Net.

1. One _each launch mixing α in {-1, 0, 0.2, 4} and epochs in {0, 1, 2, 5}, with a problem whose BEFORE test is
   already 100 % and an inactive one: every problem equals the scalar call at its own values, run alone, bit for bit;
   epochs = 0 returns initial bit for bit although BEFORE is below 100 %.
2. The distance term per problem: a NaN initial gets AFL_ERR_NAN_DIST_LOSS at α > 0 and not at α = 0.
3. A NaN α or a negative epoch count gets AFL_ERR_BAD_ARG and leaves its out row alone; the others keep their bits.
4. Mixed sweeps (MNIST pattern and sample 1, CIFAR10 pattern) with drift experiments in the batch: every backdoor
   experiment has the bits of a sweep at its own α and mal_epochs, every drift one those of a drift-only sweep;
   captured equals eager; the first weight step is harness.main(..., alpha=0.2, mal_epochs=k)'s.
"""
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

D = {"mnist": 79_510, "cifar10": 117_706}
DATASET = {"mnist": "MNIST", "cifar10": "CIFAR10"}
N_TRAIN = {"mnist": 2000, "cifar10": 400}        # pattern sets of 2000 and 400 rows (10 and 2 minibatches)
SPLITS = "4"
SENTINEL = -7.25


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


def dev(v, dtype):
    return torch.as_tensor(np.asarray(v), dtype=dtype, device="cuda")


def bits(t):
    return t.contiguous().view(torch.int32).cpu()


def setup(harness, sweep, net):
    """The seed-0 training set's backdoor sets (pattern, then a one-sample set whose label is not 0, so that NaN logits,
    which torch's argmax reads as class 0, miss it) and noisy initial vectors around the seed's weights."""
    (x, y), _, model = harness.experiment_setup(0, N_TRAIN[net], 10, "cuda", DATASET[net])
    k = next(k for k in (1, 2, 3) if int(harness.backdoor_set(k, x, y)[1][0]) != 0)
    sets = sweep.backdoor_sets([("pattern", x, y, 0), (k, x, y, 0)])
    w = harness.ParamLayout(model.parameters()).flatten(list(model.parameters()))
    g = torch.Generator(device="cuda").manual_seed(13)
    inits = torch.stack([w + 0.01 * (1 + i % 3) * torch.randn(D[net], device="cuda", generator=g)
                         for i in range(8)]).contiguous()
    return sets, inits


def trainer(nat, net, initial, sets, index, alpha, epochs, f=None):
    """The scalar call when alpha and epochs are numbers, the _each call when they are lists.  Returns (out, status)."""
    B = initial.shape[0]
    xs, ys, lens = sets
    f = dev([1] * B if f is None else f, torch.int32)
    z = dev([1.0] * B, torch.float64)
    status = dev([0] * B, torch.int32)
    out = torch.full_like(initial, SENTINEL)
    index = dev(index, torch.int32)
    each = isinstance(alpha, list)
    a = dev(alpha, torch.float32) if each else float(alpha)
    e = dev(epochs, torch.int32) if each else int(epochs)
    L = nat.lib()
    head = (initial.data_ptr(), out.data_ptr(), B, D[net], xs.data_ptr(), ys.data_ptr(), xs.shape[0], xs.shape[1],
            lens.data_ptr(), index.data_ptr(), f.data_ptr(), z.data_ptr(), status.data_ptr(),
            a.data_ptr() if each else a, e.data_ptr() if each else e, 200)
    fn = getattr(L, f"afl_{net}_backdoor_train{'_each' if each else ''}")
    stream = torch.cuda.current_stream().cuda_stream
    if net == "cifar10":
        ws = torch.empty(L.afl_cifar10_backdoor_train_workspace_bytes(B), dtype=torch.uint8, device="cuda")
        nat.check(fn(*head, ws.data_ptr(), ws.numel(), stream))
    else:
        nat.check(fn(*head, stream))
    torch.cuda.current_stream().synchronize()       # every array the kernel reads stays alive until it has run
    return out, status


@pytest.mark.parametrize("net", ["mnist", "cifar10"])
def test_each_problem_equals_the_scalar_call_alone(env, net):
    nat, harness, sweep = env
    sets, inits = setup(harness, sweep, net)
    inits[4, D[net] - 10] = 1e4                     # the last bias's class 0: every pattern row is right already
    alphas = [-1.0, 0.0, 0.2, 4.0, 4.0, 0.2, 0.2, 4.0]
    epochs = [2, 1, 5, 0, 2, 1, 1, 5]
    index = [0, 0, 0, 0, 0, 0, 1, 0]
    f = [1, 1, 1, 1, 1, 0, 1, 1]                    # problem 5 does not attack
    got, status = trainer(nat, net, inits, sets, index, alphas, epochs, f=f)
    assert status.cpu().tolist() == [0] * 8
    assert bool((got[5] == SENTINEL).all())
    for b in (0, 1, 2, 3, 4, 6, 7):
        alone, st = trainer(nat, net, inits[b:b + 1].contiguous(), sets, [index[b]], alphas[b], epochs[b])
        assert int(st[0]) == 0
        assert torch.equal(bits(got[b]), bits(alone[0])), (b, alphas[b], epochs[b])
    for b in (3, 4):                                # epochs 0, and BEFORE at 100 %: initial bit for bit
        assert torch.equal(bits(got[b]), bits(inits[b])), b
    for b in (0, 1, 2, 7):
        assert not torch.equal(got[b], inits[b]), b
    # problem 3's BEFORE is below 100 %: with one epoch it trains
    once, _ = trainer(nat, net, inits[3:4].contiguous(), sets, [0], 4.0, 1)
    assert not torch.equal(once[0], inits[3])
    # the α <= 0 problems train without the distance term: -1 and 0 give the same bits
    neg, _ = trainer(nat, net, inits[:1].contiguous(), sets, [0], 0.0, 2)
    assert torch.equal(bits(neg[0]), bits(got[0]))


@pytest.mark.parametrize("net", ["mnist", "cifar10"])
def test_distance_term_is_per_problem(env, net):
    nat, harness, sweep = env
    sets, inits = setup(harness, sweep, net)
    inits = inits[:3].clone()
    inits[0, D[net] - 3] = float("nan")
    inits[1, D[net] - 3] = float("nan")
    got, status = trainer(nat, net, inits, sets, [1, 1, 1], [4.0, 0.0, 4.0], [2, 2, 2])
    st = status.cpu().tolist()
    assert st[0] == nat.AFL_ERR_NAN_DIST_LOSS and st[1] != nat.AFL_ERR_NAN_DIST_LOSS and st[2] == 0
    for b, a in ((1, 0.0), (2, 4.0)):
        alone, st_a = trainer(nat, net, inits[b:b + 1].contiguous(), sets, [1], a, 2)
        assert int(st_a[0]) == st[b]
        assert torch.equal(bits(got[b]), bits(alone[0])), b


@pytest.mark.parametrize("net", ["mnist", "cifar10"])
def test_invalid_values_flag_their_problem_only(env, net):
    nat, harness, sweep = env
    sets, inits = setup(harness, sweep, net)
    inits = inits[:4].contiguous()
    got, status = trainer(nat, net, inits, sets, [0, 0, 1, 0], [float("nan"), 0.2, 0.2, 4.0], [1, -1, 1, 2])
    assert status.cpu().tolist() == [nat.AFL_ERR_BAD_ARG, nat.AFL_ERR_BAD_ARG, 0, 0]
    assert bool((got[:2] == SENTINEL).all())
    for b, (s, a, e) in ((2, (1, 0.2, 1)), (3, (0, 4.0, 2))):
        alone, _ = trainer(nat, net, inits[b:b + 1].contiguous(), sets, [s], a, e)
        assert torch.equal(bits(got[b]), bits(alone[0])), b


def run_sweep(sweep, exps, epochs, capture=True, **kw):
    kw = dict(dict(learning_rate=0.1, batch_size=83, train_size=2000, test_size=500, test_step=2), **kw)
    sw = sweep.Sweep(exps, epochs, capture=capture, **kw)
    for e in range(epochs):
        sw.step(e)
    return sw, sw.results()


KEYS = ("accuracies", "losses", "backdoor_accuracies", "backdoor_losses")


def assert_alone(sweep, exps, epochs, **kw):
    """Each backdoor experiment of a mixed run against a sweep of its own (α, mal_epochs) as the 6-tuple, the drift
    experiments against a drift-only sweep."""
    mixed, res = run_sweep(sweep, exps, epochs, **kw)
    for i, e in enumerate(exps):
        e = sweep.Experiment(*e)
        if e.backdoor is False:
            continue
        own = {} if e.alpha is None else dict(alpha=e.alpha, mal_epochs=e.mal_epochs)
        alone, ra = run_sweep(sweep, [tuple(e[:6])], epochs, **dict(kw, **own))
        p = mixed.order.index(i)
        assert res[i]["error"] is None and ra[0]["error"] is None, e
        assert torch.equal(bits(mixed.W[p]), bits(alone.W[0])), e
        assert torch.equal(bits(mixed.V[p]), bits(alone.V[0])), e
        for k in KEYS:
            assert res[i].get(k) == ra[0].get(k), (e, k)
    drift = [i for i, e in enumerate(exps) if len(e) == 5]
    only, ro = run_sweep(sweep, [exps[i] for i in drift], epochs, **kw)
    for j, i in enumerate(drift):
        pm, po = mixed.order.index(i), only.order.index(j)
        assert torch.equal(bits(mixed.W[pm]), bits(only.W[po])), exps[i]
        assert res[i]["accuracies"] == ro[j]["accuracies"] and res[i]["losses"] == ro[j]["losses"]
    return mixed


MNIST_MIXED = [("TrimmedMean", 0.24, 1.5, 10, 0), ("NoDefense", 0.24, 1.0, 10, 0, "pattern", 0.1, 83, 0.2, 1),
               ("Krum", 0.1, 1.0, 10, 1, 1, 0.1, 83, 4, 2), ("NoDefense", 0.1, 1.0, 10, 1),
               ("TrimmedMean", 0.24, 0.5, 10, 1, "pattern", 0.1, 83, 0, 5),
               ("NoDefense", 0.24, 1.0, 10, 1, "pattern", 0.1, 83, 4, 0), ("TrimmedMean", 0.24, 1.0, 10, 0, 1)]


def test_mnist_mixed_sweep_equals_each_experiment_alone(env, pinned_splits):
    _, _, sweep = env
    sw = assert_alone(sweep, MNIST_MIXED, 4, alpha=1.0, mal_epochs=2)
    # batch order: Krum, TrimmedMean (a 10-tuple, then a 6-tuple at the run's values), NoDefense
    assert sw.bd_alpha.tolist() == pytest.approx([4.0, 0.0, 1.0, 0.2, 4.0])
    assert sw.bd_mal_epochs.tolist() == [2, 5, 2, 1, 0]


def test_cifar10_mixed_sweep_equals_each_experiment_alone(env, pinned_splits):
    _, _, sweep = env
    exps = [("NoDefense", 0.24, 1.0, 10, 0, "pattern", 0.1, 83, 0.2, 1), ("TrimmedMean", 0.24, 1.5, 10, 0),
            ("NoDefense", 0.24, 1.0, 10, 0, "pattern", 0.1, 83, 4, 2), ("NoDefense", 0.24, 1.0, 10, 0, "pattern")]
    assert_alone(sweep, exps, 2, dataset="CIFAR10", fading_rate=2000, cifar10_backdoor=True, train_size=400,
                 test_size=200, mal_epochs=1)


def test_captured_mixed_sweep_equals_eager(env, pinned_splits):
    _, _, sweep = env
    (a, ra), (b, rb) = (run_sweep(sweep, MNIST_MIXED, 5, capture=c) for c in (False, True))
    for t in ("W", "V", "loss_sum", "correct", "bd_loss_sum", "bd_correct", "bd_mal"):
        assert torch.equal(bits(getattr(a, t)), bits(getattr(b, t))), t
    for k in KEYS:
        assert [r.get(k) for r in ra] == [r.get(k) for r in rb], k
    assert all(r["error"] is None for r in ra + rb)


@pytest.mark.parametrize("k", [1, 2])
def test_first_weight_step_against_harness_main(env, k, monkeypatch, tmp_path):
    """The sweep's first weight step, in a batch with another (α, mal_epochs), against harness.main(alpha=0.2,
    mal_epochs=k)'s: ||dW_sweep - dW_h|| / ||dW_h|| <= 1e-3 (sums run in other fp32 orders)."""
    _, harness, sweep = env
    kw = dict(learning_rate=0.1, batch_size=128, train_size=4000, test_size=1000)
    e = ("NoDefense", 0.24, 1.0, 10, 0, "pattern", 0.1, 128, 0.2, k)
    other = ("NoDefense", 0.24, 1.0, 10, 0, "pattern", 0.1, 128, 4, 5)
    sw = sweep.Sweep([e, other], 1, **kw)
    p = sw.order.index(0)
    w0 = sw.W[p].clone()
    sw.step(0)
    seen = []
    orig = harness.AggregationServer.defend

    def defend(self, *a, **kk):
        out = orig(self, *a, **kk)
        seen.append(self.current_weights.clone())
        return out
    monkeypatch.setattr(harness.AggregationServer, "defend", defend)
    harness.main(e[1], e[2], e[0], users_count=e[3], epochs=1, out_dir=str(tmp_path), seed=e[4],
                 output=str(tmp_path / "log.txt"), backdoor="pattern", alpha=0.2, mal_epochs=k, **kw)
    monkeypatch.undo()
    step_h, step_s = seen[0] - w0, sw.W[p] - w0
    err = float(torch.linalg.norm((step_s - step_h).double()) / torch.linalg.norm(step_h.double()))
    assert err <= 1e-3, err


def test_run_writes_per_experiment_names_and_columns(env, tmp_path):
    _, _, sweep = env
    exps = [("NoDefense", 0.1, 1.0, 10, 0, "pattern", 0.1, 83, 0.2, 1),
            ("NoDefense", 0.1, 1.0, 10, 0, "pattern", 0.1, 83, 4, 1), ("NoDefense", 0.1, 1.0, 10, 0),
            ("NoDefense", 0.1, 1.0, 10, 0, "pattern")]
    res = sweep.run(exps, 2, train_size=2000, test_size=500, out_dir=str(tmp_path), mal_epochs=2)
    names = [os.path.basename(r["csv"]) for r in res]
    assert len(set(names)) == 4 and all(r["error"] is None for r in res)
    assert names[0].endswith("_alpha_0.2_lr_0.1_batch_83_malepochs_1_seed_0.csv")
    assert names[1].endswith("_alpha_4.0_lr_0.1_batch_83_malepochs_1_seed_0.csv")
    assert "_malepochs_" not in names[3] and names[3].endswith("_alpha_4_lr_0.1_seed_0.csv")
    rows = open(os.path.join(tmp_path, "logs", sweep.SUMMARY)).read().splitlines()
    assert rows[0].split(",") == sweep.summary_header(True, True, False, True)
    assert [r.split(",")[6:10] for r in rows[1:]] == [["0.1", "83", "0.2", "1"], ["0.1", "83", "4.0", "1"],
                                                      ["0.1", "83", "", ""], ["0.1", "83", "4", "2"]]
