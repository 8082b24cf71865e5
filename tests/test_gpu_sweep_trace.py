"""The attack trace on an H100 (afl_attack_trace_dev, DeviceRound.attack_trace, Sweep(trace=True)).

1. The kernel against afl_attack_metrics_batched_dev bit for bit and a float64 oracle within 1e-5: ragged batches
   with per-problem f (0 and rows_b included), Krum index -1, Bulyan selections with -1 / -2, N = 10, 129 and 1000,
   16-byte and scalar loads.  Slots -1 and n_slots write nothing; every other entry keeps its sentinel.
2. A captured call replayed with an advancing slot fills successive rows, equal to eager calls.
3. Training with trace equals training without it bit for bit (MNIST drift and backdoor with every rule and
   N = 1000 beside N = 10; CIFAR10 with its backdoor).
4. The sweep's trace equals an eager recompute with DeviceRound.attack_metrics at every epoch, and replayed epochs
   equal eager ones; a backdoor experiment's malicious deviation is its crafted row's.
5. Epoch 0 against harness.main(trace=True); a failing Bulyan experiment gets trace None and leaves the others alone.
"""
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

SENT = -9
NAMES = ("agg_deviation", "malicious_deviation", "krum_index", "bulyan_malicious", "bulyan_selected")


@pytest.fixture(scope="module")
def env():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    import __graft_entry__ as g
    g.build()
    from attacking_federate_learning_b200 import batched, harness, sweep
    return batched, harness, sweep


@pytest.fixture
def pinned_splits():
    saved = os.environ.get("AFL_GRAM_SPLITS")
    os.environ["AFL_GRAM_SPLITS"] = "4"
    yield
    if saved is None:
        os.environ.pop("AFL_GRAM_SPLITS", None)
    else:
        os.environ["AFL_GRAM_SPLITS"] = saved


def bits(t):
    return t.contiguous().view(torch.int32)


def tables(B, n_slots, pad=2):
    """[n_slots, B + pad] sentinel tables; the first B columns are the call's."""
    return {k: torch.full((n_slots, B + pad), SENT, dtype=torch.float32 if k.endswith("deviation") else torch.int32,
                          device="cuda") for k in NAMES}


def oracle_dev(G, f, rows, a):
    """float64 ||a - h|| / ||h||, h the mean of rows f..rows-1 of G (numpy)."""
    if f >= rows:
        return float("nan")
    h = G[f:rows].astype(np.float64).mean(0)
    return float(np.linalg.norm(a.astype(np.float64) - h) / np.linalg.norm(h))


@pytest.mark.parametrize("N, D, ragged", [(10, 4096, True), (10, 1001, True), (129, 3000, True), (1000, 2048, True),
                                          (129, 2000, False)])
def test_trace_against_attack_metrics(env, N, D, ragged):
    bt, _, _ = env
    rng = np.random.default_rng(N + D)
    B = 6
    G = torch.from_numpy(rng.standard_normal((B, N, D)).astype(np.float32) + 0.5).cuda()
    rows = [N, max(1, N // 2), N, 3, N, N - 1] if ragged else [N] * B
    fs = [0, rows[1] // 4, rows[2], 1, N // 5, 0]                   # f = 0, f = rows_b included
    rnd = bt.DeviceRound(G, rows=ragged, rules=())
    rnd.f.copy_(torch.tensor(fs, dtype=torch.int32))
    if ragged:
        rnd.rows.copy_(torch.tensor(rows, dtype=torch.int32))
    agg = torch.from_numpy(rng.standard_normal((B, D)).astype(np.float32)).cuda()
    idx = torch.tensor([0, -1, 2, 1, N - 1, 0], dtype=torch.int32, device="cuda")
    sel = torch.from_numpy(rng.integers(0, 3, (B, N)).astype(np.int32)).cuda()
    sel[1, 2:] = -1
    sel[2, N // 2:] = -2
    sel[3, 0] = -1
    tab, slot = tables(B, 3), torch.tensor([1], dtype=torch.int32, device="cuda")
    views = {k: v[:, :B] for k, v in tab.items()}
    rnd.attack_trace(agg, slot, views, krum_index=idx, selection=sel)
    for s in (-1, 3):                                              # outside [0, n_slots): nothing written
        rnd.attack_trace(agg, torch.tensor([s], dtype=torch.int32, device="cuda"), views, krum_index=idx,
                         selection=sel)
    by_agg = rnd.attack_metrics(aggregated=agg, selection=sel)
    by_row0 = rnd.attack_metrics(krum_index=torch.zeros(B, dtype=torch.int32, device="cuda"))
    torch.cuda.synchronize()
    assert not rnd.status.any()
    got = {k: v[1, :B] for k, v in tab.items()}
    assert torch.equal(bits(got["agg_deviation"]), bits(by_agg["rel_deviation"]))
    pos = torch.tensor([f > 0 for f in fs], device="cuda")
    assert torch.equal(bits(got["malicious_deviation"][pos]), bits(by_row0["rel_deviation"][pos]))
    assert torch.isnan(got["malicious_deviation"][~pos]).all()
    assert torch.equal(got["krum_index"], idx)
    frac = got["bulyan_malicious"].float() / got["bulyan_selected"].clamp(min=1).float()
    assert torch.equal(bits(frac), bits(by_agg["bulyan_malicious_fraction"]))
    Gh, ah, sh = G.cpu().numpy(), agg.cpu().numpy(), sel.cpu().numpy()
    for b in range(B):
        s = sh[b]
        assert int(got["bulyan_selected"][b]) == int((s >= 0).sum())
        assert int(got["bulyan_malicious"][b]) == int(((s >= 0) & (s < fs[b])).sum())
        for key, a in (("agg_deviation", ah[b]), ("malicious_deviation", Gh[b, 0])):
            want = oracle_dev(Gh[b], fs[b], rows[b], a)
            if key == "malicious_deviation" and fs[b] == 0:
                continue
            v = float(got[key][b])
            assert (np.isnan(v) and np.isnan(want)) or abs(v - want) <= 1e-5 * want, (key, b, v, want)
    for k, v in tab.items():                                       # other rows and the pad columns keep the sentinel
        keep = torch.ones_like(v, dtype=torch.bool)
        keep[1, :B] = False
        assert (v[keep] == SENT).all(), k


def test_captured_trace_fills_successive_rows(env):
    bt, _, _ = env
    rng = np.random.default_rng(5)
    B, N, D, S = 4, 12, 3000, 5
    G = torch.from_numpy(rng.standard_normal((B, N, D)).astype(np.float32)).cuda()
    rnd = bt.DeviceRound(G, rows=True, rules=(bt.DefenseTypes.Krum,))
    rnd.f.copy_(torch.tensor([1, 2, 0, 3], dtype=torch.int32))
    rnd.rows.copy_(torch.tensor([12, 10, 7, 12], dtype=torch.int32))
    slot = torch.zeros(1, dtype=torch.int32, device="cuda")
    eager, graph = tables(B, S), tables(B, S)
    names = ("agg_deviation", "malicious_deviation", "krum_index")

    def round_(tab):
        G.add_(0.125)                                              # a new round's matrix
        agg = rnd.krum()
        rnd.attack_trace(agg, slot, {k: tab[k][:, :B] for k in names}, krum_index=rnd.krum_index)
        slot.add_(1)
    G0 = G.clone()
    for _ in range(S):
        round_(eager)
    G.copy_(G0)
    slot.zero_()
    round_(graph)                                                  # eager warm-up: row 0
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        round_(graph)
    G.copy_(G0)
    G.add_(0.125)
    slot.fill_(1)                                                  # the capture ran round 1's work once
    for _ in range(S - 1):
        g.replay()
    torch.cuda.synchronize()
    assert int(slot) == S
    for k in names:
        assert torch.equal(bits(eager[k]), bits(graph[k])), k
        assert (eager[k][:, :B] != SENT).all(), k


def small_sweep(sweep, exps, epochs, capture, trace, **kw):
    kw = dict(dict(learning_rate=0.1, batch_size=83, train_size=2000, test_size=500, test_step=2), **kw)
    return sweep.Sweep(exps, epochs, capture=capture, trace=trace, **kw)


MNIST_GRID = [("Krum", 0.1, 1.0, 10, 0), ("Bulyan", 0.1, 1.5, 11, 1), ("TrimmedMean", 0.24, 0.5, 10, 0),
              ("NoDefense", 0.24, 2.0, 10, 1), ("TrimmedMean", 0.1, 1.0, 1000, 0),
              ("Krum", 0.24, 1.0, 10, 0, "pattern"), ("Bulyan", 0.1, 1.0, 10, 1, 1),
              ("TrimmedMean", 0.24, 1.5, 10, 1, "pattern"), ("NoDefense", 0.1, 1.0, 10, 0, 1)]
CIFAR_GRID = [("NoDefense", 0.24, 1.0, 10, 0, "pattern"), ("Krum", 0.1, 1.0, 10, 1, 1), ("TrimmedMean", 0.24, 1.5, 10, 0),
              ("Bulyan", 0.1, 0.5, 11, 1)]


@pytest.mark.parametrize("grid, kw", [(MNIST_GRID, {}),
                                      (CIFAR_GRID, dict(dataset="CIFAR10", cifar10_backdoor=True, mal_epochs=2,
                                                        fading_rate=2000))])
def test_trace_leaves_training_alone(env, pinned_splits, grid, kw):
    _, _, sweep = env
    runs = []
    for trace in (False, True):
        sw = small_sweep(sweep, grid, 4, True, trace, **kw)
        for e in range(4):
            sw.step(e)
        torch.cuda.synchronize()
        runs.append(sw)
    a, b = runs
    assert a.trace is None and b.trace is not None
    for t in ("W", "V", "correct", "loss_sum", "bd_correct", "bd_loss_sum"):
        assert torch.equal(getattr(a, t).view(torch.uint8), getattr(b, t).view(torch.uint8)), t
    assert (a.status() == b.status()).all() and not b.status().any()
    ra, rb = a.results(), b.results()
    for x, y in zip(ra, rb):
        assert x["accuracies"] == y["accuracies"] and x["losses"] == y["losses"]
        assert x.get("backdoor_accuracies") == y.get("backdoor_accuracies")
        assert "trace" not in x and y["trace"] is not None
        assert len(y["trace"]["agg_deviation"]) == 4 and np.isfinite(y["trace"]["agg_deviation"]).all()


def test_sweep_trace_equals_eager_recompute(env, pinned_splits):
    bt, _, sweep = env
    E = 4
    sw = small_sweep(sweep, MNIST_GRID, E, False, True)
    for e in range(E):
        sw.client_grads()
        sw.aggregate()
        for bd, rounds in ((False, sw.rounds), (True, sw.backdoor_rounds)):
            for r, (sl, rnd) in rounds.items():
                agg = rnd.krum_rows if r == "Krum" else rnd.out[r]
                m = rnd.attack_metrics(aggregated=agg, selection=rnd.selection if r == "Bulyan" else None)
                row0 = rnd.attack_metrics(krum_index=torch.zeros(rnd.B, dtype=torch.int32, device="cuda"))
                fs = torch.tensor([x.corrupted_count for x in sw.experiments[sl]], device="cuda")
                assert torch.equal(bits(sw.trace["agg_deviation"][e, sl]), bits(m["rel_deviation"])), (e, r)
                got = sw.trace["malicious_deviation"][e, sl]
                assert torch.equal(bits(got[fs > 0]), bits(row0["rel_deviation"][fs > 0])), (e, r)
                assert torch.isnan(got[fs == 0]).all()
                if bd:                                             # row 0 is the crafted vector
                    cr = rnd.attack_metrics(aggregated=rnd.crafted)["rel_deviation"]
                    assert torch.equal(bits(got[fs > 0]), bits(cr[fs > 0])), (e, r)
                if r == "Krum":
                    assert torch.equal(sw.trace["krum_index"][e, sl], rnd.krum_index)
                if r == "Bulyan":
                    frac = (sw.trace["bulyan_malicious"][e, sl].float() /
                            sw.trace["bulyan_selected"][e, sl].clamp(min=1).float())
                    assert torch.equal(bits(frac), bits(m["bulyan_malicious_fraction"])), e
        sw.epoch_counter.add_(1)
        if sw.is_test_epoch(e):
            sw.test_epoch()
    cap = small_sweep(sweep, MNIST_GRID, E, True, True)
    for e in range(E):
        cap.step(e)
    torch.cuda.synchronize()
    for k in NAMES:
        assert torch.equal(bits(sw.trace[k]), bits(cap.trace[k])), k
    res = cap.results()
    for r in res:
        e, tr = r["experiment"], r["trace"]
        assert set(tr) >= {"agg_deviation", "malicious_deviation"}
        assert ("krum_malicious" in tr) == (e.defense == "Krum")
        assert ("bulyan_malicious_fraction" in tr) == (e.defense == "Bulyan")


def test_epoch0_against_harness(env, tmp_path):
    from oracle import c_oracle as co
    _, harness, sweep = env
    exps = [("Krum", 0.1, 1.0, 10, 0), ("Krum", 0.24, 0.5, 10, 1), ("Bulyan", 0.1, 1.5, 11, 0),
            ("TrimmedMean", 0.24, 1.0, 10, 1), ("NoDefense", 0.0, 1.0, 10, 0)]
    kw = dict(batch_size=83, train_size=2000, test_size=500)
    sw = sweep.Sweep(exps, 1, capture=False, trace=True, **kw)
    sw.step(0)
    res = sw.results()
    for i, (r, e) in enumerate(zip(res, exps)):
        out = harness.main(e[1], e[2], e[0], users_count=e[3], epochs=1, seed=e[4], out_dir=str(tmp_path),
                           output=str(tmp_path / "log.txt"), trace=True, **kw)
        assert len(out) == 4
        want, got = out[3], r["trace"]
        assert os.path.exists(out[2][:-4] + "_trace.csv")
        if e[0] == "Krum":
            b = sw.order.index(i)
            G = sw.G[b, :e[3]].cpu().numpy()
            k, margin = co.krum_select(np.sqrt(co.pairwise_sqdist(np.ascontiguousarray(G))), e[3],
                                       sweep.Experiment(*e).corrupted_count, with_margin=True)
            if margin > 1e-5:
                assert int(got["krum_index"][0]) == int(want["krum_index"][0]) == k
            else:
                continue
        if e[0] == "Bulyan":
            assert got["bulyan_malicious_fraction"][0] == want["bulyan_malicious_fraction"][0]
        for key in ("agg_deviation", "malicious_deviation"):
            g, w = float(got[key][0]), float(want[key][0])
            assert (np.isnan(g) and np.isnan(w)) or abs(g - w) <= 1e-4 * abs(w), (e, key, g, w)


def test_failed_experiment_gets_no_trace(env, pinned_splits):
    _, _, sweep = env
    failing = ("Bulyan", 0.1, 1.0, 10, 0)
    others = [("Bulyan", 0.1, 1.5, 12, 1), ("TrimmedMean", 0.24, 1.0, 10, 0), ("Krum", 0.1, 0.5, 10, 1)]
    runs = []
    for exps in ([failing] + others, others):
        sw = small_sweep(sweep, exps, 4, True, True)
        sw.step(0)
        if len(exps) > len(others):
            sw.W[sw.order.index(0)] = float("nan")                 # every distance NaN: no eligible user
        for e in range(1, 4):
            sw.step(e)
        runs.append(sw.results())
    ra, rb = runs
    assert isinstance(ra[0]["error"], KeyError) and ra[0]["trace"] is None
    for x, y in zip(ra[1:], rb):
        assert x["error"] is None and y["error"] is None
        assert x["trace"].keys() == y["trace"].keys()
        for k in x["trace"]:
            assert np.array_equal(x["trace"][k].view(np.uint8), y["trace"][k].view(np.uint8)), k
