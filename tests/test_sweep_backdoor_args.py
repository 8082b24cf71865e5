"""CPU checks of the backdoor sweep (sweep.py, csrc/backdoor_train.cu, the _dev backdoor crafting): the backdoor axis of
`check` and `grid`, CSV names and the summary header, the backdoor sets packed for the trainer against
BackdoorTrainer's, the device learning-rate formula against the harness's, and the new entry points' host-side
rejections."""
import ctypes

import numpy as np
import pytest
import torch

D = 79_510
P = ctypes.c_void_p(256)                 # a non-NULL pointer that is never dereferenced
Q = ctypes.c_void_p(1 << 40)             # another one, far from P


@pytest.fixture(scope="module")
def lib():
    import __graft_entry__ as g
    g.build()
    from attacking_federate_learning_b200 import _native
    return _native.lib()


@pytest.mark.parametrize("bd, want", [("pattern", "pattern"), (1, 1), ("2", 2), (np.int64(3), 3)])
def test_check_accepts_and_normalises_backdoors(bd, want):
    from attacking_federate_learning_b200 import sweep
    e = sweep.check(("Krum", 0.1, 1.5, 10, 0, bd))
    assert e == ("Krum", 0.1, 1.5, 10, 0, want) and e.backdoor == want and len(e) == 6
    assert "backdoor=" in repr(e) and e.corrupted_count == 1


@pytest.mark.parametrize("bd", [False, "No"])
def test_a_drift_experiment_is_the_five_tuple(bd):
    from attacking_federate_learning_b200 import sweep
    e = sweep.check(("Krum", 0.1, 1.5, 10, 0, bd))
    assert e == ("Krum", 0.1, 1.5, 10, 0) == sweep.Experiment("Krum", 0.1, 1.5, 10, 0)
    assert len(e) == 5 and e.backdoor is False and list(e) == ["Krum", 0.1, 1.5, 10, 0]
    assert repr(e) == "Experiment(defense='Krum', mal_prop=0.1, num_std=1.5, users_count=10, seed=0)"
    assert sweep.Experiment(*e) == e and hash(e) == hash(tuple(e))


@pytest.mark.parametrize("cell, exc", [
    (("Krum", 0.1, 1.5, 10, 0, "square"), ValueError),
    (("Krum", 0.1, 1.5, 10, 0, 0), ValueError),
    (("Krum", 0.1, 1.5, 10, 0, 4), ValueError),
    (("Krum", 0.1, 1.5, 10, 0, True), ValueError),
    (("Krum", 0.1, 1.5, 10, 0, None), ValueError),
    (("Krum", 0.1, 1.5, 10, 0, "pattern", 1), ValueError),
    (("Krum", 0.1, 1.5, 10), ValueError),
])
def test_check_rejects_unknown_backdoors(cell, exc):
    from attacking_federate_learning_b200 import sweep
    with pytest.raises(exc):
        sweep.check(cell)


def test_check_rejects_a_sample_past_the_training_set():
    from attacking_federate_learning_b200 import sweep
    assert sweep.check(("NoDefense", 0.1, 1.0, 2, 0, 3), train_size=3).backdoor == 3
    with pytest.raises(ValueError, match="past the training set"):
        sweep.check(("NoDefense", 0.1, 1.0, 2, 0, 3), train_size=2)


def test_grid_with_a_backdoor_axis():
    from attacking_federate_learning_b200 import sweep
    kept, dropped = sweep.grid(["Krum", "Bulyan"], [1.0], [0.24], [10], [0, 1], backdoors=(False, "pattern", 2))
    bds = ((), ("pattern",), (2,))
    assert [tuple(e) for e in kept] == [("Krum", 0.24, 1.0, 10, s, *b) for s in (0, 1) for b in bds]
    assert [c for c, _ in dropped] == [("Bulyan", 0.24, 1.0, 10, s, *b) for s in (0, 1) for b in bds]   # 10 < 4*2+3
    assert all(isinstance(e, AssertionError) for _, e in dropped)
    kept0, _ = sweep.grid(["Krum"], [1.0], [0.1], [10], [0])
    assert kept0 == [("Krum", 0.1, 1.0, 10, 0)] and len(kept0[0]) == 5


def test_csv_names_are_the_harness_names_with_the_seed():
    from attacking_federate_learning_b200 import harness, sweep
    for bd in ("pattern", 1, 3):
        e = sweep.Experiment("Krum", 0.24, 1.0, 10, 7, bd)
        assert sweep.csv_name(e, 0.1) == harness.csv_name(1.0, "Krum", bd, 0.24, 10, 4, 0.1)[:-4] + "_seed_7.csv"
    assert sweep.csv_name(sweep.Experiment("Krum", 0.24, 1.0, 10, 7, "pattern"), 0.1) == \
        "SYNTH-MNIST_stdev_1.0_Krum_backdoor-pattern_mal_prop_0.24_users_10_alpha_4_lr_0.1_seed_7.csv"
    e = sweep.Experiment("Krum", 0.24, 1.0, 10, 7)
    assert sweep.csv_name(e, 0.1) == harness.csv_name(1.0, "Krum", False, 0.24, 10, 4, 0.1)[:-4] + "_seed_7.csv"


def test_summary_header():
    from attacking_federate_learning_b200 import sweep
    assert sweep.summary_header(False) == ["defense", "mal_prop", "num_std", "users_count", "seed", "max_accuracy",
                                           "final_accuracy", "status"]
    assert sweep.summary_header(True) == ["defense", "mal_prop", "num_std", "users_count", "seed", "backdoor",
                                          "max_accuracy", "final_accuracy", "max_backdoor_accuracy",
                                          "final_backdoor_accuracy", "status"]


def test_backdoor_sets_equal_the_trainers():
    from attacking_federate_learning_b200 import harness, sweep
    specs, want = [], []
    for n_train in (2000, 3300, 5000, 20000):            # pattern lengths 2000, 3300, 2500 and 2000
        for seed in (0, 3, 11):
            (x, y), _, net = harness.experiment_setup(seed, n_train, 10, "cpu")
            layout = harness.ParamLayout(net.parameters())
            for bd in ("pattern", 1, 2, 3):
                tr = harness.BackdoorTrainer(bd, 4, 5, layout, x, y, "cpu", print, seed)
                specs.append((bd, x, y, seed))
                want.append((tr.x, tr.y))
    xs, ys, lens = sweep.backdoor_sets(specs)
    assert xs.dtype == torch.float32 and ys.dtype == torch.int64 and lens.dtype == torch.int32
    assert any(int(n) % sweep.BACKDOOR_BATCH for n in lens)                   # a tail minibatch is covered
    for k, (x, y) in enumerate(want):
        n = int(lens[k])
        assert n == len(x) == len(y)
        assert torch.equal(xs[k, :n], x) and torch.equal(ys[k, :n], y)
        assert not xs[k, n:].any() and not ys[k, n:].any()


def test_device_lr_formula_equals_the_harness():
    from attacking_federate_learning_b200 import sweep
    for lr, fr in ((0.1, 10000), (0.05, 10000), (0.3, 7), (0.1, 1)):
        got = sweep.fading_lr(torch.arange(301, dtype=torch.int32), lr, fr)
        assert got.dtype == torch.float64
        want = [lr * fr / (epoch + fr) for epoch in range(301)]            # harness.main's Python doubles
        assert got.tolist() == want


def test_nan_status_codes_are_the_reference_exceptions():
    from attacking_federate_learning_b200 import _native as nat, sweep
    e = sweep.status_error(nat.AFL_ERR_NAN_LOSS, "experiment x")
    assert type(e) is Exception and str(e) == "experiment x: Got nan loss"
    e = sweep.status_error(nat.AFL_ERR_NAN_DIST_LOSS, "experiment x")
    assert type(e) is Exception and str(e) == "experiment x: Got nan dist loss"


def train(lib, **kw):
    a = dict(initial=P, out=Q, batch=2, d=D, x=P, y=P, n_sets=1, max_len=200, set_len=P, data_index=P, f=P, z=P,
             status=P, alpha=4.0, mal_epochs=5, m=200, stream=None)
    a.update(kw)
    return lib.afl_mnist_backdoor_train(*a.values())


def btest(lib, **kw):
    a = dict(weights=P, batch=2, d=D, x=P, y=P, n_sets=1, max_len=200, set_len=P, data_index=P, m=200, slot=P,
             n_slots=1, loss_sum=P, correct=P, stream=None)
    a.update(kw)
    return lib.afl_mnist_backdoor_test(*a.values())


def test_trainer_rejects_bad_arguments_before_any_cuda_call(lib):
    from attacking_federate_learning_b200 import _native as nat
    for name in ("initial", "out", "x", "y", "set_len", "data_index", "f", "z", "status"):
        assert train(lib, **{name: None}) == nat.AFL_ERR_BAD_ARG, name
    assert train(lib, d=D - 1) == nat.AFL_ERR_UNSUPPORTED
    assert train(lib, m=201) == nat.AFL_ERR_UNSUPPORTED
    assert train(lib, batch=65536) == nat.AFL_ERR_UNSUPPORTED
    for k in ("batch", "n_sets", "max_len", "m"):
        assert train(lib, **{k: 0}) == nat.AFL_ERR_BAD_ARG, k
    assert train(lib, mal_epochs=-1) == nat.AFL_ERR_BAD_ARG
    assert train(lib, alpha=float("nan")) == nat.AFL_ERR_BAD_ARG
    assert train(lib, out=ctypes.c_void_p(256 + 4 * D)) == nat.AFL_ERR_BAD_ARG          # overlaps problem 1's initial
    assert b"overlaps" in lib.afl_last_error()


def test_backdoor_test_rejects_bad_arguments_before_any_cuda_call(lib):
    from attacking_federate_learning_b200 import _native as nat
    for name in ("weights", "x", "y", "set_len", "data_index", "slot", "loss_sum", "correct"):
        assert btest(lib, **{name: None}) == nat.AFL_ERR_BAD_ARG, name
    assert btest(lib, d=D + 1) == nat.AFL_ERR_UNSUPPORTED
    assert btest(lib, m=201) == nat.AFL_ERR_UNSUPPORTED
    assert btest(lib, batch=65536) == nat.AFL_ERR_UNSUPPORTED
    assert btest(lib, n_slots=0) == nat.AFL_ERR_BAD_ARG


def start_dev(lib, **kw):
    a = dict(G=P, batch=2, bs=10 * 256, n=10, d=200, ld=256, dtype=0, f=P, z=P, lr=P, w=P, w_bs=0, mu=P, sigma=P,
             initial=P, ws=P, ws_bytes=1 << 20, status=P, stream=None)
    a.update(kw)
    return lib.afl_backdoor_start_batched_dev(*a.values())


def finish_dev(lib, **kw):
    a = dict(batch=2, n=10, d=200, f=P, z=P, lr=P, mu=P, sigma=P, initial=P, mal=P, mal_bs=200, crafted=P, bcast=P,
             bcast_bs=10 * 256, bcast_ld=256, ws=P, ws_bytes=1 << 20, status=P, stream=None)
    a.update(kw)
    return lib.afl_backdoor_finish_batched_dev(*a.values())


def test_dev_crafting_rejects_bad_arguments_before_any_cuda_call(lib):
    from attacking_federate_learning_b200 import _native as nat
    for name in ("G", "f", "z", "lr", "w", "mu", "sigma", "initial", "status"):
        assert start_dev(lib, **{name: None}) == nat.AFL_ERR_BAD_ARG, name
    assert start_dev(lib, w_bs=199) == nat.AFL_ERR_BAD_ARG
    assert start_dev(lib, bs=9 * 256) == nat.AFL_ERR_BAD_ARG
    assert start_dev(lib, dtype=7) == nat.AFL_ERR_UNSUPPORTED
    assert start_dev(lib, batch=65536) == nat.AFL_ERR_UNSUPPORTED
    assert start_dev(lib, ws_bytes=64) == nat.AFL_ERR_WORKSPACE
    assert start_dev(lib, ws=ctypes.c_void_p(257)) == nat.AFL_ERR_WORKSPACE
    for name in ("f", "z", "lr", "mu", "sigma", "initial", "mal", "crafted", "status"):
        assert finish_dev(lib, **{name: None}) == nat.AFL_ERR_BAD_ARG, name
    assert finish_dev(lib, n=0) == nat.AFL_ERR_BAD_ARG
    assert finish_dev(lib, mal_bs=199) == nat.AFL_ERR_BAD_ARG
    assert finish_dev(lib, bcast_bs=9 * 256) == nat.AFL_ERR_BAD_ARG
    assert finish_dev(lib, bcast_ld=199) == nat.AFL_ERR_BAD_ARG
    assert finish_dev(lib, batch=65536) == nat.AFL_ERR_UNSUPPORTED
    assert finish_dev(lib, ws_bytes=64) == nat.AFL_ERR_WORKSPACE
