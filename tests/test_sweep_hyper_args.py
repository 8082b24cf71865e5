"""CPU checks of per-experiment learning rates and batch sizes in training sweeps (sweep.py, the _each entry points in
csrc/client_grad.cu and csrc/cifar_grad.cu, afl_momentum_step_batched in csrc/colstats.cu): the 5-, 6- and 8-tuple
experiments, the grid's shape and order, the per-experiment batch-size rule, CSV names and summary headers, the CLI
with one and with several values, and the new entry points' host-side rejections."""
import ctypes
import itertools

import pytest

P = ctypes.c_void_p(256)                 # a non-NULL pointer that is never dereferenced
NETS = {"mnist": 79_510, "cifar10": 117_706}


@pytest.fixture(scope="module")
def lib():
    import __graft_entry__ as g
    g.build()
    from attacking_federate_learning_b200 import _native
    return _native.lib()


def test_short_forms_are_unchanged():
    from attacking_federate_learning_b200.sweep import Experiment
    e5 = Experiment("Krum", 0.24, 1.5, 10, 0)
    assert e5 == ("Krum", 0.24, 1.5, 10, 0) and len(e5) == 5
    assert repr(e5) == "Experiment(defense='Krum', mal_prop=0.24, num_std=1.5, users_count=10, seed=0)"
    e6 = Experiment("Krum", 0.24, 1.5, 10, 0, "pattern")
    assert e6 == ("Krum", 0.24, 1.5, 10, 0, "pattern")
    assert repr(e6).endswith("seed=0, backdoor='pattern')")
    for e in (e5, e6):
        assert e.learning_rate is None and e.batch_size is None


def test_the_eight_tuple():
    from attacking_federate_learning_b200.sweep import Experiment
    e = Experiment("Krum", 0.24, 1.5, 10, 0, False, 0.05, 32)
    assert e == ("Krum", 0.24, 1.5, 10, 0, False, 0.05, 32) and len(e) == 8
    assert e.backdoor is False and e.learning_rate == 0.05 and e.batch_size == 32
    assert repr(e) == ("Experiment(defense='Krum', mal_prop=0.24, num_std=1.5, users_count=10, seed=0, "
                       "backdoor=False, learning_rate=0.05, batch_size=32)")
    b = Experiment("Krum", 0.24, 1.5, 10, 0, 2, 0.2, 128)
    assert b.backdoor == 2 and b[5:] == (2, 0.2, 128)
    assert Experiment(*e) == e
    with pytest.raises(ValueError):
        Experiment("Krum", 0.24, 1.5, 10, 0, False, 0.05)


def test_check_normalises_eight_tuples_and_their_batch_size():
    from attacking_federate_learning_b200 import sweep
    e = sweep.check(("Krum", "0.24", 1.5, "10", 0, "No", "0.05", "32"))
    assert e == ("Krum", 0.24, 1.5, 10, 0, False, 0.05, 32) and isinstance(e.batch_size, int)
    assert sweep.check(("Krum", 0.24, 1.5, 10, 0, "1", 0.1, 128)).backdoor == 1
    # the 8-tuple's own batch size is checked, not the run's
    assert sweep.check(("Krum", 0.24, 1.5, 10, 0, False, 0.1, 128), batch_size=500).batch_size == 128
    with pytest.raises(ValueError):
        sweep.check(("Krum", 0.24, 1.5, 10, 0, False, 0.1, 0))
    with pytest.raises(NotImplementedError):
        sweep.check(("Krum", 0.24, 1.5, 10, 0, False, 0.1, 129))
    with pytest.raises(NotImplementedError):                               # a short tuple keeps the run's rule
        sweep.check(("Krum", 0.24, 1.5, 10, 0), batch_size=129)
    with pytest.raises(ValueError):
        sweep.check(("Krum", 0.24, 1.5, 10, 0, False, 0.1))                 # 7 elements


def test_grid_shapes_and_order():
    from attacking_federate_learning_b200 import sweep
    kept, dropped = sweep.grid(["Krum", "NoDefense"], [1.5], [0.24], [10], [0, 1], backdoors=[False, "pattern"],
                               learning_rates=[0.05, 0.1], batch_sizes=[32, 83, 129])
    cells = list(itertools.product(["Krum", "NoDefense"], [0.24], [1.5], [10], [0, 1], [False, "pattern"],
                                   [0.05, 0.1], [32, 83]))
    assert kept == cells and all(len(e) == 8 for e in kept)
    assert len(dropped) == 16 and all(c[7] == 129 and isinstance(e, NotImplementedError) for c, e in dropped)
    # the one not given is the run's
    kept, _ = sweep.grid(["Krum"], [1.5], [0.24], [10], [0], batch_size=64, learning_rates=[0.05, 0.2])
    assert kept == [("Krum", 0.24, 1.5, 10, 0, False, 0.05, 64), ("Krum", 0.24, 1.5, 10, 0, False, 0.2, 64)]
    kept, _ = sweep.grid(["Krum"], [1.5], [0.24], [10], [0], batch_sizes=[16], learning_rate=0.3)
    assert kept == [("Krum", 0.24, 1.5, 10, 0, False, 0.3, 16)]
    # neither given: today's tuples
    kept, _ = sweep.grid(["Krum"], [1.5], [0.24], [10], [0], backdoors=[False, 1])
    assert kept == [("Krum", 0.24, 1.5, 10, 0), ("Krum", 0.24, 1.5, 10, 0, 1)]


def test_csv_names():
    from attacking_federate_learning_b200 import harness, sweep
    e5 = sweep.Experiment("Krum", 0.24, 1.5, 10, 3)
    assert sweep.csv_name(e5, 0.1) == harness.csv_name(1.5, "Krum", False, 0.24, 10, 4, 0.1)[:-4] + "_seed_3.csv"
    e8 = sweep.Experiment("Krum", 0.24, 1.5, 10, 3, False, 0.05, 32)
    want = harness.csv_name(1.5, "Krum", False, 0.24, 10, 4, 0.05)[:-4] + "_batch_32_seed_3.csv"
    assert sweep.csv_name(e8, 0.1) == want                                 # its own lr, not the run's
    b8 = sweep.Experiment("Krum", 0.24, 1.5, 10, 3, "pattern", 0.2, 128)
    assert sweep.csv_name(b8, 0.1, dataset="CIFAR10") == \
        harness.csv_name(1.5, "Krum", "pattern", 0.24, 10, 4, 0.2, "CIFAR10")[:-4] + "_batch_128_seed_3.csv"
    names = {sweep.csv_name(sweep.Experiment("Krum", 0.24, 1.5, 10, 3, False, 0.1, c), 0.1) for c in (32, 83, 128)}
    assert len(names) == 3


def test_summary_headers():
    from attacking_federate_learning_b200 import sweep
    base = ["defense", "mal_prop", "num_std", "users_count", "seed"]
    assert sweep.summary_header(False) == sweep.summary_header(False, False) == \
        base + ["max_accuracy", "final_accuracy", "status"]
    assert sweep.summary_header(False, True) == base + ["learning_rate", "batch_size", "max_accuracy",
                                                       "final_accuracy", "status"]
    assert sweep.summary_header(True, True) == base + ["backdoor", "learning_rate", "batch_size", "max_accuracy",
                                                      "final_accuracy", "max_backdoor_accuracy",
                                                      "final_backdoor_accuracy", "status"]


def test_per_problem_lr_products_equal_the_harness():
    import torch
    from attacking_federate_learning_b200 import sweep
    lrs, fr = [0.05, 0.1, 0.2, 0.3], 10000
    num = sweep.lr_products(lrs, fr, "cpu")
    epoch = torch.tensor([7], dtype=torch.int32)
    got = sweep.fading_lr(epoch, num, fr)
    assert got.tolist() == [lr * fr / (7 + fr) for lr in lrs]
    out = torch.empty(4, dtype=torch.float64)
    sweep.fading_lr(epoch, num, fr, out=out)
    assert out.tolist() == got.tolist()


def _cli(monkeypatch, argv):
    from attacking_federate_learning_b200 import sweep
    seen = {}
    real_grid = sweep.grid

    def fake_grid(*a, **kw):
        seen["grid"] = (a, kw)
        return real_grid(*a, **kw)

    def fake_run(kept, epochs, lr, **kw):
        seen["run"] = (kept, epochs, lr, kw)
        return []
    monkeypatch.setattr(sweep, "grid", fake_grid)
    monkeypatch.setattr(sweep, "run", fake_run)
    sweep.main(argv)
    return seen


def test_cli_with_one_value_calls_grid_and_run_as_before(monkeypatch):
    seen = _cli(monkeypatch, ["-d", "Krum", "-z", "1.0", "-e", "3", "-l", "0.05", "-c", "32"])
    a, kw = seen["grid"]
    assert a == (["Krum"], [1.0], [0.24], [10], [0], 32, 20000)
    assert kw == dict(backdoors=[False], dataset="MNIST", cifar10_backdoor=False)
    kept, epochs, lr, kw = seen["run"]
    assert kept == [("Krum", 0.24, 1.0, 10, 0)] and epochs == 3 and lr == 0.05 and kw["batch_size"] == 32
    seen = _cli(monkeypatch, ["-d", "Krum", "-e", "3"])                     # the defaults
    assert seen["grid"][0][5] == 83 and seen["run"][2] == 0.1 and seen["run"][3]["batch_size"] == 83


def test_cli_with_several_values_gives_eight_tuples(monkeypatch):
    seen = _cli(monkeypatch, ["-d", "Krum", "-z", "1.0", "-e", "3", "-l", "0.05", "0.2", "-c", "32", "83", "128"])
    kept = seen["run"][0]
    assert kept == [("Krum", 0.24, 1.0, 10, 0, False, lr, c) for lr in (0.05, 0.2) for c in (32, 83, 128)]
    seen = _cli(monkeypatch, ["-d", "Krum", "-e", "3", "-c", "32", "64"])   # one lr, several batch sizes
    assert seen["run"][0] == [("Krum", 0.24, 1.5, 10, 0, False, 0.1, c) for c in (32, 64)]


def grads_each(lib, net, **kw):
    d = NETS[net]
    ld = (d + 31) // 32 * 32
    a = dict(weights=P, batch=2, d=d, x=P, y=P, n_sets=1, n_rows=100, set_len=P, data_index=P, rows=P, n=10, m=P,
             max_m=83, epoch=P, G=P, batch_stride=10 * ld, ld=ld, stream=None)
    a.update(kw)
    return getattr(lib, f"afl_{net}_client_grads_each")(*a.values())


def evaluate_each(lib, net, **kw):
    a = dict(weights=P, batch=2, d=NETS[net], x=P, y=P, n_sets=1, n_test=10_000, data_index=P, m=P, min_m=16,
             max_m=83, slot=P, n_slots=1, loss_sum=P, correct=P, ws=P, ws_bytes=1 << 20, stream=None)
    a.update(kw)
    return getattr(lib, f"afl_{net}_evaluate_each")(*a.values())


@pytest.mark.parametrize("net", sorted(NETS))
def test_client_grads_each_rejects_bad_arguments_before_any_cuda_call(lib, net):
    from attacking_federate_learning_b200 import _native as nat
    for name in ("weights", "x", "y", "set_len", "data_index", "rows", "m", "epoch", "G"):
        assert grads_each(lib, net, **{name: None}) == nat.AFL_ERR_BAD_ARG, name
    assert grads_each(lib, net, d=NETS[net] + 1) == nat.AFL_ERR_UNSUPPORTED
    assert grads_each(lib, net, max_m=129) == nat.AFL_ERR_UNSUPPORTED
    assert b"m <= 128" in lib.afl_last_error()
    assert grads_each(lib, net, max_m=0) == nat.AFL_ERR_BAD_ARG
    assert grads_each(lib, net, n=1025) == nat.AFL_ERR_UNSUPPORTED
    assert grads_each(lib, net, n=101) == nat.AFL_ERR_BAD_ARG
    assert grads_each(lib, net, batch=65536) == nat.AFL_ERR_UNSUPPORTED
    assert grads_each(lib, net, batch_stride=9 * 79_520) == nat.AFL_ERR_BAD_ARG
    assert b"_client_grads_each" in lib.afl_last_error()


@pytest.mark.parametrize("net", sorted(NETS))
def test_evaluate_each_rejects_bad_arguments_before_any_cuda_call(lib, net):
    from attacking_federate_learning_b200 import _native as nat
    for name in ("weights", "x", "y", "data_index", "m", "slot", "loss_sum", "correct", "ws"):
        assert evaluate_each(lib, net, **{name: None}) == nat.AFL_ERR_BAD_ARG, name
    assert evaluate_each(lib, net, d=NETS[net] - 1) == nat.AFL_ERR_UNSUPPORTED
    assert evaluate_each(lib, net, max_m=129) == nat.AFL_ERR_UNSUPPORTED
    assert evaluate_each(lib, net, min_m=0) == nat.AFL_ERR_BAD_ARG
    assert evaluate_each(lib, net, min_m=84) == nat.AFL_ERR_BAD_ARG                      # min_m > max_m
    assert evaluate_each(lib, net, n_slots=0) == nat.AFL_ERR_BAD_ARG
    ws_bytes = getattr(lib, f"afl_{net}_evaluate_workspace_bytes")
    need = ws_bytes(2, 10_000, 16)                                                     # the batch count at min_m
    assert need > ws_bytes(2, 10_000, 83)
    assert evaluate_each(lib, net, ws_bytes=need - 1) == nat.AFL_ERR_WORKSPACE
    assert evaluate_each(lib, net, ws_bytes=ws_bytes(2, 10_000, 83)) == nat.AFL_ERR_WORKSPACE
    assert evaluate_each(lib, net, ws=ctypes.c_void_p(128)) == nat.AFL_ERR_WORKSPACE     # not 256-byte aligned
    assert b"_evaluate_each" in lib.afl_last_error()


def test_momentum_step_batched_rejects_bad_arguments_before_any_cuda_call(lib):
    from attacking_federate_learning_b200 import _native as nat

    def step(**kw):
        a = dict(w=P, v=P, g=P, batch=2, d=10, momentum=0.9, lr=P, stream=None)
        a.update(kw)
        return lib.afl_momentum_step_batched(*a.values())
    for name in ("w", "v", "g", "lr"):
        assert step(**{name: None}) == nat.AFL_ERR_BAD_ARG, name
    assert step(batch=0) == nat.AFL_ERR_BAD_ARG
    assert step(d=0) == nat.AFL_ERR_BAD_ARG
    assert step(batch=65536) == nat.AFL_ERR_UNSUPPORTED
