"""CPU checks of the training sweep (sweep.py, csrc/client_grad.cu): the new entry points' argument checks, the grid
and its up-front rejections, the CSV names, the closed-form minibatch position against harness.Client's stepping, and
the shared setup helper against harness.main's initial weights."""
import ctypes

import numpy as np
import pytest
import torch

D = 79_510
P = ctypes.c_void_p(256)                 # a non-NULL pointer that is never dereferenced


@pytest.fixture(scope="module")
def lib():
    import __graft_entry__ as g
    g.build()
    from attacking_federate_learning_b200 import _native
    return _native.lib()


def grads(lib, **kw):
    a = dict(weights=P, batch=2, d=D, x=P, y=P, n_sets=1, n_train=100, data_index=P, rows=P, n=10, m=83, epoch=P, G=P,
             batch_stride=10 * 79_520, ld=79_520, stream=None)
    a.update(kw)
    return lib.afl_mnist_client_grads(*a.values())


def evaluate(lib, **kw):
    a = dict(weights=P, batch=2, d=D, x=P, y=P, n_sets=1, n_test=100, data_index=P, m=83, slot=P, n_slots=1,
             loss_sum=P, correct=P, ws=P, ws_bytes=1 << 20, stream=None)
    a.update(kw)
    return lib.afl_mnist_evaluate(*a.values())


def test_client_grads_rejects_bad_arguments_before_any_cuda_call(lib):
    from attacking_federate_learning_b200 import _native as nat
    for name in ("weights", "x", "y", "data_index", "rows", "epoch", "G"):
        assert grads(lib, **{name: None}) == nat.AFL_ERR_BAD_ARG, name
    assert grads(lib, d=D + 1) == nat.AFL_ERR_UNSUPPORTED
    assert b"79510" in lib.afl_last_error()
    assert grads(lib, m=129) == nat.AFL_ERR_UNSUPPORTED
    assert grads(lib, m=0) == nat.AFL_ERR_BAD_ARG
    assert grads(lib, n=1025) == nat.AFL_ERR_UNSUPPORTED
    assert grads(lib, n=0) == nat.AFL_ERR_BAD_ARG
    assert grads(lib, n=101) == nat.AFL_ERR_BAD_ARG                      # more clients than training rows
    assert grads(lib, ld=D - 1) == nat.AFL_ERR_BAD_ARG
    assert grads(lib, batch_stride=9 * 79_520) == nat.AFL_ERR_BAD_ARG     # problems would overlap
    assert grads(lib, batch=0) == nat.AFL_ERR_BAD_ARG
    assert grads(lib, batch=65536) == nat.AFL_ERR_UNSUPPORTED


def test_evaluate_rejects_bad_arguments_before_any_cuda_call(lib):
    from attacking_federate_learning_b200 import _native as nat
    for name in ("weights", "x", "y", "data_index", "slot", "loss_sum", "correct", "ws"):
        assert evaluate(lib, **{name: None}) == nat.AFL_ERR_BAD_ARG, name
    assert evaluate(lib, d=D - 1) == nat.AFL_ERR_UNSUPPORTED
    assert evaluate(lib, m=129) == nat.AFL_ERR_UNSUPPORTED
    assert evaluate(lib, n_slots=0) == nat.AFL_ERR_BAD_ARG
    need = lib.afl_mnist_evaluate_workspace_bytes(2, 100, 83)
    assert need >= 2 * 2 * 8
    assert evaluate(lib, ws_bytes=need - 1) == nat.AFL_ERR_WORKSPACE
    assert evaluate(lib, ws=ctypes.c_void_p(128)) == nat.AFL_ERR_WORKSPACE          # not 256-byte aligned
    assert lib.afl_mnist_evaluate_workspace_bytes(0, 100, 83) == 0


def test_grid_keeps_valid_cells_and_drops_what_main_py_rejects():
    from attacking_federate_learning_b200 import sweep
    kept, dropped = sweep.grid(["Krum", "Bulyan", "NoDefense"], [1.5], [0.1, 0.24], [10], [0, 1])
    assert len(kept) + len(dropped) == 3 * 2 * 2
    bad = {(c[0], c[1]) for c, _ in dropped}
    assert bad == {("Bulyan", 0.24)}                                       # n = 10 < 4 * 2 + 3
    assert all(isinstance(e, AssertionError) for _, e in dropped)
    assert kept[0] == sweep.Experiment("Krum", 0.1, 1.5, 10, 0)
    assert [k.seed for k in kept[:2]] == [0, 1]


@pytest.mark.parametrize("exp, exc", [
    (("Median", 0.1, 1.0, 10, 0), KeyError),
    (("Krum", 0.1, 1.0, 0, 0), ValueError),
    (("Krum", 0.1, 1.0, 1025, 0), NotImplementedError),
    (("Krum", 0.5, 1.0, 10, 0), AssertionError),                           # 10 < 2 * 5 + 1
    (("Bulyan", 0.24, 1.0, 10, 0), AssertionError),                        # 10 < 4 * 2 + 3
])
def test_check_raises_what_main_py_raises(exp, exc):
    from attacking_federate_learning_b200 import sweep
    with pytest.raises(exc) as e:
        sweep.check(exp)
    if exc is AssertionError:
        assert str(exp[0]) in str(e.value) and "Experiment" in str(e.value)


def test_run_rejects_before_any_gpu_work():
    from attacking_federate_learning_b200 import sweep
    with pytest.raises(AssertionError):
        sweep.run([("Krum", 0.1, 1.0, 10, 0), ("Bulyan", 0.24, 1.0, 10, 0)], 1, device="cpu")
    with pytest.raises(NotImplementedError):
        sweep.run([("Krum", 0.1, 1.0, 10, 0)], 1, batch_size=129, device="cpu")
    with pytest.raises(ValueError):
        sweep.run([("Krum", 0.1, 1.0, 10, 0)], 1, batch_size=0, device="cpu")


def test_csv_names_are_the_harness_names_with_the_seed():
    from attacking_federate_learning_b200 import harness, sweep
    e = sweep.Experiment("TrimmedMean", 0.24, 1.5, 10, 3)
    assert sweep.csv_name(e, 0.1) == "SYNTH-MNIST_stdev_1.5_TrimmedMean_backdoor-False_mal_prop_0.24_users_10_alpha_None" \
                                     "_lr_0.1_seed_3.csv"
    assert sweep.csv_name(e, 0.1) == harness.csv_name(1.5, "TrimmedMean", False, 0.24, 10, 4, 0.1)[:-4] + "_seed_3.csv"


@pytest.mark.parametrize("n, n_train, m, users", [
    (1, 24, 8, [0]),                     # L = 24: m divides it
    (1, 25, 8, [0]),                     # a 1-row tail
    (7, 100, 5, [0, 1, 2, 6]),           # L = 15 (u < 2) and 14
    (7, 100, 3, [0, 3, 6]),
    (10, 2000, 83, [0, 9]),              # the C1 shape: L = 200, tail of 34
    (1000, 2500, 2, [0, 499, 500, 999]), # L = 3 and 2
])
def test_closed_form_minibatch_equals_client_stepping(n, n_train, m, users):
    from attacking_federate_learning_b200 import harness, sweep
    torch.manual_seed(0)
    x, y = torch.randn(n_train, 784), torch.randint(0, 10, (n_train,))
    net = harness.MnistNet()
    layout = harness.ParamLayout(net.parameters())
    w = layout.flatten(list(net.parameters()))
    row = torch.empty(layout.dim)
    for u in users:
        c = harness.Client(u, False, x[u::n], y[u::n], m, layout, "cpu")
        L = len(c.x)
        steps = 3 * -(-L // m) + 2                                          # three wraps and a bit
        for e in range(steps):
            lo = c.pos
            c.step(w, 0.1, row)
            hi = c.pos if c.pos else L
            assert sweep.minibatch(n_train, n, u, m, e) == (lo, hi), (n, u, e)


def test_setup_helper_gives_harness_main_initial_weights(monkeypatch):
    from attacking_federate_learning_b200 import harness

    class Stop(Exception):
        pass
    seen = {}

    def fake_server(*a, initial_weights=None, **k):
        seen["w"] = initial_weights.clone()
        raise Stop
    monkeypatch.setattr(harness, "AggregationServer", fake_server)
    for seed in (0, 5):
        with pytest.raises(Stop):
            harness.main(0.24, 1.5, "Krum", users_count=10, epochs=1, device="cpu", seed=seed, train_size=200,
                         test_size=40, output=None)
        torch.manual_seed(1234)                                             # the helper must reseed
        (xtr, _), (xte, _), net = harness.experiment_setup(seed, 200, 40, "cpu")
        w = harness.ParamLayout(net.parameters()).flatten(list(net.parameters()))
        assert torch.equal(w.view(torch.int32), seen["w"].view(torch.int32))
        assert torch.equal(xtr, harness.synthetic_problem(200, 40, "cpu", seed)[0][0])
