"""CPU checks of the CIFAR10 backdoor sweep (sweep.py with cifar10_backdoor=True, csrc/cifar_backdoor.cu): the new
entry points' host-side rejections and workspace sizes, `check` and `grid` with and without the switch, the backdoor
sets packed for [n, 3, 32, 32] images against BackdoorTrainer's (MNIST's unchanged), and the CLI flag."""
import ctypes

import numpy as np
import pytest
import torch

D = 117_706
P = ctypes.c_void_p(256)                 # a non-NULL pointer that is never dereferenced
Q = ctypes.c_void_p(1 << 40)             # another one, far from P
W = ctypes.c_void_p(1 << 41)             # a workspace far from both


@pytest.fixture(scope="module")
def lib():
    import __graft_entry__ as g
    g.build()
    from attacking_federate_learning_b200 import _native
    return _native.lib()


def train(lib, **kw):
    a = dict(initial=P, out=Q, batch=2, d=D, x=P, y=P, n_sets=1, max_len=200, set_len=P, data_index=P, f=P, z=P,
             status=P, alpha=4.0, mal_epochs=5, m=200, ws=W, ws_bytes=2 * D * 4, stream=None)
    a.update(kw)
    return lib.afl_cifar10_backdoor_train(*a.values())


def btest(lib, **kw):
    a = dict(weights=P, batch=2, d=D, x=P, y=P, n_sets=1, max_len=200, set_len=P, data_index=P, m=200, slot=P,
             n_slots=1, loss_sum=P, correct=P, ws=W, ws_bytes=1 << 20, stream=None)
    a.update(kw)
    return lib.afl_cifar10_backdoor_test(*a.values())


def test_workspace_sizes(lib):
    assert lib.afl_cifar10_backdoor_train_workspace_bytes(1) == D * 4
    assert lib.afl_cifar10_backdoor_train_workspace_bytes(7) == 7 * D * 4              # a slice's rows: b D floats on
    assert lib.afl_cifar10_backdoor_train_workspace_bytes(0) == 0
    assert lib.afl_cifar10_backdoor_test_workspace_bytes(1, 200, 200) == 512           # one batch: two 256-byte tables
    assert lib.afl_cifar10_backdoor_test_workspace_bytes(3, 2500, 200) == 2 * 256      # 3 x 13 entries each
    assert lib.afl_cifar10_backdoor_test_workspace_bytes(100, 2001, 200) == 2 * 4608    # 100 x 11 x 4 = 4400 -> 4608
    for a in ((0, 200, 200), (1, 0, 200), (1, 200, 0)):
        assert lib.afl_cifar10_backdoor_test_workspace_bytes(*a) == 0


def test_trainer_rejects_bad_arguments_before_any_cuda_call(lib):
    from attacking_federate_learning_b200 import _native as nat
    for name in ("initial", "out", "x", "y", "set_len", "data_index", "f", "z", "status", "ws"):
        assert train(lib, **{name: None}) == nat.AFL_ERR_BAD_ARG, name
    assert train(lib, d=D - 1) == nat.AFL_ERR_UNSUPPORTED
    assert train(lib, d=79_510) == nat.AFL_ERR_UNSUPPORTED                              # MnistNet's D
    assert train(lib, m=201) == nat.AFL_ERR_UNSUPPORTED
    assert train(lib, batch=65536) == nat.AFL_ERR_UNSUPPORTED
    for k in ("batch", "n_sets", "max_len", "m"):
        assert train(lib, **{k: 0}) == nat.AFL_ERR_BAD_ARG, k
    assert train(lib, mal_epochs=-1) == nat.AFL_ERR_BAD_ARG
    assert train(lib, alpha=float("nan")) == nat.AFL_ERR_BAD_ARG
    assert train(lib, ws_bytes=2 * D * 4 - 1) == nat.AFL_ERR_BAD_ARG
    assert b"workspace" in lib.afl_last_error()
    assert train(lib, ws=ctypes.c_void_p((1 << 41) + 2)) == nat.AFL_ERR_BAD_ARG         # not float-aligned
    assert train(lib, out=ctypes.c_void_p(256 + 4 * D)) == nat.AFL_ERR_BAD_ARG          # overlaps problem 1's initial
    assert b"overlap" in lib.afl_last_error()
    assert train(lib, ws=ctypes.c_void_p((1 << 40) + 4 * D)) == nat.AFL_ERR_BAD_ARG     # overlaps problem 1's out
    assert train(lib, ws=ctypes.c_void_p(256 - 4)) == nat.AFL_ERR_BAD_ARG               # overlaps initial


def test_backdoor_test_rejects_bad_arguments_before_any_cuda_call(lib):
    from attacking_federate_learning_b200 import _native as nat
    for name in ("weights", "x", "y", "set_len", "data_index", "slot", "loss_sum", "correct", "ws"):
        assert btest(lib, **{name: None}) == nat.AFL_ERR_BAD_ARG, name
    assert btest(lib, d=D + 1) == nat.AFL_ERR_UNSUPPORTED
    assert btest(lib, m=201) == nat.AFL_ERR_UNSUPPORTED
    assert btest(lib, batch=65536) == nat.AFL_ERR_UNSUPPORTED
    for k in ("batch", "n_sets", "max_len", "m"):
        assert btest(lib, **{k: 0}) == nat.AFL_ERR_BAD_ARG, k
    assert btest(lib, n_slots=0) == nat.AFL_ERR_BAD_ARG
    need = lib.afl_cifar10_backdoor_test_workspace_bytes(2, 200, 200)
    assert btest(lib, ws_bytes=need - 1) == nat.AFL_ERR_BAD_ARG
    assert btest(lib, ws=ctypes.c_void_p((1 << 41) + 128)) == nat.AFL_ERR_BAD_ARG       # not 256-byte aligned
    assert btest(lib, max_len=65536 * 200, m=200, ws_bytes=1 << 40) == nat.AFL_ERR_UNSUPPORTED   # 65,536 batches


CELL = ("Krum", 0.1, 1.5, 10, 0, "pattern")


def test_check_takes_cifar10_backdoors_only_with_the_switch():
    from attacking_federate_learning_b200 import sweep
    with pytest.raises(NotImplementedError, match="cifar10_backdoor"):
        sweep.check(CELL, dataset="CIFAR10")
    for bd, want in (("pattern", "pattern"), (1, 1), ("3", 3)):
        e = sweep.check(CELL[:5] + (bd,), dataset="CIFAR10", cifar10_backdoor=True)
        assert e == CELL[:5] + (want,) and e.backdoor == want
    assert sweep.check(CELL[:5], dataset="CIFAR10", cifar10_backdoor=True) == CELL[:5]
    assert sweep.check(CELL, cifar10_backdoor=True) == sweep.check(CELL)                  # MNIST: no change


@pytest.mark.parametrize("cell, kw, exc", [
    (("Krum", 0.5, 1.5, 10, 0, "pattern"), {}, AssertionError),             # n < 2 f + 1
    (("Bulyan", 0.24, 1.5, 10, 0, 1), {}, AssertionError),                  # n < 4 f + 3
    (("NoDefense", 0.1, 1.5, 10, 0, 3), dict(train_size=2), ValueError),    # sample past the training set
    (("NoDefense", 0.1, 1.5, 10, 0, "square"), {}, ValueError),
    (("Median", 0.1, 1.5, 10, 0, "pattern"), {}, KeyError),
    (("NoDefense", 0.1, 1.5, 1025, 0, "pattern"), {}, NotImplementedError),
    (("NoDefense", 0.1, 1.5, 10, 0, "pattern"), dict(batch_size=129), NotImplementedError),
])
def test_other_rejections_still_apply_with_the_switch(cell, kw, exc):
    from attacking_federate_learning_b200 import sweep
    with pytest.raises(exc):
        sweep.check(cell, dataset="CIFAR10", cifar10_backdoor=True, **kw)


def test_grid_keeps_cifar10_backdoor_cells_with_the_switch():
    from attacking_federate_learning_b200 import sweep
    args = (["Krum", "NoDefense"], [1.5], [0.1, 0.5], [10], [0, 1])
    kept, dropped = sweep.grid(*args, backdoors=(False, "pattern", 1), dataset="CIFAR10", cifar10_backdoor=True)
    assert len(kept) == 18 and all(c[0] == "Krum" and c[1] == 0.5 for c, _ in dropped)
    assert len(dropped) == 6 and all(isinstance(e, AssertionError) for _, e in dropped)
    assert [e.backdoor for e in kept[:3]] == [False, "pattern", 1]
    kept_off, dropped_off = sweep.grid(*args, backdoors=(False, "pattern", 1), dataset="CIFAR10")
    assert kept_off == [e for e in kept if e.backdoor is False]
    assert sum(isinstance(e, NotImplementedError) for _, e in dropped_off) == 16      # checked first
    kept_m, _ = sweep.grid(*args, backdoors=(False, "pattern", 1))
    assert kept_m == sweep.grid(*args, backdoors=(False, "pattern", 1), cifar10_backdoor=True)[0]


def test_run_without_the_switch_still_rejects_before_any_gpu_work():
    from attacking_federate_learning_b200 import sweep
    with pytest.raises(NotImplementedError, match="--cifar10-backdoor"):
        sweep.run([("Krum", 0.1, 1.0, 10, 0), CELL], 1, device="cpu", dataset="CIFAR10")
    with pytest.raises(AssertionError):                     # with it, main.py's asserts still come first
        sweep.run([("Krum", 0.5, 1.0, 10, 0, 1)], 1, device="cpu", dataset="CIFAR10", cifar10_backdoor=True)


def test_backdoor_sets_for_cifar10_images_equal_the_trainers():
    from attacking_federate_learning_b200 import harness, sweep
    specs, want = [], []
    for n_train, seed in ((2000, 0), (3300, 3), (500, 11)):       # pattern lengths 2000, 3300 and 500
        (x, y), _, net = harness.experiment_setup(seed, n_train, 10, "cpu", "CIFAR10")
        layout = harness.ParamLayout(net.parameters())
        for bd in ("pattern", 1, 2, 3):
            tr = harness.BackdoorTrainer(bd, 4, 5, layout, x, y, "cpu", print, seed, dataset="CIFAR10")
            specs.append((bd, x, y, seed))
            want.append((tr.x, tr.y))
    xs, ys, lens = sweep.backdoor_sets(specs)
    assert xs.shape == (len(specs), 3300, 3, 32, 32) and xs.is_contiguous()
    assert xs.dtype == torch.float32 and ys.dtype == torch.int64 and lens.dtype == torch.int32
    for k, (x, y) in enumerate(want):
        n = int(lens[k])
        assert n == len(x) == len(y)
        assert torch.equal(xs[k, :n], x) and torch.equal(ys[k, :n], y)
        assert not xs[k, n:].any() and not ys[k, n:].any()
    pat = xs[0, :int(lens[0])]
    assert (pat[:, :, :5, :5] == 2.8).all() and not (pat[:, :, 5:, :] == 2.8).all()   # every channel's corner
    assert (ys[0, :int(lens[0])] == 0).all()


def test_backdoor_sets_for_mnist_are_unchanged():
    from attacking_federate_learning_b200 import harness, sweep
    (x, y), _, _ = harness.experiment_setup(1, 5000, 10, "cpu")
    specs = [("pattern", x, y, 1), (2, x, y, 1)]
    xs, ys, lens = sweep.backdoor_sets(specs)
    assert xs.shape == (2, 2500, 784) and lens.tolist() == [2500, 1]
    bx, by = harness.backdoor_set("pattern", x, y, 1)
    assert torch.equal(xs[0], bx) and torch.equal(ys[0], by)
    assert (bx.view(-1, 28, 28)[:, :5, :5] == 2.8).all()


def test_cli_flag(monkeypatch):
    from attacking_federate_learning_b200 import sweep
    seen = {}

    def fake_run(kept, epochs, lr, **kw):
        seen.update(kw, kept=kept)
        return []
    monkeypatch.setattr(sweep, "run", fake_run)
    argv = ["-s", "CIFAR10", "-d", "Krum", "NoDefense", "-z", "1.0", "-b", "pattern", "1", "--seeds", "0", "1",
            "-e", "10"]
    sweep.main(argv + ["--cifar10-backdoor"])
    assert seen["cifar10_backdoor"] is True and seen["dataset"] == "CIFAR10" and seen["fading_rate"] == 2000
    assert len(seen["kept"]) == 8 and {e.backdoor for e in seen["kept"]} == {"pattern", 1}
    seen.clear()
    assert sweep.main(argv) == [] and not seen                       # every cell skipped: nothing runs
    sweep.main(argv[:8] + ["No", "pattern"] + argv[10:])
    assert seen["cifar10_backdoor"] is False and all(e.backdoor is False for e in seen["kept"])
