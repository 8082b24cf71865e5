"""CPU checks of the CIFAR10 training sweep (harness.Cifar10Net, sweep.py's dataset option, csrc/cifar_grad.cu): the
new entry points' argument checks, Cifar10Net's parameter layout, the setup helper against harness.main's initial
weights, the log names, the grid's CIFAR10 backdoor rejections, and harness.main with dataset='CIFAR10' on the CPU."""
import ctypes
import os

import pytest
import torch

D = 117_706
P = ctypes.c_void_p(256)                 # a non-NULL pointer that is never dereferenced


@pytest.fixture(scope="module")
def lib():
    import __graft_entry__ as g
    g.build()
    from attacking_federate_learning_b200 import _native
    return _native.lib()


def grads(lib, **kw):
    a = dict(weights=P, batch=2, d=D, x=P, y=P, n_sets=1, n_train=100, data_index=P, rows=P, n=10, m=83, epoch=P, G=P,
             batch_stride=10 * 117_728, ld=117_728, stream=None)
    a.update(kw)
    return lib.afl_cifar10_client_grads(*a.values())


def evaluate(lib, **kw):
    a = dict(weights=P, batch=2, d=D, x=P, y=P, n_sets=1, n_test=100, data_index=P, m=83, slot=P, n_slots=1,
             loss_sum=P, correct=P, ws=P, ws_bytes=1 << 20, stream=None)
    a.update(kw)
    return lib.afl_cifar10_evaluate(*a.values())


def test_client_grads_rejects_bad_arguments_before_any_cuda_call(lib):
    from attacking_federate_learning_b200 import _native as nat
    for name in ("weights", "x", "y", "data_index", "rows", "epoch", "G"):
        assert grads(lib, **{name: None}) == nat.AFL_ERR_BAD_ARG, name
    assert grads(lib, d=79_510) == nat.AFL_ERR_UNSUPPORTED                # MnistNet's D
    assert b"117706" in lib.afl_last_error()
    assert grads(lib, m=129) == nat.AFL_ERR_UNSUPPORTED
    assert grads(lib, m=0) == nat.AFL_ERR_BAD_ARG
    assert grads(lib, n=1025) == nat.AFL_ERR_UNSUPPORTED
    assert grads(lib, n=0) == nat.AFL_ERR_BAD_ARG
    assert grads(lib, n=101) == nat.AFL_ERR_BAD_ARG                       # more clients than training rows
    assert grads(lib, n_sets=0) == nat.AFL_ERR_BAD_ARG
    assert grads(lib, n_train=0) == nat.AFL_ERR_BAD_ARG
    assert grads(lib, ld=D - 1) == nat.AFL_ERR_BAD_ARG
    assert grads(lib, batch_stride=9 * 117_728) == nat.AFL_ERR_BAD_ARG    # problems would overlap
    assert grads(lib, batch=0) == nat.AFL_ERR_BAD_ARG
    assert grads(lib, batch=65536) == nat.AFL_ERR_UNSUPPORTED


def test_evaluate_rejects_bad_arguments_before_any_cuda_call(lib):
    from attacking_federate_learning_b200 import _native as nat
    for name in ("weights", "x", "y", "data_index", "slot", "loss_sum", "correct", "ws"):
        assert evaluate(lib, **{name: None}) == nat.AFL_ERR_BAD_ARG, name
    assert evaluate(lib, d=D + 1) == nat.AFL_ERR_UNSUPPORTED
    assert evaluate(lib, m=129) == nat.AFL_ERR_UNSUPPORTED
    assert evaluate(lib, m=0) == nat.AFL_ERR_BAD_ARG
    assert evaluate(lib, batch=65536) == nat.AFL_ERR_UNSUPPORTED
    assert evaluate(lib, n_slots=0) == nat.AFL_ERR_BAD_ARG
    need = lib.afl_cifar10_evaluate_workspace_bytes(2, 100, 83)
    assert need == 2 * 256                                                # 2 x 2 floats and 2 x 2 ints, 256-aligned
    assert need == lib.afl_mnist_evaluate_workspace_bytes(2, 100, 83)
    assert lib.afl_cifar10_evaluate_workspace_bytes(300, 4000, 83) >= 2 * 300 * 49 * 4
    assert evaluate(lib, ws_bytes=need - 1) == nat.AFL_ERR_WORKSPACE
    assert evaluate(lib, ws=ctypes.c_void_p(128)) == nat.AFL_ERR_WORKSPACE          # not 256-byte aligned
    assert evaluate(lib, n_test=65536 * 2, m=1, ws_bytes=1 << 30) == nat.AFL_ERR_UNSUPPORTED   # > 65535 test batches
    for bad in ((0, 100, 83), (2, 0, 83), (2, 100, 0)):
        assert lib.afl_cifar10_evaluate_workspace_bytes(*bad) == 0


def test_cifar10net_layout_matches_the_kernel_offsets():
    from attacking_federate_learning_b200 import harness
    net = harness.Cifar10Net()
    layout = harness.ParamLayout(net.parameters())
    assert layout.dim == D
    want = [("conv1.weight", 0, 432), ("conv1.bias", 432, 16), ("conv2.weight", 448, 16_384),
            ("conv2.bias", 16_832, 64), ("fc1.weight", 16_896, 24_576), ("fc1.bias", 41_472, 384),
            ("fc2.weight", 41_856, 73_728), ("fc2.bias", 115_584, 192), ("fc3.weight", 115_776, 1_920),
            ("fc3.bias", 117_696, 10)]
    off = 0
    for (name, p), (want_name, want_off, want_size) in zip(net.named_parameters(), want):
        assert (name, off, p.numel()) == (want_name, want_off, want_size)
        off += p.numel()
    # the flattened vector puts each tensor at its offset
    w = layout.flatten(list(net.parameters()))
    for (name, p), (_, o, n) in zip(net.named_parameters(), want):
        assert torch.equal(w[o:o + n], p.detach().flatten()), name
    assert net(torch.zeros(2, 3, 32, 32)).shape == (2, 10)


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
                         test_size=40, output=None, dataset="CIFAR10")
        torch.manual_seed(1234)                                             # the helper must reseed
        (xtr, ytr), (xte, _), net = harness.experiment_setup(seed, 200, 40, "cpu", dataset="CIFAR10")
        assert isinstance(net, harness.Cifar10Net)
        w = harness.ParamLayout(net.parameters()).flatten(list(net.parameters()))
        assert w.numel() == D
        assert torch.equal(w.view(torch.int32), seen["w"].view(torch.int32))
        assert xtr.shape == (200, 3, 32, 32) and xte.shape == (40, 3, 32, 32)
        assert torch.equal(xtr, harness.synthetic_cifar_problem(200, 40, "cpu", seed)[0][0])
        assert ytr.min() >= 0 and ytr.max() <= 9
    # MNIST stays the default and keeps its data
    (xm, _), _, netm = harness.experiment_setup(0, 200, 40, "cpu")
    assert isinstance(netm, harness.MnistNet) and xm.shape == (200, 784)
    with pytest.raises(ValueError):
        harness.experiment_setup(0, 200, 40, "cpu", dataset="CIFAR100")


def test_csv_names_carry_the_dataset():
    from attacking_federate_learning_b200 import harness, sweep
    e = sweep.Experiment("TrimmedMean", 0.24, 1.5, 10, 3)
    assert sweep.csv_name(e, 0.1, dataset="CIFAR10") == \
        "SYNTH-CIFAR10_stdev_1.5_TrimmedMean_backdoor-False_mal_prop_0.24_users_10_alpha_None_lr_0.1_seed_3.csv"
    assert harness.csv_name(1.5, "Krum", "pattern", 0.1, 10, 4, 0.1, "CIFAR10") == \
        "SYNTH-CIFAR10_stdev_1.5_Krum_backdoor-pattern_mal_prop_0.1_users_10_alpha_4_lr_0.1.csv"
    assert sweep.csv_name(e, 0.1) == sweep.csv_name(e, 0.1, dataset="MNIST")
    assert sweep.csv_name(e, 0.1).startswith("SYNTH-MNIST_")


def test_grid_drops_cifar10_backdoor_cells_and_keeps_mnist_ones():
    from attacking_federate_learning_b200 import sweep
    args = (["Krum", "NoDefense"], [1.5], [0.1], [10], [0, 1])
    kept, dropped = sweep.grid(*args, backdoors=(False, "pattern", 1), dataset="CIFAR10")
    assert [tuple(k) for k in kept] == [("Krum", 0.1, 1.5, 10, 0), ("Krum", 0.1, 1.5, 10, 1),
                                        ("NoDefense", 0.1, 1.5, 10, 0), ("NoDefense", 0.1, 1.5, 10, 1)]
    assert len(dropped) == 8 and all(isinstance(e, NotImplementedError) for _, e in dropped)
    assert all(len(c) == 6 and c[5] in ("pattern", 1) for c, _ in dropped)
    kept_m, dropped_m = sweep.grid(*args, backdoors=(False, "pattern", 1))
    assert kept_m == sweep.grid(*args, backdoors=(False, "pattern", 1), dataset="MNIST")[0]
    assert len(kept_m) == 12 and not dropped_m
    with pytest.raises(NotImplementedError):
        sweep.check(("Krum", 0.1, 1.5, 10, 0, "pattern"), dataset="CIFAR10")
    assert sweep.check(("Krum", 0.1, 1.5, 10, 0, "pattern")).backdoor == "pattern"
    with pytest.raises(ValueError):
        sweep.check(("Krum", 0.1, 1.5, 10, 0), dataset="CIFAR100")


def test_run_rejects_a_cifar10_backdoor_before_any_gpu_work():
    from attacking_federate_learning_b200 import sweep
    with pytest.raises(NotImplementedError):
        sweep.run([("Krum", 0.1, 1.0, 10, 0), ("Krum", 0.1, 1.0, 10, 0, 1)], 1, device="cpu", dataset="CIFAR10")


class CpuServer:
    """server.py:86-90 on the CPU for NoDefense (the mean), in place of the CUDA AggregationServer."""

    def __init__(self, users_count, dim, mal_prop, learning_rate, momentum=0.9, device="cpu", initial_weights=None):
        self.users_grads = torch.zeros(users_count, dim)
        self.velocity = torch.zeros(dim)
        self.current_weights = initial_weights.clone()
        self.learning_rate, self.momentum = learning_rate, momentum

    def defend(self, defence_method, cur_epoch=0):
        assert defence_method == "NoDefense"
        self.velocity = self.momentum * self.velocity - self.learning_rate * self.users_grads.mean(0)
        self.current_weights += self.velocity


@pytest.mark.parametrize("backdoor", [False, "pattern"])
def test_harness_main_runs_cifar10_on_the_cpu(monkeypatch, tmp_path, backdoor):
    """Two epochs of harness.main(dataset='CIFAR10') through autograd (no malicious user, so the attack is a no-op;
    with -b pattern the global model is tested on the patterned set at each test epoch)."""
    from attacking_federate_learning_b200 import harness
    monkeypatch.setattr(harness, "AggregationServer", CpuServer)
    log = tmp_path / "out.txt"
    acc, epochs, csv = harness.main(0.0, 1.5, "NoDefense", users_count=4, epochs=2, device="cpu", seed=1,
                                    train_size=240, test_size=60, batch_size=16, test_step=1, out_dir=str(tmp_path),
                                    output=str(log), backdoor=backdoor, dataset="CIFAR10")
    assert epochs == [0, 1] and len(acc) == 2 and all(0.0 <= a <= 100.0 for a in acc)
    assert os.path.basename(csv) == harness.csv_name(1.5, "NoDefense", backdoor, 0.0, 4, 4, 0.1, "CIFAR10")
    text = log.read_text()
    assert "SYNTH-CIFAR10" in text and text.count("Test set:") == 2
    assert text.count("[POST]") == (2 if backdoor else 0)


def test_backdoor_trainer_trains_a_cifar10net_on_patterned_images():
    from attacking_federate_learning_b200 import harness
    torch.manual_seed(0)
    (x, y), _ = harness.synthetic_cifar_problem(400, 10, "cpu", seed=2)
    bx, by = harness.backdoor_set("pattern", x, y, seed=2)
    assert bx.shape[1:] == (3, 32, 32) and bool((by == 0).all())
    assert bool((bx[:, :, :5, :5] == 2.8).all())                           # add_pattern on every channel
    # 400 rows: u = max(400 // 200 // 10, 1) = 1, so the set is every row, patched
    assert len(bx) == 400 and torch.equal(bx[:, :, 5:], x[:, :, 5:]) and torch.equal(bx[:, :, :, 5:], x[:, :, :, 5:])
    net = harness.Cifar10Net()
    layout = harness.ParamLayout(net.parameters())
    w0 = layout.flatten(list(net.parameters()))
    t = harness.BackdoorTrainer("pattern", 4, 1, layout, x, y, "cpu", lambda *a, **k: None, seed=2,
                                dataset="CIFAR10")
    assert isinstance(t.net, harness.Cifar10Net)
    out = t.train(w0)
    assert out.shape == (D,) and bool(torch.isfinite(out).all()) and not torch.equal(out, w0)
