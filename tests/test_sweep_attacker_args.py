"""CPU checks of per-experiment backdoor α and malicious epochs in training sweeps (sweep.py, harness.py's CLI and the
afl_*_backdoor_train_each entry points in csrc/backdoor_train.cu and csrc/cifar_backdoor.cu): the 10-tuple experiment,
`check`'s rejections, the grid's shape, CSV names and summary columns, the CLIs, and the new entry points' host-side
rejections."""
import ctypes
import itertools
import os

import pytest

P = ctypes.c_void_p(256)                 # a non-NULL pointer that is never dereferenced
NETS = {"mnist": 79_510, "cifar10": 117_706}


@pytest.fixture(scope="module")
def lib():
    import __graft_entry__ as g
    g.build()
    from attacking_federate_learning_b200 import _native
    return _native.lib()


def test_the_ten_tuple():
    from attacking_federate_learning_b200.sweep import Experiment
    e = Experiment("Krum", 0.24, 1.5, 10, 0, "pattern", 0.1, 83, 0.2, 1)
    assert e == ("Krum", 0.24, 1.5, 10, 0, "pattern", 0.1, 83, 0.2, 1) and len(e) == 10
    assert e.backdoor == "pattern" and e.learning_rate == 0.1 and e.batch_size == 83
    assert e.alpha == 0.2 and e.mal_epochs == 1
    assert repr(e) == ("Experiment(defense='Krum', mal_prop=0.24, num_std=1.5, users_count=10, seed=0, "
                       "backdoor='pattern', learning_rate=0.1, batch_size=83, alpha=0.2, mal_epochs=1)")
    assert Experiment(*e) == e
    with pytest.raises(ValueError):
        Experiment("Krum", 0.24, 1.5, 10, 0, "pattern", 0.1, 83, 0.2)                   # alpha without mal_epochs
    with pytest.raises(ValueError):
        Experiment("Krum", 0.24, 1.5, 10, 0, "pattern", alpha=0.2, mal_epochs=1)        # no lr and batch size


def test_short_forms_are_unchanged():
    from attacking_federate_learning_b200.sweep import Experiment
    e5 = Experiment("Krum", 0.24, 1.5, 10, 0)
    e6 = Experiment("Krum", 0.24, 1.5, 10, 0, 1)
    e8 = Experiment("Krum", 0.24, 1.5, 10, 0, "pattern", 0.05, 32)
    assert (e5, e6, e8) == (("Krum", 0.24, 1.5, 10, 0), ("Krum", 0.24, 1.5, 10, 0, 1),
                            ("Krum", 0.24, 1.5, 10, 0, "pattern", 0.05, 32))
    assert repr(e5) == "Experiment(defense='Krum', mal_prop=0.24, num_std=1.5, users_count=10, seed=0)"
    assert repr(e8).endswith("backdoor='pattern', learning_rate=0.05, batch_size=32)")
    for e in (e5, e6, e8):
        assert e.alpha is None and e.mal_epochs is None
    assert e8.learning_rate == 0.05 and e8.batch_size == 32


def test_check_normalises_and_rejects():
    from attacking_federate_learning_b200 import sweep
    e = sweep.check(("Krum", "0.24", 1.5, "10", 0, "pattern", "0.1", "83", "0.2", "0"))
    assert e == ("Krum", 0.24, 1.5, 10, 0, "pattern", 0.1, 83, 0.2, 0)
    assert isinstance(e.alpha, float) and isinstance(e.mal_epochs, int)
    assert sweep.check(("Krum", 0.24, 1.5, 10, 0, "1", 0.1, 83, -1, 2)).alpha == -1.0     # α <= 0: no distance term
    with pytest.raises(ValueError, match="backdoor"):
        sweep.check(("Krum", 0.24, 1.5, 10, 0, False, 0.1, 83, 0.2, 1))                  # a drift 10-tuple
    with pytest.raises(ValueError, match="alpha"):
        sweep.check(("Krum", 0.24, 1.5, 10, 0, "pattern", 0.1, 83, float("nan"), 1))
    with pytest.raises(ValueError, match="mal_epochs"):
        sweep.check(("Krum", 0.24, 1.5, 10, 0, "pattern", 0.1, 83, 0.2, -1))
    with pytest.raises(ValueError):
        sweep.check(("Krum", 0.24, 1.5, 10, 0, "pattern", 0.1, 83, 0.2))                 # 9 elements
    with pytest.raises(NotImplementedError):                                               # its own batch size is checked
        sweep.check(("Krum", 0.24, 1.5, 10, 0, "pattern", 0.1, 129, 0.2, 1))


def test_grid_multiplies_backdoor_cells_only():
    from attacking_federate_learning_b200 import sweep
    args = (["Krum", "NoDefense"], [1.0], [0.1, 0.24], [10], [0, 1])
    base, _ = sweep.grid(*args, backdoors=[False, "pattern", 1])
    kept, dropped = sweep.grid(*args, backdoors=[False, "pattern", 1], alphas=[0.2, 1, 4], mal_epochs=[1, 5])
    assert not dropped
    drift = [e for e in base if e.backdoor is False]
    assert [e for e in kept if e.backdoor is False] == drift and all(len(e) == 5 for e in drift)
    want = []
    for e in base:
        if e.backdoor is False:
            want.append(e)
        else:
            want += [tuple(e) + (0.1, 83, a, k) for a, k in itertools.product([0.2, 1, 4], [1, 5])]
    assert kept == want and len(kept) == len(drift) + 6 * (len(base) - len(drift))
    # the axis not given is the run's value; lr and c are the run's too
    kept, _ = sweep.grid(["Krum"], [1.0], [0.1], [10], [0], 64, backdoors=["pattern"], alphas=[0.2, 4],
                         learning_rate=0.05, run_mal_epochs=3)
    assert kept == [("Krum", 0.1, 1.0, 10, 0, "pattern", 0.05, 64, a, 3) for a in (0.2, 4)]
    kept, _ = sweep.grid(["Krum"], [1.0], [0.1], [10], [0], backdoors=["pattern"], mal_epochs=[0, 2], alpha=0.5)
    assert kept == [("Krum", 0.1, 1.0, 10, 0, "pattern", 0.1, 83, 0.5, k) for k in (0, 2)]
    # with learning-rate and batch-size axes: lr, c, α, mal_epochs innermost in that order; drift cells are 8-tuples
    kept, _ = sweep.grid(["Krum"], [1.0], [0.1], [10], [0], backdoors=[False, 2], learning_rates=[0.05, 0.1],
                         batch_sizes=[32], alphas=[0.2, 4], mal_epochs=[1])
    assert kept == [("Krum", 0.1, 1.0, 10, 0, False, lr, 32) for lr in (0.05, 0.1)] + \
        [("Krum", 0.1, 1.0, 10, 0, 2, lr, 32, a, 1) for lr in (0.05, 0.1) for a in (0.2, 4)]
    # a bad value is dropped with check's rejection, cell by cell
    kept, dropped = sweep.grid(["Krum"], [1.0], [0.1], [10], [0], backdoors=["pattern"], mal_epochs=[-1, 1])
    assert [len(e) for e in kept] == [10] and kept[0].mal_epochs == 1
    assert len(dropped) == 1 and dropped[0][0][9] == -1 and isinstance(dropped[0][1], ValueError)


def test_csv_names():
    from attacking_federate_learning_b200 import harness, sweep
    e10 = sweep.Experiment("Krum", 0.24, 1.5, 10, 3, "pattern", 0.05, 32, 0.2, 1)
    want = harness.csv_name(1.5, "Krum", "pattern", 0.24, 10, 0.2, 0.05)[:-4] + "_batch_32_malepochs_1_seed_3.csv"
    assert sweep.csv_name(e10, 0.1, alpha=4) == want                                     # its own α, not the run's
    assert "_alpha_0.2_lr_0.05_batch_32_malepochs_1_seed_3.csv" in want
    names = {sweep.csv_name(sweep.Experiment("Krum", 0.24, 1.5, 10, 3, 1, 0.1, 83, a, k), 0.1)
             for a in (0.2, 1.0, 4.0) for k in (1, 5)}
    assert len(names) == 6
    e6 = sweep.Experiment("Krum", 0.24, 1.5, 10, 3, "pattern")                            # the short forms as before
    assert sweep.csv_name(e6, 0.1, alpha=4) == \
        harness.csv_name(1.5, "Krum", "pattern", 0.24, 10, 4, 0.1)[:-4] + "_seed_3.csv"
    e8 = sweep.Experiment("Krum", 0.24, 1.5, 10, 3, "pattern", 0.05, 32)
    assert sweep.csv_name(e8, 0.1).endswith("_alpha_4_lr_0.05_batch_32_seed_3.csv")


def test_summary_headers():
    from attacking_federate_learning_b200 import sweep
    base = ["defense", "mal_prop", "num_std", "users_count", "seed"]
    assert sweep.summary_header(True, True) == sweep.summary_header(True, True, False, False)
    assert sweep.summary_header(True, True, False, True) == base + [
        "backdoor", "learning_rate", "batch_size", "alpha", "mal_epochs", "max_accuracy", "final_accuracy",
        "max_backdoor_accuracy", "final_backdoor_accuracy", "status"]


def results(sweep):
    exps = [sweep.Experiment("Krum", 0.24, 1.0, 10, 0), sweep.Experiment("Krum", 0.24, 1.0, 10, 0, 1, 0.1, 83, 0.2, 1)]
    return [dict(experiment=exps[0], accuracies=[10.0, 20.0], error=None),
            dict(experiment=exps[1], accuracies=[10.0, 30.0], backdoor_accuracies=[0.0, 100.0], error=None)]


def test_write_logs_columns(tmp_path):
    from attacking_federate_learning_b200 import sweep
    res = results(sweep)
    names = [sweep.csv_name(r["experiment"], 0.1) for r in res]
    sweep.write_logs(res, str(tmp_path), names, True, [[0.1, 83], [0.1, 83]], attack=[["", ""], [0.2, 1]])
    rows = open(os.path.join(tmp_path, sweep.SUMMARY)).read().splitlines()
    assert rows[0].split(",") == sweep.summary_header(True, True, False, True)
    assert rows[1].split(",")[5:10] == ["False", "0.1", "83", "", ""]                    # empty for the drift row
    assert rows[2].split(",")[5:10] == ["1", "0.1", "83", "0.2", "1"]
    assert os.path.exists(os.path.join(tmp_path, names[1])) and "_malepochs_1_" in names[1]


def test_write_logs_without_ten_tuples_keeps_every_byte(tmp_path):
    from attacking_federate_learning_b200 import sweep
    res = results(sweep)
    res[1]["experiment"] = sweep.Experiment("Krum", 0.24, 1.0, 10, 0, 1)
    names = [sweep.csv_name(r["experiment"], 0.1) for r in res]
    for d, kw in (("a", {}), ("b", dict(attack=None))):
        os.makedirs(tmp_path / d)
        sweep.write_logs([dict(r) for r in res], str(tmp_path / d), names, True, None, **kw)
    for f in [sweep.SUMMARY] + names:
        assert open(tmp_path / "a" / f, "rb").read() == open(tmp_path / "b" / f, "rb").read()
    rows = open(tmp_path / "a" / sweep.SUMMARY).read().splitlines()
    assert rows[0].split(",") == sweep.summary_header(True) and "alpha" not in rows[0]


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


def test_cli_with_one_value_makes_no_ten_tuple(monkeypatch):
    seen = _cli(monkeypatch, ["-d", "Krum", "-z", "1.0", "-e", "3", "-b", "No", "pattern", "--alpha", "0.2",
                              "--mal-epochs", "2"])
    assert seen["grid"][1] == dict(backdoors=[False, "pattern"], dataset="MNIST", cifar10_backdoor=False)
    kept, _, _, kw = seen["run"]
    assert kept == [("Krum", 0.24, 1.0, 10, 0), ("Krum", 0.24, 1.0, 10, 0, "pattern")]
    assert kw["alpha"] == 0.2 and kw["mal_epochs"] == 2
    seen = _cli(monkeypatch, ["-d", "Krum", "-e", "3", "-b", "pattern"])                   # the defaults: main.py's
    assert seen["run"][3]["alpha"] == 4 and seen["run"][3]["mal_epochs"] == 5
    assert len(seen["run"][0][0]) == 6


def test_cli_with_several_values_makes_ten_tuples(monkeypatch):
    seen = _cli(monkeypatch, ["-d", "Krum", "-z", "1.0", "-e", "3", "-b", "No", "pattern", "-l", "0.05",
                              "--alpha", "0.2", "1", "4", "--mal-epochs", "1", "5"])
    kept = seen["run"][0]
    assert kept == [("Krum", 0.24, 1.0, 10, 0)] + [("Krum", 0.24, 1.0, 10, 0, "pattern", 0.05, 83, a, k)
                                                    for a in (0.2, 1.0, 4.0) for k in (1, 5)]
    seen = _cli(monkeypatch, ["-d", "Krum", "-e", "3", "-b", "1", "--mal-epochs", "1", "5"])   # one α: the run's
    assert seen["run"][0] == [("Krum", 0.24, 1.5, 10, 0, 1, 0.1, 83, 4, k) for k in (1, 5)]
    assert seen["run"][3]["alpha"] == 4 and seen["run"][3]["mal_epochs"] == 1


def test_harness_flags(monkeypatch):
    from attacking_federate_learning_b200 import harness
    seen = {}
    monkeypatch.setattr(harness, "main", lambda *a, **kw: seen.update(a=a, kw=kw))
    harness.cli(["-d", "Krum", "-b", "pattern", "--alpha", "0.2", "--mal-epochs", "1"])
    assert seen["a"] == (0.24, 1.5, "Krum") and seen["kw"]["backdoor"] == "pattern"
    assert seen["kw"]["alpha"] == 0.2 and seen["kw"]["mal_epochs"] == 1
    harness.cli(["-d", "Krum", "-b", "pattern"])                                            # today's values and name
    assert seen["kw"]["alpha"] == 4 and seen["kw"]["mal_epochs"] == 5
    assert harness.csv_name(1.5, "Krum", "pattern", 0.24, 10, seen["kw"]["alpha"], 0.1).endswith("_alpha_4_lr_0.1.csv")


def train_each(lib, net, **kw):
    a = dict(initial=P, out=ctypes.c_void_p(1 << 30), batch=2, d=NETS[net], x=P, y=P, n_sets=1, max_len=100,
             set_len=P, data_index=P, f=P, z=P, status=P, alpha=P, mal_epochs=P, m=200)
    if net == "cifar10":
        a.update(ws=ctypes.c_void_p(1 << 31), ws_bytes=1 << 30)
    a.update(kw)
    return getattr(lib, f"afl_{net}_backdoor_train_each")(*a.values(), None)


@pytest.mark.parametrize("net", sorted(NETS))
def test_backdoor_train_each_rejects_bad_arguments_before_any_cuda_call(lib, net):
    from attacking_federate_learning_b200 import _native as nat
    names = ["initial", "out", "x", "y", "set_len", "data_index", "f", "z", "status", "alpha", "mal_epochs"]
    for name in names + (["ws"] if net == "cifar10" else []):
        assert train_each(lib, net, **{name: None}) == nat.AFL_ERR_BAD_ARG, name
        assert b"NULL" in lib.afl_last_error() and f"afl_{net}_backdoor_train_each".encode() in lib.afl_last_error()
    assert train_each(lib, net, d=NETS[net] + 1) == nat.AFL_ERR_UNSUPPORTED
    assert train_each(lib, net, m=201) == nat.AFL_ERR_UNSUPPORTED
    assert train_each(lib, net, m=0) == nat.AFL_ERR_BAD_ARG
    assert train_each(lib, net, batch=65536) == nat.AFL_ERR_UNSUPPORTED
    assert train_each(lib, net, out=P) == nat.AFL_ERR_BAD_ARG                               # out overlaps initial
    if net == "cifar10":
        assert train_each(lib, net, ws_bytes=lib.afl_cifar10_backdoor_train_workspace_bytes(2) - 1) == \
            nat.AFL_ERR_BAD_ARG
