"""Device-parameter rounds of up to 1024 clients per problem (afl_defend_batched_large_dev, DeviceRound(large=True)) on
an H100.

1. Grouping: perm and start[] that class_perm_kernel leaves in the workspace equal a stable argsort of the problems'
   slot classes and the class offsets, for TrimmedMean (rows in all 8 classes, B = 1, 37 and 4097, which crosses the
   kernel's 1024-problem chunks) and for Bulyan's second stage (theta_b across classes).
2. Bit identity with the host-parameter calls (afl_defend_batched_large) for Krum, Bulyan, TrimmedMean and NoDefense at
   N = 129, 500 and 1000, fp32 on an aligned pitch (tensor-core Gram) and an odd one (SIMT Gram), bf16 and fp16, whole
   and ragged slots, per-problem users counts for Krum, and batches whose problems all fall in class 0 or all in 7.
3. Flagged problems: each gets the host call's error through raise_for_status and the host call's result on the safe
   row, and the other problems equal a batch without them.
4. Captured rounds at N = 1000, replayed over refilled grids of different class mixes, equal eager host calls.
5. Oracles: Krum's index equals the C oracle's wherever its margin exceeds 1e-5, and the trimmed mean of exact-integer
   columns across every class equals the reference's fp32 bits.
"""
import numpy as np
import pytest
import torch

from oracle import c_oracle as co
from test_gpu_batched_oracle import TM_ROWS, batch_of, class_order_checks, collect, slot_class
from test_gpu_trimmed_mean_exact import assert_same_bits, exact_matrix, f_values, ref_tm

pytestmark = pytest.mark.gpu

LAYOUTS = ["fp32", "fp32_unaligned", "bf16", "fp16"]
RULES = ("Krum", "Bulyan", "TrimmedMean", "NoDefense")
PROBLEM_BYTES = 40                       # sizeof(ProblemParams)


@pytest.fixture(scope="module")
def env():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    import __graft_entry__ as g
    g.build()
    from attacking_federate_learning_b200 import _device, _native, batched
    return _native, batched, _device


def dev_i32(v):
    return torch.as_tensor(np.asarray(v, np.int32), device="cuda")


def bits(t):
    t = t.contiguous()
    return t.view({4: torch.int32, 8: torch.int64, 2: torch.int16, 1: torch.uint8}[t.element_size()])


def assert_bits(a, b, what):
    assert a.shape == b.shape and a.dtype == b.dtype, (what, a.shape, b.shape, a.dtype, b.dtype)
    assert torch.equal(bits(a), bits(b)), what


def check_selection(dev_sel, host_sel):
    w = host_sel.shape[1]
    assert torch.equal(dev_sel[:, :w], host_sel)
    assert bool((dev_sel[:, w:] == -2).all())


def make_g(layout, seed, B, N, D):
    gen = torch.Generator(device="cuda").manual_seed(seed)
    pitch = D + 1 if layout == "fp32_unaligned" else D
    base = torch.randn(B, N, pitch, device="cuda", generator=gen)
    base += 0.3 * torch.randn(B, 1, pitch, device="cuda", generator=gen)
    base *= torch.exp(0.25 * torch.randn(B, N, 1, device="cuda", generator=gen))
    dt = {"bf16": torch.bfloat16, "fp16": torch.float16}.get(layout, torch.float32)
    return base.to(dt)[:, :, :D]


def fill(rm, fs, zs=None, rows=None, ucs=None):
    rm.f.copy_(dev_i32(fs))
    rm.z.copy_(torch.tensor(np.zeros(len(fs)) if zs is None else zs, dtype=torch.float64))
    if rows is not None:
        rm.rows.copy_(dev_i32(rows))
    if ucs is not None:
        rm.users_count.copy_(dev_i32(ucs))


def bulyan_f(rows):
    """Per-problem corrupted counts valid for Bulyan (4f + 3 <= rows), spread over [0, its largest]."""
    return [max(0, (r - 3) // 4 - (b % 3) * ((r - 3) // 12)) for b, r in enumerate(rows)]


# ---- 1. grouping -------------------------------------------------------------------------------------------------------
def read_grouping(nat, rm, rule):
    """(perm, start) as the last call left them in rm's workspace: perm after the table, start at the large call's
    workspace size (DESIGN 1b)."""
    L = nat.lib()
    B = rm.B
    ws = rm._ws.cpu().numpy()
    perm = ws[B * PROBLEM_BYTES: B * (PROBLEM_BYTES + 4)].view(np.int32)
    off = L.afl_batched_large_workspace_bytes(rule.encode(), B, rm.N, rm.D, rm._code)
    start = ws[off: off + 4 * 9].view(np.int32)
    return perm, start


def expected_grouping(n_rows):
    cls = np.array([slot_class(int(r)) for r in n_rows])
    counts = np.bincount(cls, minlength=8)
    return np.argsort(cls, kind="stable").astype(np.int32), np.concatenate([[0], np.cumsum(counts)]).astype(np.int32)


@pytest.mark.parametrize("B", [1, 37, 4097])
def test_trimmed_mean_grouping(env, B):
    nat, bt, _ = env
    rng = np.random.default_rng(B)
    N, D = 1024, 16
    rows = rng.integers(1, N + 1, B)
    if B >= 8:
        rows[rng.permutation(B)[:8]] = [1, 129, 257, 385, 513, 641, 769, 1024]      # every class present
    G = torch.randn(B, N, D, device="cuda")
    rm = bt.DeviceRound(G, rows=True, large=True, rules=("TrimmedMean",))
    fill(rm, rows // 5, rows=rows)
    out = rm.trimmed_mean()
    perm, start = read_grouping(nat, rm, "TrimmedMean")
    want_perm, want_start = expected_grouping(rows)
    assert np.array_equal(start, want_start)
    assert np.array_equal(perm, want_perm)
    host = bt.trimmed_mean(G, None, rows // 5, rows=rows)
    assert_bits(out, host, "trimmed mean")
    assert not rm.status.any()


@pytest.mark.parametrize("B", [1, 37])
def test_bulyan_grouping_on_theta(env, B):
    nat, bt, _ = env
    rng = np.random.default_rng(100 + B)
    N, D = 1000, 64
    rows = rng.integers(3, N + 1, B)
    fs = np.array([int(rng.integers(0, (r - 3) // 4 + 1)) for r in rows], np.int32)
    G = make_g("fp32", 5 + B, B, N, D).contiguous()
    rm = bt.DeviceRound(G, rows=True, large=True, rules=("Bulyan",))
    fill(rm, fs, rows=rows)
    out, sel = rm.bulyan(return_selection=True)
    perm, start = read_grouping(nat, rm, "Bulyan")
    thetas = rows - 2 * fs
    if B > 8:
        assert len({slot_class(int(t)) for t in thetas}) > 4                          # theta_b crosses classes
    want_perm, want_start = expected_grouping(thetas)
    assert np.array_equal(start, want_start)
    assert np.array_equal(perm, want_perm)
    hb, hs = bt.bulyan(G, None, fs, return_selection=True, rows=rows)
    assert_bits(out, hb, "bulyan")
    check_selection(sel, hs)


# ---- 2. bit identity ---------------------------------------------------------------------------------------------------
def ragged_rows(N):
    return [N, N - 1, N // 2 + 1, 3, min(N, 128)]


def run_and_compare(bt, G, rows, fs, ucs=None):
    """Every defence of DeviceRound(large=True) on G against the host-parameter calls on the same values."""
    B, N, _ = G.shape
    rm = bt.DeviceRound(G, rows=rows is not None, large=True)
    fill(rm, fs, rows=rows)
    idx = rm.krum(return_index=True).clone()
    krow = rm.krum().clone()
    out_b, sel = (t.clone() for t in rm.bulyan(return_selection=True))
    tm, mean = rm.trimmed_mean().clone(), rm.no_defense().clone()
    users = N if rows is None else None
    assert torch.equal(idx, bt.krum(G, users, fs, return_index=True, rows=rows))
    assert_bits(krow, bt.krum(G, users, fs, rows=rows), "krum rows")
    hb, hs = bt.bulyan(G, users, fs, return_selection=True, rows=rows)
    assert_bits(out_b, hb, "bulyan")
    check_selection(sel, hs)
    assert_bits(tm, bt.trimmed_mean(G, users, fs, rows=rows), "trimmed mean")
    assert_bits(mean, bt.no_defense(G, users, fs, rows=rows), "mean")
    assert not rm.status.any()
    rm.raise_for_status()
    if ucs is not None:                        # Krum with users counts of its own (Bulyan needs users_count == rows)
        rk = bt.DeviceRound(G, rows=True, per_problem_users_count=True, large=True, rules=("Krum",))
        fill(rk, fs, rows=rows, ucs=ucs)
        assert torch.equal(rk.krum(return_index=True), bt.krum(G, ucs, fs, return_index=True, rows=rows))
        assert not rk.status.any()


@pytest.mark.parametrize("ragged", [False, True], ids=["whole", "ragged"])
@pytest.mark.parametrize("layout", LAYOUTS)
@pytest.mark.parametrize("N", [129, 500, 1000])
def test_device_round_large_equals_host_calls(env, N, layout, ragged):
    _, bt, _ = env
    B, D = 5, 200
    G = make_g(layout, N + LAYOUTS.index(layout), B, N, D)
    rows = ragged_rows(N) if ragged else None
    fs = bulyan_f(rows if ragged else [N] * B)
    ucs = [max(2 * f + 1, r - 1 - (b % 2) * (r // 3)) for b, (r, f) in enumerate(zip(rows, fs))] if ragged else None
    run_and_compare(bt, G, rows, fs, ucs)


@pytest.mark.parametrize("mix", ["class0", "class7"])
def test_batches_in_one_class(env, mix):
    _, bt, _ = env
    N, D = 1000, 300
    rows = [128, 5, 100, 64] if mix == "class0" else [1000, 999, 950, 990]
    fs = [10, 0, 20, 15] if mix == "class0" else [0, 1, 2, 20]          # thetas in the class of the rows too
    assert {slot_class(r - 2 * f) for r, f in zip(rows, fs)} == {0 if mix == "class0" else 7}
    G = make_g("fp32", 7, len(rows), N, D)
    run_and_compare(bt, G, rows, fs)


# ---- 3. flagged problems -----------------------------------------------------------------------------------------------
def test_flagged_problems(env):
    nat, bt, _ = env
    N, D = 500, 256
    G = make_g("fp32", 21, 6, N, D)
    rows = [500, 400, 300, 250, 200, 130]
    fs = [20, -1, 10, 70, 30, 5]               # problem 1: f < 0
    bad_rows = list(rows)
    bad_rows[2] = 0                            # problem 2: rows outside [1, N]
    ucs = list(bad_rows)
    ucs[4] = 199                               # problem 4: Bulyan's users_count != rows (Krum runs it)
    # problem 3: 4f + 3 > rows (Bulyan's precondition), Krum and the trimmed mean accept f = 70 of 250
    flagged = {"Krum": {1: nat.AFL_ERR_BAD_ARG, 2: nat.AFL_ERR_BAD_ARG},
               "Bulyan": {1: nat.AFL_ERR_BAD_ARG, 2: nat.AFL_ERR_BAD_ARG, 3: nat.AFL_ERR_PRECONDITION,
                          4: nat.AFL_ERR_UNSUPPORTED},
               "TrimmedMean": {1: nat.AFL_ERR_BAD_ARG, 2: nat.AFL_ERR_BAD_ARG},
               "NoDefense": {1: nat.AFL_ERR_BAD_ARG, 2: nat.AFL_ERR_BAD_ARG}}
    exc = {nat.AFL_ERR_BAD_ARG: ValueError, nat.AFL_ERR_PRECONDITION: AssertionError,
           nat.AFL_ERR_UNSUPPORTED: NotImplementedError}
    rm = bt.DeviceRound(G, rows=True, per_problem_users_count=True, large=True)
    fill(rm, fs, rows=bad_rows, ucs=ucs)
    for rule in RULES:
        rm.clear_status()
        res = {"Krum": lambda: rm.krum(return_index=True), "Bulyan": lambda: rm.bulyan(return_selection=True),
               "TrimmedMean": rm.trimmed_mean, "NoDefense": rm.no_defense}[rule]()
        st = rm.status.cpu().tolist()
        assert st == [flagged[rule].get(b, 0) for b in range(6)], (rule, st)
        # the batch without them: the flagged problems replaced by the safe row (N rows and users, f = 0)
        safe = lambda v, s: [s if b in flagged[rule] else x for b, x in enumerate(v)]
        gr, gu, gf = safe(bad_rows, N), safe(ucs, N), safe(fs, 0)
        if rule == "Krum":
            assert torch.equal(res, bt.krum(G, gu, gf, return_index=True, rows=gr)), rule
        elif rule == "Bulyan":
            hb, hs = bt.bulyan(G, gu, gf, return_selection=True, rows=gr)
            assert_bits(res[0], hb, rule)
            check_selection(res[1], hs)
        else:
            assert_bits(res, bt.defend[rule](G, gu, gf, rows=gr), rule)
        # each flagged problem raises what the host call raises on that problem alone
        for b, code in flagged[rule].items():
            rm.status[:b] = 0
            with pytest.raises(exc[code], match=f"problem {b}"):
                rm.raise_for_status()
            with pytest.raises(exc[code]):
                bt.defend[rule](G[b:b + 1], [ucs[b]], [fs[b]], rows=[bad_rows[b]])


# ---- 4. captured rounds ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", ["bulyan", "krum_tm"])
def test_captured_round_at_1000(env, kind):
    _, bt, _device = env
    B, N, D = 4, 1000, 512
    G = make_g("fp32", 30, B, N, D).contiguous()
    rules = ("Bulyan",) if kind == "bulyan" else ("Krum", "TrimmedMean")
    rm = bt.DeviceRound(G, rows=True, large=True, rules=rules)
    w = torch.zeros(B, D, device="cuda")
    v = torch.zeros(B, D, device="cuda")

    def round_():
        crafted, mu, sigma = rm.alie()
        if kind == "bulyan":
            agg, sel = rm.bulyan(return_selection=True)
            met = rm.attack_metrics(aggregated=agg, selection=sel)
            res = dict(agg=agg, sel=sel, rel=met["rel_deviation"], frac=met["bulyan_malicious_fraction"])
        else:
            idx = rm.krum(return_index=True)
            agg = rm.trimmed_mean()
            met = rm.attack_metrics(krum_index=idx)
            res = dict(idx=idx, agg=agg, rel=met["rel_deviation"], hit=met["krum_success"])
        _device.momentum_step(w, v, agg, 0.9, 0.1)
        return dict(crafted=crafted, mu=mu, sigma=sigma, **res)

    fill(rm, [10, 50, 100, 200], [1.0, 0.5, 1.5, 2.0], [1000, 900, 600, 1000])
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        round_()                                                 # eager warm-up
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        outs = round_()

    def check(seed, fs, zs, rows):
        new = make_g("fp32", seed, B, N, D)
        G.copy_(new)
        fill(rm, fs, zs, rows)
        w0, v0 = torch.randn(B, D, device="cuda"), torch.randn(B, D, device="cuda")
        w.copy_(w0), v.copy_(v0)
        graph.replay()
        torch.cuda.synchronize()
        Gh = new.clone()
        for a, b, what in zip((outs["crafted"], outs["mu"], outs["sigma"]), bt.alie_rows(Gh, fs, zs),
                              ("crafted", "mu", "sigma")):
            assert_bits(a, b, what)
        assert_bits(G, Gh, "written rows")
        if kind == "bulyan":
            hb, hs = bt.bulyan(Gh, None, fs, return_selection=True, rows=rows)
            assert_bits(outs["agg"], hb, "bulyan")
            check_selection(outs["sel"], hs)
            hm = bt.attack_metrics(Gh, fs, aggregated=hb, selection=hs, rows=rows)
            assert_bits(outs["frac"], hm["bulyan_malicious_fraction"], "fraction")
        else:
            hk = bt.krum(Gh, None, fs, return_index=True, rows=rows)
            assert torch.equal(outs["idx"], hk)
            hb = bt.trimmed_mean(Gh, None, fs, rows=rows)
            assert_bits(outs["agg"], hb, "trimmed mean")
            hm = bt.attack_metrics(Gh, fs, krum_index=hk, rows=rows)
            assert torch.equal(outs["hit"], hm["krum_success"])
        assert_bits(outs["rel"], hm["rel_deviation"], "rel")
        _device.momentum_step(w0, v0, hb, 0.9, 0.1)
        assert_bits(w, w0, "weights")
        assert_bits(v, v0, "velocity")
        assert not rm.status.any()

    check(40, [2, 0, 30, 5], [1.0, 0.5, 0.0, -1.2], [100, 12, 128, 27])              # every problem in class 0
    check(41, [240, 100, 0, 30], [1.5] * 4, [1000] * 4)                               # rows = N
    check(42, [0, 60, 1, 120], [0.0, 3.0, 1.0, 0.2], [3, 700, 129, 500])              # mixed


# ---- 5. oracles --------------------------------------------------------------------------------------------------------
def test_krum_index_equals_the_c_oracle(env):
    _, bt, _ = env
    B, N, D = 3, 500, 2000
    rows, fs = [500, 333, 129], [100, 50, 20]
    G = make_g("fp32", 50, B, N, D).contiguous()
    rm = bt.DeviceRound(G, rows=True, large=True, rules=("Krum",))
    fill(rm, fs, rows=rows)
    idx = rm.krum(return_index=True).cpu().tolist()
    Gh = G.cpu().numpy()
    checked = 0
    for b, (r, f) in enumerate(zip(rows, fs)):
        o, margin = co.krum_select(np.sqrt(co.pairwise_sqdist(np.ascontiguousarray(Gh[b, :r]))), r, f, with_margin=True)
        if margin > 1e-5:
            assert idx[b] == o, (b, idx[b], o, margin)
            checked += 1
    assert checked >= 2


@pytest.mark.parametrize("dtype", ["f32", "bf16"])
def test_trimmed_mean_exact_across_classes(env, dtype):
    _, bt, _ = env
    rows = TM_ROWS
    class_order_checks(rows)
    rng = np.random.default_rng(47000 + len(dtype))
    cols = 16 if dtype == "f32" else 32
    mats = [exact_matrix(rng, r, dtype, cols, [max(r - f - 1, 0) for f in f_values(r)]) for r in rows]
    G = batch_of(mats, max(rows), dtype, "aligned")
    rm = bt.DeviceRound(G, rows=True, large=True, rules=("TrimmedMean",))
    failures = []
    for k in range(4):                         # keep = rows_b - 1, about 3/4, 1, 0 (NaN)
        fs = [f_values(r)[min(k, len(f_values(r)) - 1)] for r in rows]
        fill(rm, fs, rows=rows)
        out = rm.trimmed_mean().cpu().numpy()
        for b, (M, f) in enumerate(zip(mats, fs)):
            with collect(failures, f"trimmed mean problem {b} rows {rows[b]} f {f}"):
                assert_same_bits(out[b], ref_tm(M, f), (b, rows[b], f))
    assert not rm.status.any()
    assert not failures, "\n".join(failures)
