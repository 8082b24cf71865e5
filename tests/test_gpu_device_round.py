"""Device-parameter batched calls (afl_*_dev, batched.DeviceRound) on an H100.

* Table: afl_batched_table_dev's rows against the rows the host-parameter calls leave at their workspace start, over
  rule x rows x users_count x f with the edges; invalid values give the status code and the safe row, read back
  before any kernel runs on that table.
* Bit identity: every DeviceRound method against the host-parameter batched call on the same values, for fp32 on an
  aligned pitch (tensor-core Gram) and an unaligned one (SIMT Gram), bf16 and fp16, with per-problem f and with ragged
  rows.  ALIE's 16-bit rows, written in the kernel, must equal the cast route's.
* Status: flagged problems leave the others as a batch of valid problems gives them, and raise_for_status raises what
  the host call raises.
* Capture: one round captured with torch.cuda.graph, replayed over three grids refilled in place, equals eager
  host-parameter calls, also after an eager module-level call has grown the shared workspace cache.
"""
import ctypes

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

ROW_INTS = (0, 1, 2, 3, 5, 6)          # f, take, theta, write, tm.n_rows, tm.keep of a 40-byte ProblemParams
ROW_FLOATS = (4, 7, 8, 9)              # z, tm.med_density, tm.key_q, tm.key_density


@pytest.fixture(scope="module")
def env():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    import __graft_entry__ as g
    g.build()
    from attacking_federate_learning_b200 import _native, batched
    return _native, batched


def dev_i32(v):
    return torch.as_tensor(np.asarray(v, np.int32), device="cuda")


def bits(t):
    t = t.contiguous()
    return t.view({4: torch.int32, 8: torch.int64, 2: torch.int16, 1: torch.uint8}[t.element_size()])


def assert_bits(a, b, what):
    assert a.shape == b.shape and a.dtype == b.dtype, (what, a.shape, b.shape, a.dtype, b.dtype)
    assert torch.equal(bits(a), bits(b)), what


def host_table(nat, rule, rows, ucs, fs, n, zs=None):
    """The table a host-parameter call leaves at its workspace start: [B, 10] int32 and the same bytes as float32."""
    L = nat.lib()
    B, d = len(fs), 8
    G = torch.randn(B, n, d, device="cuda")
    fs = np.asarray(fs, np.int32)
    if rule == "ALIE":
        ws = torch.empty(L.afl_batched_each_workspace_bytes(b"ALIE", B, 1, d, 0), dtype=torch.uint8, device="cuda")
        zs = np.asarray(zs, np.float64)
        out = [torch.empty(B, d, device="cuda") for _ in range(3)]
        nat.check(L.afl_alie_batched_large(G.data_ptr(), B, n * d, n, d, d, 0, fs.ctypes.data, zs.ctypes.data,
                                           *(o.data_ptr() for o in out), None, 0, 0, ws.data_ptr(), ws.numel(), None))
    elif rule == "AttackMetrics":
        ws = torch.empty(L.afl_metrics_workspace_bytes(B, n, d, 0), dtype=torch.uint8, device="cuda")
        agg, dev = torch.zeros(B, d, device="cuda"), torch.empty(B, device="cuda")
        args = (G.data_ptr(), B, n * d, n, d, d, 0)
        tail = (agg.data_ptr(), None, None, 0, dev.data_ptr(), None, None, None, None, None, ws.data_ptr(), ws.numel(), None)
        if rows is None:
            nat.check(L.afl_attack_metrics_batched_each(*args, fs.ctypes.data, *tail))
        else:
            rs = np.asarray(rows, np.int32)
            nat.check(L.afl_attack_metrics_batched_rows(*args, rs.ctypes.data, fs.ctypes.data, *tail))
    else:
        ws = torch.empty(L.afl_batched_rows_workspace_bytes(rule.encode(), B, n, d, 0), dtype=torch.uint8, device="cuda")
        out, idx = torch.empty(B, d, device="cuda"), torch.empty(B, dtype=torch.int32, device="cuda")
        sel = torch.empty(B, n, dtype=torch.int32, device="cuda")
        outs = (out.data_ptr(), idx.data_ptr(), sel.data_ptr(), ws.data_ptr(), ws.numel(), None)
        if rows is None:
            nat.check(L.afl_defend_batched_each(rule.encode(), G.data_ptr(), B, n * d, n, d, d, 0, int(ucs),
                                                fs.ctypes.data, *outs))
        else:
            rs, us = np.asarray(rows, np.int32), np.asarray(ucs, np.int32)
            nat.check(L.afl_defend_batched_rows(rule.encode(), G.data_ptr(), B, n * d, n, d, d, 0, rs.ctypes.data,
                                                us.ctypes.data, fs.ctypes.data, *outs))
    torch.cuda.synchronize()
    raw = ws[:B * 40].clone()
    return raw.view(torch.int32).view(B, 10), raw.view(torch.float32).view(B, 10)


def device_table(nat, rule, n, rows, ucs, fs, users_count=0, zs=None, status=None):
    B = len(fs)
    ws = torch.full((B * 40 + 256,), 0xAB, dtype=torch.uint8, device="cuda")
    st = torch.zeros(B, dtype=torch.int32, device="cuda") if status is None else status
    r = None if rows is None else dev_i32(rows)
    u = None if ucs is None else dev_i32(ucs)
    f = dev_i32(fs)
    z = None if zs is None else torch.as_tensor(np.asarray(zs, np.float64), device="cuda")
    nat.check(nat.lib().afl_batched_table_dev(rule.encode(), B, n, None if r is None else r.data_ptr(), users_count,
                                              None if u is None else u.data_ptr(), f.data_ptr(),
                                              None if z is None else z.data_ptr(), ws.data_ptr(), ws.numel(),
                                              st.data_ptr(), None))
    torch.cuda.synchronize()
    raw = ws[:B * 40].clone()
    return raw.view(torch.int32).view(B, 10), raw.view(torch.float32).view(B, 10), st.cpu().numpy()


def grid(rule, n):
    """Valid (rows, users_count, f) triples of a rule at slot size n, edges included."""
    out = []
    for m in sorted({1, 2, 3, 4, 7, n // 2, n - 1, n}):
        for f in sorted({0, 1, 2, (m - 3) // 4 if m >= 3 else 0, (m - 1) // 2, m - 1, m, m + 2}):
            for uc in sorted({m, m + 1, max(m - 1, 0), 2 * f + 1}):
                if rule == "Krum" and uc < 2 * f + 1:
                    continue
                if rule == "Bulyan" and (uc != m or uc < 4 * f + 3):
                    continue
                out.append((m, uc, f))
    return out


@pytest.mark.parametrize("rule", ["Krum", "Bulyan", "TrimmedMean", "NoDefense", "AttackMetrics"])
def test_table_rows_equal_host_rows(env, rule):
    nat, _ = env
    n = 24
    g = grid("Krum" if rule == "AttackMetrics" else rule, n)
    rows, ucs, fs = (list(x) for x in zip(*g))
    hi, hf = host_table(nat, rule if rule != "Bulyan" else "TrimmedMean", rows, ucs, fs, n)
    di, df, st = device_table(nat, rule, n, rows, ucs, fs)
    assert not st.any()
    cols = list(ROW_INTS)
    if rule == "Bulyan":            # the rows call leaves its second-stage table; stage one's tm is TrimmedMean's
        hb, _ = host_table(nat, "Bulyan", rows, ucs, fs, n)
        assert torch.equal(di[:, [0, 1, 2, 3]], hb[:, [0, 1, 2, 3]])
        cols = [5, 6]
    assert torch.equal(di[:, cols], hi[:, cols]), rule
    torch.testing.assert_close(df[:, 7:], hf[:, 7:], rtol=1e-6, atol=0)
    # the whole-slot form (rows NULL, one users_count): afl_defend_batched_each's table
    if rule in ("Krum", "Bulyan", "TrimmedMean"):
        uc = n
        fs2 = [f for f in range(0, n + 2) if rule == "TrimmedMean" or (rule == "Krum" and uc >= 2 * f + 1)
               or (rule == "Bulyan" and uc >= 4 * f + 3)]
        hi, hf = host_table(nat, rule, None, uc, fs2, n)
        di, df, st = device_table(nat, rule, n, None, None, fs2, users_count=uc)
        assert not st.any()
        assert torch.equal(di[:, list(ROW_INTS)], hi[:, list(ROW_INTS)]), rule
        torch.testing.assert_close(df[:, 7:], hf[:, 7:], rtol=1e-6, atol=0)


def test_alie_table_rows_equal_host_rows(env):
    nat, _ = env
    fs = [0, 1, 2, 5, 24, 24, 0, 3]
    zs = [1.5, 0.0, -0.7, 1e-8, 3.0, 0.0, 0.0, np.pi]
    hi, hf = host_table(nat, "ALIE", None, None, fs, 24, zs)
    di, df, st = device_table(nat, "ALIE", 24, None, None, fs, zs=zs)
    assert not st.any()
    assert torch.equal(di, hi)


@pytest.mark.parametrize("rule", ["Krum", "Bulyan", "TrimmedMean", "NoDefense", "AttackMetrics", "ALIE"])
def test_invalid_values_flag_the_problem_and_get_the_safe_row(env, rule):
    nat, _ = env
    n = 24
    ok = (n, n, 0)
    bad = {"Krum": [((n, 10, 5), nat.AFL_ERR_PRECONDITION), ((0, 0, 0), nat.AFL_ERR_BAD_ARG), ((25, 25, 0), nat.AFL_ERR_BAD_ARG),
                    ((10, 10, -1), nat.AFL_ERR_BAD_ARG)],
           "Bulyan": [((n, n, 6), nat.AFL_ERR_PRECONDITION), ((20, 19, 1), nat.AFL_ERR_UNSUPPORTED), ((-3, -3, 0), nat.AFL_ERR_BAD_ARG),
                      ((10, 10, -2), nat.AFL_ERR_BAD_ARG), ((10, 5, 2), nat.AFL_ERR_PRECONDITION)],
           "TrimmedMean": [((0, 1, 0), nat.AFL_ERR_BAD_ARG), ((4, 4, -1), nat.AFL_ERR_BAD_ARG), ((4, 4, 2 ** 30), nat.AFL_ERR_BAD_ARG)],
           "NoDefense": [((n + 1, 1, 0), nat.AFL_ERR_BAD_ARG), ((4, 4, -1), nat.AFL_ERR_BAD_ARG)],
           "AttackMetrics": [((0, 0, 1), nat.AFL_ERR_BAD_ARG), ((4, 4, -1), nat.AFL_ERR_BAD_ARG)],
           "ALIE": [((n, n, n + 1), nat.AFL_ERR_BAD_ARG), ((n, n, -1), nat.AFL_ERR_BAD_ARG)]}[rule]
    triples = [ok] + [t for t, _ in bad] + [ok]
    rows, ucs, fs = (list(x) for x in zip(*triples))
    zs = [1.0] * len(fs)
    prior = torch.zeros(len(fs), dtype=torch.int32, device="cuda")
    prior[-1] = nat.AFL_ERR_NO_WINNER                            # sticky: a set code is never overwritten
    di, df, st = device_table(nat, rule, n, None if rule == "ALIE" else rows, None if rule == "ALIE" else ucs, fs,
                              zs=zs if rule == "ALIE" else None, status=prior)
    assert st.tolist() == [0] + [c for _, c in bad] + [nat.AFL_ERR_NO_WINNER]
    host_rule = rule if rule != "Bulyan" else "TrimmedMean"
    hi, _ = host_table(nat, host_rule, None if rule == "ALIE" else [n], [n], [0], n, zs=[1.0])
    for b in range(len(fs)):
        cols = [0, 1, 3, 4, 5, 6] if rule != "Bulyan" else [0, 1, 4, 5, 6]
        assert torch.equal(di[b, cols], hi[0, cols]), (rule, b, di[b], hi[0])
        if rule == "Bulyan":
            assert int(di[b, 2]) == n                           # theta of the safe row


# ---- bit identity with the host-parameter calls --------------------------------------------------------------------
B, N, D = 6, 40, 3000
FS = [0, 1, 3, 5, 7, 2]
ZS = [0.0, 1.5, -0.7, 2.0, 0.3, 1.0]
ROWS = [40, 35, 24, 40, 31, 19]
LAYOUTS = ["fp32", "fp32_unaligned", "bf16", "fp16"]


def make_g(layout, seed):
    gen = torch.Generator(device="cuda").manual_seed(seed)
    pitch = D + 1 if layout == "fp32_unaligned" else D
    base = torch.randn(B, N, pitch, device="cuda", generator=gen)
    base += 0.3 * torch.randn(B, 1, pitch, device="cuda", generator=gen)
    base *= torch.exp(0.25 * torch.randn(B, N, 1, device="cuda", generator=gen))
    dt = {"bf16": torch.bfloat16, "fp16": torch.float16}.get(layout, torch.float32)
    return base.to(dt)[:, :, :D]


def fill(rm, fs, zs, rows=None):
    rm.f.copy_(dev_i32(fs))
    rm.z.copy_(torch.tensor(zs, dtype=torch.float64))
    if rows is not None:
        rm.rows.copy_(dev_i32(rows))


def host_round(bt, G, fs, zs, rows, rules=("Krum", "Bulyan", "TrimmedMean", "NoDefense")):
    """The eager host-parameter calls of one round on G (modified in place by ALIE)."""
    res = {}
    res["alie"] = bt.alie_rows(G, fs, zs)
    users = N if rows is None else None
    if "Krum" in rules:
        res["krum"] = bt.krum(G, users, fs, return_index=True, rows=rows)
    if "Bulyan" in rules:
        res["bulyan"] = bt.bulyan(G, users, fs, return_selection=True, rows=rows)
    if "TrimmedMean" in rules:
        res["tm"] = bt.trimmed_mean(G, users, fs, rows=rows)
    if "NoDefense" in rules:
        res["mean"] = bt.no_defense(G, users, fs, rows=rows)
    return res


def check_selection(dev_sel, host_sel):
    w = host_sel.shape[1]
    assert torch.equal(dev_sel[:, :w], host_sel)
    assert bool((dev_sel[:, w:] == -2).all())


@pytest.mark.parametrize("ragged", [False, True], ids=["whole", "ragged"])
@pytest.mark.parametrize("layout", LAYOUTS)
def test_device_round_equals_host_calls(env, layout, ragged):
    nat, bt = env
    rows = ROWS if ragged else None
    G = make_g(layout, 1)
    Gh = G.clone()
    rm = bt.DeviceRound(G, rows=ragged)
    fill(rm, FS, ZS, rows)
    crafted, mu, sigma = rm.alie()
    idx = rm.krum(return_index=True).clone()
    krow = rm.krum().clone()
    out_b, sel = (t.clone() for t in rm.bulyan(return_selection=True))
    tm, mean = rm.trimmed_mean().clone(), rm.no_defense().clone()
    met_tm = rm.attack_metrics(aggregated=tm, return_honest_mean=True)
    met_k = rm.attack_metrics(krum_index=idx, selection=sel)
    h = host_round(bt, Gh, FS, ZS, rows)
    for a, b, what in zip((crafted, mu, sigma), h["alie"], ("crafted", "mu", "sigma")):
        assert_bits(a, b, what)
    assert_bits(G, Gh, "written rows")                    # 16-bit: the in-kernel write equals the cast route
    assert torch.equal(idx, h["krum"])
    assert_bits(krow, bt.krum(Gh, N if rows is None else None, FS, rows=rows), "krum rows")
    assert_bits(out_b, h["bulyan"][0], "bulyan")
    check_selection(sel, h["bulyan"][1])
    assert_bits(tm, h["tm"], "trimmed mean")
    assert_bits(mean, h["mean"], "mean")
    hm = bt.attack_metrics(Gh, FS, aggregated=h["tm"], return_honest_mean=True, rows=rows)
    for k in hm:
        assert_bits(met_tm[k], hm[k], k)
    hk = bt.attack_metrics(Gh, FS, krum_index=h["krum"], selection=h["bulyan"][1], rows=rows)
    for k in hk:
        assert_bits(met_k[k], hk[k], k)
    assert not rm.status.any()
    rm.raise_for_status()


# ---- status ----------------------------------------------------------------------------------------------------------
def test_flagged_problems_leave_the_others_alone(env):
    nat, bt = env
    G = make_g("fp32", 2)
    Gh = G.clone()
    rm = bt.DeviceRound(G, rows=True)
    bad_f, bad_rows = list(FS), list(ROWS)
    bad_f[1] = 30                                  # Krum and Bulyan: users_count < 2f + 1; ALIE: f > rows is fine, f <= N
    bad_rows[4] = 0                                # rows outside [1, N]
    fill(rm, bad_f, ZS, bad_rows)
    idx = rm.krum(return_index=True)
    out_b, sel = rm.bulyan(return_selection=True)
    tm = rm.trimmed_mean()
    st = rm.status.cpu().tolist()
    assert st[1] == nat.AFL_ERR_PRECONDITION and st[4] == nat.AFL_ERR_BAD_ARG
    assert [s for b, s in enumerate(st) if b not in (1, 4)] == [0] * 4
    # a batch without them: the flagged problems replaced by the safe row (N rows, f = 0), which is what they ran
    good_f = [f if b not in (1, 4) else 0 for b, f in enumerate(bad_f)]
    good_rows = [r if b not in (1, 4) else N for b, r in enumerate(bad_rows)]
    hk = bt.krum(Gh, None, good_f, return_index=True, rows=good_rows)
    hb, hs = bt.bulyan(Gh, None, good_f, return_selection=True, rows=good_rows)
    assert torch.equal(idx, hk)
    assert_bits(out_b, hb, "bulyan")
    check_selection(sel, hs)
    # f = 30 on 35 rows is valid for the trimmed mean: only problem 4 runs the safe row there
    tm_f = [f if b != 4 else 0 for b, f in enumerate(bad_f)]
    tm_rows = [r if b != 4 else N for b, r in enumerate(bad_rows)]
    assert_bits(tm, bt.trimmed_mean(Gh, None, tm_f, rows=tm_rows), "trimmed mean")
    with pytest.raises(AssertionError, match="problem 1"):
        rm.raise_for_status()
    with pytest.raises(AssertionError):
        bt.krum(Gh, None, bad_f[:2] + good_f[2:], rows=good_rows)
    rm.clear_status()
    rm.raise_for_status()


def test_raise_for_status_raises_what_the_host_call_raises(env):
    nat, bt = env
    G = make_g("fp32", 3)
    Gh = G.clone()
    # rows outside [1, N]: ValueError
    rm = bt.DeviceRound(G, rows=True)
    fill(rm, FS, ZS, ROWS[:2] + [N + 1] + ROWS[3:])
    rm.trimmed_mean()
    with pytest.raises(ValueError, match="problem 2"):
        rm.raise_for_status()
    with pytest.raises(ValueError):
        bt.trimmed_mean(Gh, None, FS, rows=ROWS[:2] + [N + 1] + ROWS[3:])
    # Bulyan's users_count != rows: NotImplementedError
    rm = bt.DeviceRound(G, rows=True, per_problem_users_count=True)
    fill(rm, FS, ZS, ROWS)
    rm.users_count.copy_(dev_i32(ROWS[:3] + [ROWS[3] - 1] + ROWS[4:]))
    rm.bulyan()
    with pytest.raises(NotImplementedError, match="problem 3"):
        rm.raise_for_status()
    with pytest.raises(NotImplementedError):
        bt.bulyan(Gh, ROWS[:3] + [ROWS[3] - 1] + ROWS[4:], FS, rows=ROWS)
    # a Bulyan round with no eligible user: KeyError(-1), the other problems unaffected
    G[3] = float("nan")
    Gh[3] = float("nan")
    rm = bt.DeviceRound(G)
    fill(rm, FS, ZS)
    out_b, sel = rm.bulyan(return_selection=True)
    assert rm.status.cpu().tolist() == [0, 0, 0, nat.AFL_ERR_NO_WINNER, 0, 0]
    with pytest.raises(KeyError) as e:
        rm.raise_for_status()
    assert e.value.args == (-1,)
    with pytest.raises(KeyError):
        bt.bulyan(Gh, N, FS)
    ok = [0, 1, 2, 4, 5]
    Gv = Gh.clone()
    Gv[3] = Gh[0]
    hb, hs = bt.bulyan(Gv, N, FS, return_selection=True)
    assert_bits(out_b[ok], hb[ok], "bulyan")
    check_selection(sel[ok], hs[ok])
    # ALIE's f > N: ValueError; the precondition: AssertionError
    rm = bt.DeviceRound(G, rules=())
    fill(rm, FS[:5] + [N + 1], ZS)
    rm.alie()
    with pytest.raises(ValueError, match="problem 5"):
        rm.raise_for_status()
    with pytest.raises(ValueError):
        bt.alie_rows(Gh.clone(), FS[:5] + [N + 1], ZS)


# ---- capture ---------------------------------------------------------------------------------------------------------
def test_captured_round_replays_refilled_grids(env):
    nat, bt = env
    from attacking_federate_learning_b200 import _device
    G = make_g("fp32", 4).contiguous()
    rm = bt.DeviceRound(G, rows=True)
    w = torch.zeros(B, D, device="cuda")
    v = torch.zeros(B, D, device="cuda")

    def round_():
        crafted, mu, sigma = rm.alie()
        idx = rm.krum(return_index=True)
        out_b, sel = rm.bulyan(return_selection=True)
        tm = rm.trimmed_mean()
        mean = rm.no_defense()
        met = rm.attack_metrics(aggregated=out_b, selection=sel)
        met_k = rm.attack_metrics(krum_index=idx)
        _device.momentum_step(w, v, mean, 0.9, 0.1)
        return dict(crafted=crafted, mu=mu, sigma=sigma, idx=idx, bulyan=out_b, sel=sel, tm=tm, mean=mean,
                    rel=met["rel_deviation"], frac=met["bulyan_malicious_fraction"], rel_k=met_k["rel_deviation"],
                    hit=met_k["krum_success"])

    fill(rm, FS, ZS, ROWS)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        round_()                                                 # eager warm-up
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        outs = round_()

    def check(seed, fs, zs, rows):
        new = make_g("fp32", seed)
        G.copy_(new)
        fill(rm, fs, zs, rows)
        w0, v0 = torch.randn(B, D, device="cuda"), torch.randn(B, D, device="cuda")
        w.copy_(w0), v.copy_(v0)
        graph.replay()
        torch.cuda.synchronize()
        Gh = new.clone()
        h = host_round(bt, Gh, fs, zs, rows)
        for a, b, what in zip((outs["crafted"], outs["mu"], outs["sigma"]), h["alie"], ("crafted", "mu", "sigma")):
            assert_bits(a, b, what)
        assert_bits(G, Gh, "written rows")
        assert torch.equal(outs["idx"], h["krum"])
        assert_bits(outs["bulyan"], h["bulyan"][0], "bulyan")
        check_selection(outs["sel"], h["bulyan"][1])
        assert_bits(outs["tm"], h["tm"], "trimmed mean")
        assert_bits(outs["mean"], h["mean"], "mean")
        hm = bt.attack_metrics(Gh, fs, aggregated=h["bulyan"][0], selection=h["bulyan"][1], rows=rows)
        assert_bits(outs["rel"], hm["rel_deviation"], "rel")
        assert_bits(outs["frac"], hm["bulyan_malicious_fraction"], "fraction")
        hk = bt.attack_metrics(Gh, fs, krum_index=h["krum"], rows=rows)
        assert_bits(outs["rel_k"], hk["rel_deviation"], "rel krum")
        assert torch.equal(outs["hit"], hk["krum_success"])
        _device.momentum_step(w0, v0, h["mean"], 0.9, 0.1)
        assert_bits(w, w0, "weights")
        assert_bits(v, v0, "velocity")
        assert not rm.status.any()

    check(10, [2, 0, 4, 1, 9, 3], [1.0, 0.5, 0.0, -1.2, 2.5, 0.7], [40, 12, 33, 27, 40, 15])
    check(11, [5, 5, 5, 5, 5, 5], [1.5] * 6, [40] * 6)
    check(12, [0, 0, 1, 3, 2, 8], [0.0, 3.0, 1.0, 1.0, 0.2, 0.9], [3, 7, 40, 20, 11, 39])
    # an eager module-level call that grows the shared workspace cache must not disturb the captured round
    big = torch.randn(64, 128, 4096, device="cuda")
    bt.krum(big, 128, 10, return_index=True)
    bt.bulyan(big, 128, 10)
    torch.cuda.synchronize()
    check(13, [1, 2, 3, 4, 5, 6], [0.5, 1.0, 1.5, 2.0, 2.5, 3.0], [40, 39, 38, 37, 36, 35])
