"""Host-buffer entry point (afl_defend_host) with a bounded device budget (run on an H100 with -m gpu).

The matrix stays in host memory and goes through a ring of device slab slots; Bulyan keeps as many leading slabs
resident as the budget allows and re-streams only its selected rows for the rest.  AFL_HOST_DEVICE_BYTES caps the
device memory the call may hold, which lets these tests force every streaming case on small inputs.

Every result must be bit-identical
  * across budgets: unlimited (Bulyan fully resident), a partial resident prefix, and ring only;
  * to a slab-wise device route built from the public device entry points with the same slab boundaries:
    d2 = sum over slabs of afl_sqdist_partial, added in float64 in slab order, then afl_krum_from_sqdist or
    afl_sqdist_to_dist -> afl_bulyan_select -> afl_trimmed_mean(row_index = sel); afl_trimmed_mean / afl_mean
    on the whole device matrix for the column rules.
The host call does not return Bulyan's selection; it is checked through the output vector, which depends on the
selected rows and on their order.
"""
import ctypes as C
import os
import re

import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

ENV = "AFL_HOST_DEVICE_BYTES"
RULES = ("Krum", "TrimmedMean", "NoDefense", "Bulyan")


@pytest.fixture(scope="module")
def api():
    if not torch.cuda.is_available():
        pytest.skip("no GPU")
    from attacking_federate_learning_b200 import defences, _device, _native
    _native.lib()
    return defences, _device, _native


@pytest.fixture
def budget():
    """Setter for AFL_HOST_DEVICE_BYTES (None = unset); the variable is restored when the test ends."""
    saved = os.environ.get(ENV)

    def set_budget(nbytes):
        if nbytes is None:
            os.environ.pop(ENV, None)
        else:
            os.environ[ENV] = str(int(nbytes))
    yield set_budget
    if saved is None:
        os.environ.pop(ENV, None)
    else:
        os.environ[ENV] = saved
    assert os.environ.get(ENV) == saved


def hetero(rng, n, d):
    return (0.1 * rng.standard_normal(d) + np.exp(0.25 * rng.standard_normal((n, 1))) * rng.standard_normal((n, d))).astype(np.float32)


def host_matrix(G, extra):
    """G as a view of a wider C array: host pitch ld = d + extra."""
    n, d = G.shape
    W = np.zeros((n, d + extra), np.float32)
    W[:, :d] = G
    return W[:, :d], d + extra


def slab_width(n, d, slab_cols):
    """Columns per slab as afl_defend_host rounds them (never wider than the padded matrix)."""
    if slab_cols <= 0:
        slab_cols = (96 << 20) // (n * 4)
    return min(max(32, (slab_cols + 31) // 32 * 32), (d + 31) // 32 * 32)


def call_host(nat, rule, Gh, ld, f, slab_cols):
    """afl_defend_host through ctypes.  Returns (rc, output vector, index, error message)."""
    n, d = Gh.shape
    out = np.full(d, np.nan, np.float32)
    idx = C.c_int(-7)
    rc = nat.lib().afl_defend_host(rule.encode(), Gh.ctypes.data, n, d, ld, n, f, out.ctypes.data, C.byref(idx), slab_cols)
    msg = nat.lib().afl_last_error().decode() if rc else ""
    return rc, out, idx.value, msg


def bytes_needed(nat, rule, Gh, ld, f, slab_cols, set_budget):
    """The minimal footprint, as stated by the error for a budget that is far too small."""
    set_budget(1)
    rc, _, _, msg = call_host(nat, rule, Gh, ld, f, slab_cols)
    assert rc == nat.AFL_ERR_UNSUPPORTED, msg
    m = re.search(r"needs (\d+) bytes", msg)
    assert m, msg
    return int(m.group(1))


def device_route(dev, rule, G, f, slab_cols):
    """The same arithmetic from the device entry points, slab by slab at the host path's slab boundaries."""
    n, d = G.shape
    ld = (d + 31) // 32 * 32                      # 16-byte aligned rows: the tensor-core Gram path, as on the host path
    Gd = torch.zeros((n, ld), dtype=torch.float32, device="cuda")[:, :d]
    Gd.copy_(torch.from_numpy(np.ascontiguousarray(G)))
    if rule == "TrimmedMean":
        return dev.trimmed_mean(Gd, f).cpu().numpy(), None
    if rule == "NoDefense":
        return dev.mean(Gd).cpu().numpy(), None
    w = slab_width(n, d, slab_cols)
    d2 = None
    for c0 in range(0, d, w):
        part = dev.sqdist_partial(Gd[:, c0:min(d, c0 + w)])
        d2 = part if d2 is None else d2 + part
    if rule == "Krum":
        return None, int(dev.krum_from_sqdist(d2, n, f).item())
    sel = dev.bulyan_select(dev.sqdist_to_dist(d2), n, f)
    return dev.trimmed_mean(Gd, 2 * f, row_index=sel).cpu().numpy(), sel.cpu().numpy()


def same_bits(a, b):
    return np.array_equal(np.asarray(a).view(np.uint32), np.asarray(b).view(np.uint32))


def budgets_for(nat, rule, Gh, ld, f, slab_cols, set_budget):
    """unlimited, partial resident prefix (Bulyan) / a third ring slot (others), ring only."""
    n, d = Gh.shape
    w = slab_width(n, d, slab_cols)
    nslab = -(-d // w)
    slab_bytes = n * w * 4
    need = bytes_needed(nat, rule, Gh, ld, f, slab_cols, set_budget)
    out = {"unlimited": None, "ring": need + slab_bytes // 2}
    if nslab >= 2:
        out["partial"] = need + 256 + max(1, nslab // 2) * slab_bytes + slab_bytes // 2
    return out


# (n, d, extra host pitch, slab_cols, f)
CASES = [
    (1, 300, 0, 64, 0),          # one client
    (2, 1000, 5, 96, 0),         # two clients, ld > d
    (40, 100, 0, 128, 9),        # a single slab
    (40, 250, 3, 128, 9),        # two slabs (fewer than ring slots), d % 32 != 0, ld > d, last slab partly filled
    (40, 1000, 0, 96, 9),        # eleven slabs, last one 40 columns wide
    (100, 70000, 0, 32768, 24),  # N <= 128: single-tile bf16x2 slabs and a split-TF32 tail slab
    (150, 997, 11, 160, 20),     # N > 128: two tiles, centred bf16x2 operands; odd d
]


@pytest.mark.parametrize("n,d,extra,slab_cols,f", CASES)
def test_budgets_agree_with_slabwise_device_route(api, budget, n, d, extra, slab_cols, f):
    D, dev, nat = api
    rng = np.random.default_rng(1000 + n + d)
    G = hetero(rng, n, d)
    if n >= 20:
        G[:f] = 0.5 * G[f]                        # identical rows: exact Krum ties
    Gh, ld = host_matrix(G, extra)
    for rule in RULES:
        if rule == "Bulyan" and n < 4 * f + 3 or rule == "Krum" and n < 2 * f + 1:
            continue
        want_vec, want_sel = device_route(dev, rule, G, f, slab_cols)
        if rule == "Bulyan":
            assert want_sel[-1] >= 0
        got = {}
        for name, nbytes in budgets_for(nat, rule, Gh, ld, f, slab_cols, budget).items():
            budget(nbytes)
            rc, out, idx, msg = call_host(nat, rule, Gh, ld, f, slab_cols)
            assert rc == 0, (rule, name, msg)
            got[name] = (out, idx)
        budget(None)
        for name, (out, idx) in got.items():
            if rule == "Krum":
                assert idx == want_sel, (name, idx, want_sel)
                assert same_bits(out, G[idx]), name
            else:
                assert idx == -1
                assert same_bits(out, want_vec), (rule, name)


def test_numpy_api_default_slab_width(api, budget):
    """The NumPy calls pass slab_cols = 0 (about 96 MB per slab): three slabs here, the last one partly filled."""
    D, dev, nat = api
    n, d, f = 24, 2_500_000, 5
    rng = np.random.default_rng(21)
    G = hetero(rng, n, d)
    w = slab_width(n, d, 0)
    assert -(-d // w) == 3
    want = {r: device_route(dev, r, G, f, 0) for r in RULES}
    slab_bytes = n * w * 4
    for nbytes in (None, bytes_needed(nat, "Bulyan", G, d, f, 0, budget) + slab_bytes + slab_bytes // 2,
                   bytes_needed(nat, "Bulyan", G, d, f, 0, budget) + slab_bytes // 2):
        budget(nbytes)
        row = D.krum(G, n, f)
        assert np.shares_memory(row, G) and (row.ctypes.data - G.ctypes.data) == want["Krum"][1] * G.strides[0]
        assert same_bits(D.trimmed_mean(G, n, f), want["TrimmedMean"][0])
        assert same_bits(D.no_defense(G, n, f), want["NoDefense"][0])
        assert same_bits(D.bulyan(G, n, f), want["Bulyan"][0])


def test_alie_rows_ring_only_tie_to_user_1(api, budget):
    """ALIE makes rows 0..f-1 identical; with the matrix streamed through the ring the tie still goes to user 1."""
    D, dev, nat = api
    rng = np.random.default_rng(5)
    n, d, f, slab_cols = 80, 40960, 19, 8192
    G = 5.0 * hetero(rng, n, d); G[:f] = 0.002 * G[f]
    budget(bytes_needed(nat, "Krum", G, d, f, slab_cols, budget))
    rc, out, idx, msg = call_host(nat, "Krum", G, d, f, slab_cols)
    assert rc == 0, msg
    assert idx == 1 and same_bits(out, G[1])
    assert device_route(dev, "Krum", G, f, slab_cols)[1] == 1


def test_failed_bulyan_round_streaming(api, budget):
    """Rows whose distances overflow to inf leave no eligible user: the round fails before anything is re-streamed,
    and the NumPy call raises KeyError(-1) as the reference does."""
    D, dev, nat = api
    n, d, f, slab_cols = 40, 1000, 9, 96
    G = np.zeros((n, d), np.float32)
    G[np.arange(n), np.arange(n)] = 1e30
    assert device_route(dev, "Bulyan", G, f, slab_cols)[1][-1] < 0
    budget(bytes_needed(nat, "Bulyan", G, d, f, slab_cols, budget) + n * slab_cols * 4 // 2)     # ring only
    rc, _, _, _ = call_host(nat, "Bulyan", G, d, f, slab_cols)
    assert rc == nat.AFL_ERR_NO_WINNER
    budget(None)
    with pytest.raises(KeyError) as e:
        D.bulyan(G, n, f)
    assert e.value.args == (-1,)


def test_budget_too_small(api, budget):
    D, dev, nat = api
    rng = np.random.default_rng(9)
    n, d, f = 40, 5000, 9
    G = hetero(rng, n, d)
    budget(1 << 16)
    with pytest.raises(NotImplementedError, match=r"needs \d+ bytes of device memory") as e:
        D.trimmed_mean(G, n, f)
    need = int(re.search(r"needs (\d+) bytes", str(e.value)).group(1))
    assert need > 1 << 16
    budget(need)                                  # exactly the stated footprint is enough
    assert same_bits(D.trimmed_mean(G, n, f), device_route(dev, "TrimmedMean", G, f, 0)[0])
    budget(need - 1)
    with pytest.raises(NotImplementedError):
        D.trimmed_mean(G, n, f)
