"""The rest of the NumPy drop-in surface on the host-buffer engine (run on an H100 with -m gpu):
afl_sqdist_host (`_krum_create_distances`, `krum(..., return_index=True)`), afl_bulyan_host
(`bulyan(..., return_selection=True)`) and afl_alie_host (`Attack.attack` on NumPy users).

AFL_HOST_DEVICE_BYTES caps the device memory a call may hold; the `budget` fixture sets it to unlimited, a partial
resident prefix (Bulyan) or a third ring slot (the others), and ring only.  Every result must be bit-identical to a
slab-wise device route built from the public device entry points with the same slab boundaries.
"""
import ctypes as C
import os
import re

import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

ENV = "AFL_HOST_DEVICE_BYTES"


@pytest.fixture(scope="module")
def api():
    if not torch.cuda.is_available():
        pytest.skip("no GPU")
    from attacking_federate_learning_b200 import defences, malicious, _device, _native
    _native.lib()
    return defences, malicious, _device, _native


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


def hetero(rng, n, d):
    return (0.1 * rng.standard_normal(d) + np.exp(0.25 * rng.standard_normal((n, 1))) * rng.standard_normal((n, d))).astype(np.float32)


def host_matrix(G, extra):
    """G as a view of a wider C array: host pitch ld = d + extra."""
    n, d = G.shape
    W = np.zeros((n, d + extra), np.float32)
    W[:, :d] = G
    return W[:, :d], d + extra


def slab_width(rows, d, slab_cols):
    """Columns per slab as the host entry points round them."""
    if slab_cols <= 0:
        slab_cols = (96 << 20) // (rows * 4)
    return min(max(32, (slab_cols + 31) // 32 * 32), (d + 31) // 32 * 32)


def same_bits(a, b):
    a, b = np.asarray(a), np.asarray(b)
    return a.shape == b.shape and np.array_equal(a.view(np.uint32), b.view(np.uint32))


def padded(G):
    """G on the device at the host path's padded pitch (16-byte aligned rows: the tensor-core Gram path)."""
    n, d = G.shape
    Gd = torch.zeros((n, (d + 31) // 32 * 32), dtype=torch.float32, device="cuda")[:, :d]
    Gd.copy_(torch.from_numpy(np.ascontiguousarray(G)))
    return Gd


def slabwise_sqdist(dev, G, slab_cols):
    n, d = G.shape
    Gd, w = padded(G), slab_width(n, d, slab_cols)
    d2 = None
    for c0 in range(0, d, w):
        part = dev.sqdist_partial(Gd[:, c0:min(d, c0 + w)])
        d2 = part if d2 is None else d2 + part
    return d2


# ---- direct C calls ----------------------------------------------------------------------------------------------
def call_sqdist(nat, Gh, ld, slab_cols):
    n, d = Gh.shape
    d2 = torch.full((n, n), float("nan"), dtype=torch.float64, device="cuda")
    torch.cuda.synchronize()
    rc = nat.lib().afl_sqdist_host(Gh.ctypes.data, n, d, ld, d2.data_ptr(), slab_cols)
    return rc, d2, nat.lib().afl_last_error().decode() if rc else ""


def call_bulyan(nat, Gh, ld, f, slab_cols):
    n, d = Gh.shape
    out = np.full(d, np.nan, np.float32)
    sel = np.full(n - 2 * f, -7, np.int32)
    rc = nat.lib().afl_bulyan_host(Gh.ctypes.data, n, d, ld, n, f, out.ctypes.data, sel.ctypes.data, slab_cols)
    return rc, (out, sel), nat.lib().afl_last_error().decode() if rc else ""


def call_alie(nat, rows, z, slab_cols, alias=True):
    f, d = len(rows), rows[0].size
    mu, sigma = np.full(d, np.nan, np.float32), np.full(d, np.nan, np.float32)
    crafted = mu if alias else np.full(d, np.nan, np.float32)
    ptrs = (C.c_void_p * f)(*[r.ctypes.data for r in rows])
    rc = nat.lib().afl_alie_host(ptrs, f, d, float(z), mu.ctypes.data, sigma.ctypes.data, crafted.ctypes.data, slab_cols)
    return rc, (mu, sigma, crafted), nat.lib().afl_last_error().decode() if rc else ""


def needs(call, set_budget, who):
    """The minimal footprint, as stated by the error for a budget that is far too small."""
    set_budget(1)
    rc, _, msg = call()
    assert rc == 4, msg                                   # AFL_ERR_UNSUPPORTED -> NotImplementedError
    assert msg.startswith(who + ": needs"), msg
    return int(re.search(r"needs (\d+) bytes", msg).group(1))


def budgets(call, set_budget, who, slab_bytes, nslab):
    """unlimited, partial resident prefix (Bulyan) / a third ring slot (the others), ring only."""
    need = needs(call, set_budget, who)
    out = {"unlimited": None, "ring": need + slab_bytes // 2}
    if nslab >= 2:
        out["partial"] = need + 256 + max(1, nslab // 2) * slab_bytes + slab_bytes // 2
    return out


def run_budgets(call, set_budget, who, slab_bytes, nslab):
    got = {}
    for name, nbytes in budgets(call, set_budget, who, slab_bytes, nslab).items():
        set_budget(nbytes)
        rc, res, msg = call()
        assert rc == 0, (name, msg)
        got[name] = res
    set_budget(None)
    return got


# (n, d, extra host pitch, slab_cols, f)
CASES = [
    (1, 300, 0, 64, 0),          # one client
    (2, 1000, 5, 96, 0),         # two clients, ld > d
    (40, 100, 0, 128, 9),        # a single slab
    (40, 250, 3, 128, 9),        # two slabs, d % 32 != 0, ld > d, last slab partly filled
    (40, 1000, 0, 96, 9),        # eleven slabs, last one 40 columns wide
    (100, 70000, 0, 32768, 24),  # N <= 128: single-tile bf16x2 slabs and a split-TF32 tail slab
    (150, 997, 11, 160, 20),     # N > 128: two tiles, centred bf16x2 operands; odd d
]


@pytest.mark.parametrize("n,d,extra,slab_cols,f", CASES)
def test_sqdist_and_krum_index_match_slabwise_route(api, budget, n, d, extra, slab_cols, f):
    D, M, dev, nat = api
    rng = np.random.default_rng(2000 + n + d)
    G = hetero(rng, n, d)
    if n >= 20:
        G[:f] = 0.5 * G[f]                                # identical rows: exact Krum ties
    Gh, ld = host_matrix(G, extra)
    want = slabwise_sqdist(dev, G, slab_cols).cpu().numpy()
    w = slab_width(n, d, slab_cols)
    got = run_budgets(lambda: call_sqdist(nat, Gh, ld, slab_cols), budget, "afl_sqdist_host", n * w * 4, -(-d // w))
    for name, d2 in got.items():
        assert same_bits(d2.cpu().numpy(), want), name
    if n >= 2 * f + 1:                                    # the same table as the Krum branch of afl_defend_host
        idx = C.c_int(-7)
        rc = nat.lib().afl_defend_host(b"Krum", Gh.ctypes.data, n, d, ld, n, f, None, C.byref(idx), slab_cols)
        assert rc == 0
        assert idx.value == int(dev.krum_from_sqdist(got["ring"], n, f).item())

    # the NumPy API (C-contiguous matrix, default slab width)
    want0 = slabwise_sqdist(dev, G, 0)
    table = D._krum_create_distances(G)
    assert same_bits(table.dense.cpu().numpy(), dev.sqdist_to_dist(want0).cpu().numpy())
    if n >= 2 * f + 1:
        i = D.krum(G, n, f, return_index=True)
        assert isinstance(i, int) and i == int(dev.krum_from_sqdist(want0, n, f).item())
        row = D.krum(G, n, f)
        assert np.shares_memory(row, G) and row.ctypes.data == G[i].ctypes.data


def test_krum_index_without_assert_and_against_c_oracle(api, budget):
    D, M, dev, nat = api
    from oracle import c_oracle as co
    rng = np.random.default_rng(31)
    n, d, f = 100, 40960, 24
    G = hetero(rng, n, d)
    want, margin = co.krum_select(np.sqrt(co.pairwise_sqdist(G)), n, f, with_margin=True)
    got = D.krum(G, n, f, return_index=True)
    assert got == want or 0.0 < margin <= 1e-5, (got, want, margin)
    assert same_bits(D.krum(G, n, f), G[got])
    # users_count < 2f + 1: the reference skips its assert when it only wants the index
    with pytest.raises(AssertionError):
        D.krum(G, 10, 5)
    i = D.krum(G, 10, 5, return_index=True)
    assert i == int(dev.krum_from_sqdist(slabwise_sqdist(dev, G, 0), 10, 5).item())


@pytest.mark.parametrize("n,d,extra,slab_cols,f", [c for c in CASES if c[0] >= 4 * c[4] + 3])
def test_bulyan_selection_matches_slabwise_route(api, budget, n, d, extra, slab_cols, f):
    D, M, dev, nat = api
    rng = np.random.default_rng(3000 + n + d)
    G = hetero(rng, n, d)
    if n >= 20:
        G[:f] = 0.5 * G[f]
    Gh, ld = host_matrix(G, extra)
    Gd = padded(G)
    sel_d = dev.bulyan_select(dev.sqdist_to_dist(slabwise_sqdist(dev, G, slab_cols)), n, f)
    want_out, want_sel = dev.trimmed_mean(Gd, 2 * f, row_index=sel_d).cpu().numpy(), sel_d.cpu().numpy()
    assert want_sel[-1] >= 0
    w = slab_width(n, d, slab_cols)
    got = run_budgets(lambda: call_bulyan(nat, Gh, ld, f, slab_cols), budget, "afl_bulyan_host", n * w * 4, -(-d // w))
    for name, (out, sel) in got.items():
        assert np.array_equal(sel, want_sel), name
        assert same_bits(out, want_out), name
    # the same call through afl_defend_host
    out = np.empty(d, np.float32)
    assert nat.lib().afl_defend_host(b"Bulyan", Gh.ctypes.data, n, d, ld, n, f, out.ctypes.data, None, slab_cols) == 0
    assert same_bits(out, want_out)

    # the NumPy API (C-contiguous matrix, default slab width)
    sel0 = dev.bulyan_select(dev.sqdist_to_dist(slabwise_sqdist(dev, G, 0)), n, f)
    out, sel = D.bulyan(G, n, f, return_selection=True)
    assert sel.dtype == np.int32 and np.array_equal(sel, sel0.cpu().numpy())
    assert same_bits(out, dev.trimmed_mean(Gd, 2 * f, row_index=sel0).cpu().numpy())
    assert same_bits(out, D.bulyan(G, n, f))


def test_failed_bulyan_round_returns_marked_selection(api, budget):
    D, M, dev, nat = api
    n, d, f, slab_cols = 40, 1000, 9, 96
    G = np.zeros((n, d), np.float32)
    G[np.arange(n), np.arange(n)] = 1e30
    want = dev.bulyan_select(dev.sqdist_to_dist(slabwise_sqdist(dev, G, slab_cols)), n, f).cpu().numpy()
    assert want[-1] < 0
    w = slab_width(n, d, slab_cols)
    for nbytes in (None, needs(lambda: call_bulyan(nat, G, d, f, slab_cols), budget, "afl_bulyan_host") + n * w * 4 // 2):
        budget(nbytes)
        rc, (_, sel), _ = call_bulyan(nat, G, d, f, slab_cols)
        assert rc == nat.AFL_ERR_NO_WINNER
        assert np.array_equal(sel, want)
    budget(None)
    with pytest.raises(KeyError) as e:
        D.bulyan(G, n, f, return_selection=True)
    assert e.value.args == (-1,)


# ---- ALIE ----------------------------------------------------------------------------------------------------------
class User:
    def __init__(self, grads):
        self.grads = grads
        self.original_params = None
        self.learning_rate = 0.1


def user_arrays(rng, f, d, kind):
    """f gradient vectors of length d, each its own allocation: C-contiguous float32, strided float32 or float64."""
    out = []
    for i in range(f):
        g = (np.exp(0.3 * rng.standard_normal()) * rng.standard_normal(d)).astype(np.float32)
        if kind == "strided":
            big = np.zeros(2 * d, np.float32)
            big[::2] = g
            g = big[::2]
        elif kind == "float64":
            g = g.astype(np.float64)
        out.append(g)
    return out


def device_alie(dev, arrays, z, alias):
    rows = torch.from_numpy(np.stack([np.asarray(a, np.float32) for a in arrays])).cuda()
    crafted, mu, sigma = dev.alie(rows, z, None, alias_mean=alias)
    return crafted.cpu().numpy(), mu.cpu().numpy(), sigma.cpu().numpy()


@pytest.mark.parametrize("f", [1, 2, 24, 240])
@pytest.mark.parametrize("z", [0.0, 1.5])
@pytest.mark.parametrize("kind", ["contiguous", "strided", "float64"])
def test_drift_attack_numpy_users(api, budget, f, z, kind):
    D, M, dev, nat = api
    rng = np.random.default_rng(f * 10 + int(z * 2))
    d = 1001 if f < 240 else 250_007                        # f = 240: three slabs at the default width
    arrays = user_arrays(rng, f, d, kind)
    if f >= 2:
        arrays[1][5] = np.inf
        arrays[0][7] = -np.inf
        arrays[1][7] = np.inf                                 # inf - inf: NaN statistics
    crafted, mu, sigma = device_alie(dev, arrays, z, alias=z != 0)
    w = slab_width(f, d, 0)
    users = [User(a) for a in arrays]
    budget(needs(lambda: call_alie(nat, [np.ascontiguousarray(a, np.float32) for a in arrays], z, 0), budget, "afl_alie_host")
           + f * w * 4 // 2)                                 # ring only
    att = M.DriftAttack(z)
    att.attack(users)
    budget(None)
    assert same_bits(att.grads_stdev, sigma)
    if z == 0:                                                # statistics only: the users keep their arrays
        assert same_bits(att.grads_mean, mu)
        assert all(u.grads is a for u, a in zip(users, arrays))
    else:
        assert same_bits(att.grads_mean, crafted)
        assert all(u.grads is att.grads_mean for u in users)


@pytest.mark.parametrize("f", [1, 2, 24, 240])
@pytest.mark.parametrize("d,slab_cols", [(1000, 96), (997, 32), (2049, 1024), (100, 128)])
def test_alie_host_narrow_slabs_ring_only(api, budget, f, d, slab_cols):
    """Slots at pitch slab_cols (16-byte loads) against one afl_alie on the stacked matrix at pitch d (scalar loads
    when d % 4 != 0), under a ring-only budget; with and without the mu/crafted aliasing."""
    D, M, dev, nat = api
    rng = np.random.default_rng(7 * f + d)
    rows = user_arrays(rng, f, d, "contiguous")
    rows[0][d // 2] = np.inf
    w = slab_width(f, d, slab_cols)
    for alias in (True, False):                           # without the aliasing the call holds one more vector
        budget(needs(lambda: call_alie(nat, rows, 1.5, slab_cols, alias=alias), budget, "afl_alie_host") + f * w * 4 // 2)
        rc, (mu, sigma, crafted), msg = call_alie(nat, rows, 1.5, slab_cols, alias=alias)
        assert rc == 0, msg
        want_c, want_mu, want_s = device_alie(dev, rows, 1.5, alias)
        assert same_bits(sigma, want_s) and same_bits(crafted, want_c)
        assert same_bits(mu, want_c if alias else want_mu)


def test_attack_hook_path(api):
    """A subclass that replaces the hook gets (mu, sigma) from the statistics-only call, then runs its hook once."""
    D, M, dev, nat = api

    class Hooked(M.DriftAttack):
        calls = 0

        def _attack_grads(self, grads_mean, grads_stdev, original_params, learning_rate):
            Hooked.calls += 1
            return super()._attack_grads(grads_mean, grads_stdev, original_params, learning_rate)

    rng = np.random.default_rng(4)
    arrays = user_arrays(rng, 24, 5003, "contiguous")
    crafted, mu, sigma = device_alie(dev, arrays, 1.5, alias=True)
    users = [User(a) for a in arrays]
    att = Hooked(1.5)
    att.attack(users)
    assert Hooked.calls == 1
    assert same_bits(att.grads_stdev, sigma)
    assert same_bits(att.grads_mean, crafted)                 # the hook shifted mu in place
    assert all(u.grads is att.grads_mean for u in users)


def test_budget_too_small_for_each_entry_point(api, budget):
    D, M, dev, nat = api
    rng = np.random.default_rng(9)
    n, d, f = 40, 5000, 9
    G = hetero(rng, n, d)
    users = [User(G[i].copy()) for i in range(f)]
    budget(1 << 16)
    for name, call in (("afl_sqdist_host", lambda: D._krum_create_distances(G)),
                       ("afl_sqdist_host", lambda: D.krum(G, n, f, return_index=True)),
                       ("afl_bulyan_host", lambda: D.bulyan(G, n, f, return_selection=True)),
                       ("afl_alie_host", lambda: M.DriftAttack(1.5).attack(users))):
        with pytest.raises(NotImplementedError, match=r"needs \d+ bytes of device memory") as e:
            call()
        assert str(e.value).startswith(name), str(e.value)
        assert int(re.search(r"needs (\d+) bytes", str(e.value)).group(1)) > 1 << 16
    assert all(u.grads is not users[0].grads for u in users[1:])   # the failed attack assigned nothing


def test_distances_past_the_selection_limit(api):
    """n = 5000 > 4096: selection refuses it, but the distance table still streams (SIMT Gram kernel)."""
    D, M, dev, nat = api
    rng = np.random.default_rng(12)
    n, d = 5000, 64
    G = hetero(rng, n, d)
    table = D._krum_create_distances(G)
    want = dev.sqdist_to_dist(dev.sqdist_partial(padded(G)))
    assert table.dense.shape == (n, n)
    assert same_bits(table.dense.cpu().numpy(), want.cpu().numpy())
