"""Pin the torch restatement of Bulyan's selection (oracle/ref_torch.py), which the GPU tests use as the float64
reference at n >= 2048, to the C oracle (oracle/oracle.c) on CPU tensors."""
import numpy as np
import pytest

from oracle import c_oracle as co

torch = pytest.importorskip("torch")
from oracle import ref_torch as rt  # noqa: E402


def _table(rng, n, d, alie_f=0, inf_rows=()):
    G = (0.1 * rng.standard_normal(d) + np.exp(0.25 * rng.standard_normal((n, 1))) * rng.standard_normal((n, d))).astype(np.float32)
    if alie_f:
        G[:alie_f] = G[:alie_f].mean(0) - 1.0 * G[:alie_f].std(0)        # identical rows: exact score ties
    t = np.sqrt(co.pairwise_sqdist(G)).astype(np.float32).astype(np.float64)
    for u in inf_rows:                                                   # a client whose row holds an inf
        t[u, :] = np.inf; t[:, u] = np.inf; t[u, u] = 0.0
    return t


@pytest.mark.parametrize("n,f,alie,n_inf,seed", [(3, 0, False, 0, 0), (7, 1, False, 0, 1), (11, 2, True, 0, 2),
                                                 (31, 7, False, 3, 3), (64, 15, True, 0, 4), (100, 24, True, 5, 5),
                                                 (203, 50, False, 0, 6), (300, 70, True, 20, 7)])
def test_bulyan_select_matches_c_oracle(n, f, alie, n_inf, seed):
    rng = np.random.default_rng(900 + seed)
    inf_rows = rng.choice(np.arange(f, n), size=n_inf, replace=False) if n_inf else ()
    t = _table(rng, n, 48, alie_f=f if alie else 0, inf_rows=inf_rows)
    want, want_m = co.bulyan_select(t, n, f, with_margins=True)
    got, got_m = rt.bulyan_select(torch.from_numpy(t), n, f, with_margins=True)
    assert got == want
    assert got_m == want_m                                               # same float64 sums in the same order
    assert not set(got) & set(int(u) for u in inf_rows)
    if alie and f >= 2:
        assert 0.0 in got_m                                              # the ALIE block produced exact ties


def test_bulyan_select_stops_without_eligible_user():
    """Every score >= 1e20 from round 0: no selection, as orc_bulyan_select_m (the reference raises KeyError(-1))."""
    n, f = 7, 1
    t = np.full((n, n), 1e30)
    np.fill_diagonal(t, 0.0)
    assert co.bulyan_select(t, n, f) == [] == rt.bulyan_select(torch.from_numpy(t), n, f)


def test_bulyan_select_float32_table_and_python_slice():
    """An fp32 input table is widened exactly; f = 0 keeps every alive neighbour (slice past the end)."""
    rng = np.random.default_rng(17)
    n = 40
    t = _table(rng, n, 16).astype(np.float32)
    assert rt.bulyan_select(torch.from_numpy(t), n, 0) == co.bulyan_select(t.astype(np.float64), n, 0)
