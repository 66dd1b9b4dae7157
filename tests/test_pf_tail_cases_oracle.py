"""CPU companion of test_gpu_pf_tail_edges.py: each raw weight case of _pf_tail_cases.py produces the class it was built for in
the oracle, and the oracle's searches relate as the GPU test needs them to.

  * S is inf, NaN, overflowed or subnormal as named; the first non-finite weight sits at the intended slot (first tile, tile
    edge, last tile, last slot at the tail shapes of an H100 SXM).
  * On the S = inf cases the reference's linear scan and a plain lower bound give different ancestors: a search that lets
    NaN count as a match (as the lower bound does) cannot pass the GPU test.
  * The lower bound on the running maximum (the oracle's search above 16384 particles) gives the linear scan's ancestors on
    every case, PF and MCL.
  * N_eff of the border cases sits on n * threshold or one ulp either side, with threshold = N_eff / n at n = 2^k."""
import math

import numpy as np
import pytest

import _pf_tail_cases as tc
import _weight_cases as wc

SEED = 23
SMS = 132


def _tile(n):
    return tc.NT * tc.pf3_shape(n, SMS)[1]


def test_tail_shapes():
    """the shapes the GPU test names: one tile; K = 1 over many tiles; K > 1 with a partial last tile; 2^18"""
    assert tc.pf3_shape(tc.SIZES["one_tile"], SMS) == (1, 1)
    t, k = tc.pf3_shape(tc.SIZES["k1_tiles"], SMS)
    assert k == 1 and t > 1
    n = tc.SIZES["k3_partial"]
    t, k = tc.pf3_shape(n, SMS)
    assert k > 1 and n % (tc.NT * k) != 0 and (t - 1) * tc.NT * k < n
    t, k = tc.pf3_shape(tc.SIZES["2^18"], SMS)
    assert t * tc.NT * k == 1 << 18 and k > 1


@pytest.mark.parametrize("size", list(tc.SIZES))
@pytest.mark.parametrize("case", tc.TAIL_CASES, ids=lambda c: c.name)
def test_case_hits_its_class(size, case):
    n = tc.SIZES[size]
    T = _tile(n)
    w = case.build(n, T)
    assert tc.classify(w) == case.cls
    bad = np.flatnonzero(~np.isfinite(w))
    if case.first_bad is None:
        assert bad.size == 0
    else:
        assert bad.size and bad[0] == case.first_bad(n, T)
    if case.name == "inf_first_tile":
        assert bad[0] < T
    if case.name == "inf_tile_edge" and T < n:
        assert bad[0] == T
    if case.name == "inf_last_tile":
        assert bad[0] >= (tc.pf3_shape(n, SMS)[0] - 1) * T
    if case.cls == "S_inf":
        c = np.add.accumulate(tc.normalised(w))
        assert np.isnan(c[bad[0]]) and not np.any(np.isnan(c[:bad[0]])), "the CDF turns NaN at the first inf"
    if case.cls == "S_overflow":
        assert np.all(tc.normalised(w) == 0.0)


def _indices(oracle, w, mode, search):
    did, _neff, idx, _p, _e, _c = tc.oracle_tail(w, mode, 1.0, SEED, search=search)
    return idx if did else np.zeros(0, dtype=np.uint32)


@pytest.mark.parametrize("mode", [0, 1], ids=["pf", "mcl"])
@pytest.mark.parametrize("case", [c for c in tc.TAIL_CASES if c.cls == "S_inf"], ids=lambda c: c.name)
def test_linear_scan_and_lower_bound_disagree_on_nan_cdfs(oracle, case, mode):
    n = 4099
    w = case.build(n, _tile(n))
    lin, lb = _indices(oracle, w, mode, 0), _indices(oracle, w, mode, 1)
    assert lin.size == n
    if mode == 1 and case.name == "inf_last_slot":
        # the forced last entry replaces the only NaN: the CDF is monotone and both searches agree
        assert tc.monotone_cdf(w, mode) and np.array_equal(lin, lb)
        return
    assert not tc.monotone_cdf(w, mode)
    if case.name == "all_inf":
        assert np.all(lin == (n - 1 if mode == 1 else 0))
        if mode == 0:
            # every entry is NaN: the first one is also PF's fallback, so here the lower bound happens to agree
            assert np.array_equal(lin, lb)
            return
    assert not np.array_equal(lin, lb), "the lower bound reproduces the linear scan: the case proves nothing"


def _all_cases(n):
    out = [(c.name, c.build(n, _tile(n))) for c in tc.TAIL_CASES]
    for c in wc.CASES:
        out.append((c.name, c.build(n, SEED, 0, L=_ORACLE[0], family="pf")))
    return out


_ORACLE = [None]


@pytest.mark.parametrize("n", [1000, 4099])
@pytest.mark.parametrize("mode", [0, 1], ids=["pf", "mcl"])
def test_running_max_search_is_the_linear_scan(oracle, n, mode):
    _ORACLE[0] = oracle
    for name, w in _all_cases(n):
        lin, rm = _indices(oracle, w, mode, 0), _indices(oracle, w, mode, "runmax")
        assert np.array_equal(lin, rm), f"{name}: {int((lin != rm).sum())} ancestors differ"


@pytest.mark.parametrize("n", [256, 16384, 1 << 18])
@pytest.mark.parametrize("case", [c for c in wc.CASES if c.name.startswith("border")], ids=lambda c: c.name)
def test_border_thresholds(oracle, n, case):
    """threshold = nth / n is exact at n = 2^k, so the gate compares N_eff with nth itself"""
    w = case.build(n, SEED, 0, L=oracle, family="pf")
    nth = case.nth(n, w)
    thr = nth / n
    assert thr * n == nth and 0.0 < thr <= 1.0
    did, neff, *_ = tc.oracle_tail(w, 0, thr, SEED)
    assert neff == wc.exact_neff(w)
    want = {"border_eq": neff == nth, "border_up": neff < nth and math.nextafter(neff, math.inf) == nth,
            "border_down": neff > nth and math.nextafter(neff, -math.inf) == nth}[case.name]
    assert want
    assert did == (neff < nth)
