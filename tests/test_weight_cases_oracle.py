"""The adversarial weight catalogue (_weight_cases.py) against the CPU oracle: every case has the property it claims, so the
GPU tests that drive it through the post kernel really reach their edge."""
import math
from fractions import Fraction

import numpy as np
import pytest

import _weight_cases as wc
from _oracle import OracleFS, OraclePF

SEED = 17
M = 4


def _fs_step(oracle, n, w, nth):
    o = OracleFS(oracle, n, M, seed=SEED, q00=0.0, q11=0.0, nth=nth)
    p = np.zeros((n, 4))
    p[:, 0] = w                                # rows are (w, x, y, yaw)
    p[:, 1] = np.arange(n) * 0.5
    o.set_state(p)
    did = bool(o.step([0.0, 0.0], []))
    return o, did


def _binade_entries(w):
    c = np.add.accumulate(np.asarray(w, dtype=np.float64))
    e = np.frexp(c)[1]
    return int(np.count_nonzero(np.diff(e) != 0))


@pytest.mark.parametrize("n", [1000, 1024, 4096])
@pytest.mark.parametrize("case", wc.CASES, ids=[c.name for c in wc.CASES])
def test_case_drives_its_path(oracle, case, n):
    w = case.build(n, SEED, 0, L=oracle, family="fs")
    assert w.shape == (n,) and w.dtype == np.float64
    nth = case.nth(n, w)
    o, did = _fs_step(oracle, n, w, nth)
    S = wc.seq_sum(w)
    opens = case.path not in ("none",) and case.name not in ("border_eq", "border_down", "subnormal", "huge")
    assert did == opens, f"{case.name}: the oracle {'did not resample' if opens else 'resampled'}"
    if case.finite:
        assert np.all(w >= 0.0)
        assert o.best() == wc.best_expected(w / S if S > 0 else w) or did
    if case.path == "border" and case.name.startswith("border"):
        neff = wc.exact_neff(w)
        assert o.last_neff() == neff, "the sequential N_eff of the catalogue is the oracle's"
        slack = 16.0 * (n + 64) * 2.0 ** -52
        assert abs(neff - nth) <= slack * max(abs(nth), abs(neff))
    if case.name == "subnormal":
        assert 0.0 < S < 1e-120 and np.all(w < 2.2250738585072014e-308)
    if case.name == "huge":
        assert S > 1e120 and np.all(np.isinf(w * w))
    if case.name.startswith("S_"):
        want = {"S_lo_in": 1e-120, "S_hi_in": 1e120, "S_lo_out": float(np.nextafter(1e-120, 0.0)),
                "S_hi_out": float(np.nextafter(1e120, math.inf))}[case.name]
        assert S == want
        assert sum(Fraction(x) for x in w) == Fraction(want), "every partial sum is exact"
    if case.name == "serial_walk":
        assert _binade_entries(w) > 512
    if case.name == "ties":
        assert S == 1.0 and sum(Fraction(x) for x in w) > 1, "every add is a tie to even"
    if case.name == "crawl":
        assert S == 1.0 - 2.0 ** -40 and sum(Fraction(x) for x in w) > Fraction(S)
    if case.name == "neg_zero":
        assert np.any(np.signbit(w) & (w == 0.0))
    if case.name == "all_minus_two":
        assert o.best() == n - 1
    if case.name == "all_minus_inf":
        assert o.best() == n - 1
    if case.name == "best_tiles":
        assert o.best() == n - 2
    if case.name == "best_edges":
        assert o.best() == max(e for e in wc.TILE_EDGES if e < n)
    if case.name == "negative":
        c = np.add.accumulate(w / S)
        assert S > 0.0 and np.any(np.diff(c) < 0.0)
    if case.name == "one_inf":
        assert S == math.inf
    if case.name == "one_nan":
        assert math.isnan(S) and o.last_neff() == 0.0


@pytest.mark.parametrize("n", [1000, 1024, 4096])
@pytest.mark.parametrize("delta", [-1, 0, 1])
def test_fs_comb_coincidences_are_exact(oracle, n, delta):
    case = wc.BY_NAME[{-1: "comb_lo", 0: "comb_eq", 1: "comb_hi"}[delta]]
    w = case.build(n, SEED, 0, L=oracle, family="fs")
    c = np.add.accumulate(w)
    assert wc.seq_sum(w) == 1.0 and c[-1] == 1.0
    assert np.all(c * 2.0 ** 53 == np.round(c * 2.0 ** 53)), "every CDF value is a multiple of 2^-53"
    assert all(Fraction(float(x)) == sum(Fraction(float(v)) for v in w[: j + 1]) for j, x in list(enumerate(c))[::97])
    r = wc.fs_comb(oracle, n, SEED, 0)
    hit = np.isin(c - delta * wc.U53, r) & (c >= 0.5) & (c < 1.0)
    js = set(np.flatnonzero(hit).tolist())
    assert any(j < 256 for j in js), "no coincidence in the first tile"
    assert any(j >= n - 256 for j in js), "no coincidence in the last tile"
    assert {255, 256} <= js, "no coincidence on both sides of a tile edge"
    # the oracle resamples on it (S = S2 = 1: the CDF it searches is c)
    o, did = _fs_step(oracle, n, w, n + 1.0)
    assert did
    idx = o.last_indices()
    want = np.minimum(np.searchsorted(c, r, side="left"), n - 1)
    assert np.array_equal(idx, want)


@pytest.mark.parametrize("mode", [0, 1])
@pytest.mark.parametrize("n", [1000, 4099])
def test_pf_comb_coincidences_are_exact(oracle, n, mode):
    case = wc.BY_NAME["comb_eq"]
    w = case.build(n, SEED, 0, L=oracle, family="pf")
    c = np.add.accumulate(w)
    r = wc.pf_draws(oracle, n, SEED, 0)
    js = np.flatnonzero(np.isin(c, r))
    assert js.size >= 5 and js.min() < 256 and js.max() >= n - 256
    o = OraclePF(oracle, n, threshold=1.0, seed=SEED, mode=mode, max_particles=n)
    o.L.orc_pf_set_fast_search(o.h, 0)
    a = np.zeros((n, 5))
    a[:, 0] = np.arange(n)
    a[:, 4] = w
    o.set_particles(a)
    assert o.resample()
    idx = o.last_indices()
    hits = np.isin(r, c)
    assert np.array_equal(idx[hits], np.searchsorted(c, r[hits], side="left")), "a draw equal to c_i picks slot i"


def test_negative_and_nan_cdfs_are_not_monotone_searches(oracle):
    """the reference's index rules on a CDF that goes down (negative weights) or turns NaN: FastSLAM's carried j is the first j
    with c_j >= r (NaN stops it), PF's linear scan the first i with r <= c_i (NaN never matches) -- neither is a bisection"""
    n = 1000
    w = wc.BY_NAME["negative"].build(n, SEED, 0)
    o, did = _fs_step(oracle, n, w, n + 1.0)
    assert did
    w1 = w / wc.seq_sum(w)                     # normalize_weights in the step, then again in resample (fs1.rs:207)
    c = np.add.accumulate(w1 / wc.seq_sum(w1))
    r = wc.fs_comb(oracle, n, SEED, 0)
    first = np.array([min(int(np.argmax(c >= x)) if np.any(c >= x) else n - 1, n - 1) for x in r])
    assert np.array_equal(o.last_indices(), first)
    bisect = np.minimum(np.searchsorted(c, r, side="left"), n - 1)
    assert not np.array_equal(first, bisect), "the case would not tell a bisection from the reference's walk"
