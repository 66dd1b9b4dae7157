"""Adversarial raw weight vectors for the resample path (normalise, N_eff gate, CDF, index search, best particle).

Each case builds w_raw for a particle count n from (n, seed, resamples so far) and names the N_eff threshold it uses and the
path of the post step it is meant to drive:
  "cert"     the certified CDF fl(P_j / S) (n = 2^p <= 2^16; other n take the exact sums)
  "refused"  a comb value coincides with a CDF value: the certificate refuses and the exact S2 / CDF sums run (n = 2^p)
  "exact"    the exact sums with dirty values (binade crossings, ties to even)
  "serial"   more than FS3_ENT_CAP = 512 dirty values: the sums take the one-thread walk
  "border"   N_eff within the shortcut's slack of NTH, or S outside [1e-120, 1e120]: the exact sequential N_eff decides
  "none"     no resample (NTH = 0): only normalisation and the best particle
The comb cases need the resample draw, so they are built for one filter family: "fs" (FastSLAM: r_t = r_0 + t / n, one
U[0, 1/n) draw) or "pf" (PF / MCL: one U[0, 1) draw per slot).  Pure numpy; the oracle is only loaded to draw uniforms."""
import math
from dataclasses import dataclass
from typing import Callable

import numpy as np

U53 = 2.0 ** -53
PFC_STREAM_PF_RESAMPLE = 1
PFC_STREAM_FS_RESAMPLE = 3
TILE_EDGES = (256, 512, 2048)        # post-kernel tile lengths of the shapes the GPU tests run (NT x K)


@dataclass(frozen=True)
class Case:
    name: str
    build: Callable                  # (n, seed, resamples_so_far, L=None, family="fs") -> w_raw
    nth: Callable                    # (n, w_raw) -> NTH for FastSLAM
    path: str
    finite: bool = True              # finite and non-negative (run at every shape, best particle compared)
    small: bool = False              # one thread walks every value: keep to small n
    min_n: int = 1


def _rng(n, seed, salt):
    return np.random.default_rng([seed, n, salt])


def seq_sum(w):
    """the reference's sequential f64 sum"""
    return float(np.add.accumulate(np.asarray(w, dtype=np.float64))[-1]) if len(w) else 0.0


def exact_neff(w_raw):
    """compute_neff after normalize_weights (fs1.rs:186-203), sequentially: 1 / sum fl(w_i / S)^2"""
    w = np.asarray(w_raw, dtype=np.float64)
    S = seq_sum(w)
    if S > 0.0:
        w = w / S
    q = seq_sum(w * w)
    return 1.0 / q if q > 0.0 else 0.0


def fs_comb(L, n, seed, resamples):
    """FastSLAM's comb r_t = r_0 + t / n, accumulated sequentially as fs1.rs:219-230 does"""
    inv = 1.0 / n
    r0 = L.orc_uniform52(seed, PFC_STREAM_FS_RESAMPLE, resamples, 0) * (inv - 0.0) + 0.0
    r = np.empty(n)
    r[0] = r0
    for t in range(1, n):
        r[t] = r[t - 1] + inv
    return r


def pf_draws(L, n, seed, resamples):
    """PF / MCL's per-slot draws r_t (pf.rs:456, mcl.rs:344)"""
    return np.array([L.orc_uniform53(seed, PFC_STREAM_PF_RESAMPLE, resamples, t) for t in range(n)])


def comb_targets(n):
    """slots whose CDF value is put on (or one ulp from) a draw: the first tile, both sides of every tile edge, the last tile"""
    js = {1, 2, 3, n - 3, n - 2}
    for e in TILE_EDGES:
        if e + 1 < n - 3:
            js |= {e - 1, e}
    return sorted(j for j in js if 0 < j < n - 1)


def comb_cdf(n, r, delta, pf=False):
    """A CDF of multiples of 2^-53 in [1/2, 1] with c_{n-1} = 1, and c_j = r_t + delta ulp at the comb_targets slots, r_t the
    draw nearest the slot's base value.  Every weight c_j - c_{j-1} and every prefix is exact, so S = S2 = 1."""
    c = np.round((0.5 + 0.5 * (np.arange(n) + 1.0) / n) / U53) * U53
    c[-1] = 1.0
    order = np.sort(r) if pf else r
    lo, hi = np.full(n, -np.inf), np.full(n, np.inf)
    last = -1
    for j in comb_targets(n):
        k = int(np.clip(np.searchsorted(order, c[j]), 0, n - 1))
        if k > 0 and abs(order[k - 1] - c[j]) <= abs(order[k] - c[j]):
            k -= 1
        k = max(k, last + 1)                   # each draw serves one slot, in increasing order
        if k >= n or not 0.5 <= order[k] < 1.0 or order[k] + delta * U53 >= 1.0:
            continue
        last = k
        lo[j] = hi[j] = float(order[k]) + delta * U53
    # every other value is clamped between the targets around it: c stays non-decreasing, the targets keep their values
    c = np.minimum(np.maximum(c, np.maximum.accumulate(lo)), np.minimum.accumulate(hi[::-1])[::-1])
    assert np.all(np.diff(c) >= 0.0) and c[-1] == 1.0
    w = np.diff(np.concatenate([[0.0], c]))
    return w


def _comb(delta):
    def build(n, seed, resamples, L=None, family="fs"):
        r = fs_comb(L, n, seed, resamples) if family == "fs" else pf_draws(L, n, seed, resamples)
        return comb_cdf(n, r, delta, pf=family != "fs")
    return build


def _scaled_to(target):
    """near-uniform weights whose sequential sum is exactly `target`: A + (n-1) y, y a power of two, every partial sum exact"""
    def build(n, seed, resamples, L=None, family="fs"):
        y = math.ldexp(1.0, math.frexp(target)[1] - 53 + 2)        # 4 ulp of target's binade
        a = target - (n - 1) * y
        w = np.full(n, y)
        w[0] = a
        return w
    return build


def _border(direction):
    def build(n, seed, resamples, L=None, family="fs"):
        return np.exp(_rng(n, seed, 11).normal(0.0, 1.0, n))
    def nth(n, w):
        e = exact_neff(w)
        return e if direction == 0 else float(np.nextafter(e, math.inf if direction > 0 else -math.inf))
    return build, nth


def _single(pos):
    def build(n, seed, resamples, L=None, family="fs"):
        w = np.zeros(n)
        w[{"first": 0, "mid": n // 2, "last": n - 1}[pos]] = 0.7
        return w
    return build


def _lognormal(sigma):
    def build(n, seed, resamples, L=None, family="fs"):
        z = _rng(n, seed, int(sigma)).normal(0.0, sigma, n)
        return np.exp(z - z.max())
    return build


def _uniform_rand(n, seed, salt):
    return _rng(n, seed, salt).uniform(0.1, 1.0, n)


def _leading_zeros(n, seed, resamples, L=None, family="fs"):
    w = _uniform_rand(n, seed, 3)
    w[: n // 2] = 0.0
    return w


def _trailing_zeros(n, seed, resamples, L=None, family="fs"):
    w = _uniform_rand(n, seed, 4)
    w[n // 2:] = 0.0
    return w


def _neg_zero(n, seed, resamples, L=None, family="fs"):
    w = _uniform_rand(n, seed, 5)
    w[::3] = -0.0
    return w


def _serial(n, seed, resamples, L=None, family="fs"):
    """w_i = 2^(0.75 (i mod 1200) - 450): the running sum enters a new binade every one or two values (> 512 dirty values)"""
    i = np.arange(n)
    return np.exp2(0.75 * (i % 1200) - 450.0)


def _best_tiles(n, seed, resamples, L=None, family="fs"):
    w = _uniform_rand(n, seed, 6)
    w[1] = w[n - 2] = 2.0
    return w


def _best_edges(n, seed, resamples, L=None, family="fs"):
    w = _uniform_rand(n, seed, 7)
    for e in TILE_EDGES:
        if e < n:
            w[e - 1] = w[e] = 2.0
    return w


def _one_inf(n, seed, resamples, L=None, family="fs"):
    w = _uniform_rand(n, seed, 8)
    w[n // 3] = math.inf
    return w


def _one_nan(n, seed, resamples, L=None, family="fs"):
    w = _uniform_rand(n, seed, 9)
    w[(3 * n) // 4] = math.nan
    return w


def _negative(n, seed, resamples, L=None, family="fs"):
    """S > 0 with every seventh weight negative: the CDF goes down at those slots"""
    w = _uniform_rand(n, seed, 10)
    w[3::7] *= -1.5
    return w


def best_expected(w):
    """get_best_particle fs1.rs:269-274: the LAST maximum (w_i >= w_best)"""
    b = 0
    for i in range(1, len(w)):
        if w[i] >= w[b]:
            b = i
    return b


_RES = lambda n, w: n + 1.0          # noqa: E731  (N_eff <= n after normalisation: the gate opens)
_HALF = lambda n, w: n / 2.0         # noqa: E731
_ZERO = lambda n, w: 0.0             # noqa: E731
_bd0, _bn0 = _border(0)
_bdu, _bnu = _border(1)
_bdd, _bnd = _border(-1)

CASES = [
    Case("ties", lambda n, s, r, L=None, family="fs": np.concatenate([[1.0], np.full(n - 1, 2.0 ** -54)]), _RES, "exact"),
    Case("crawl", lambda n, s, r, L=None, family="fs": np.concatenate([[1.0 - 2.0 ** -40], np.full(n - 1, 2.0 ** -60)]), _RES, "exact"),
    Case("uniform", lambda n, s, r, L=None, family="fs": np.ones(n), _RES, "cert"),
    Case("uniform_tenth", lambda n, s, r, L=None, family="fs": np.full(n, 0.1), _RES, "exact"),
    Case("lognormal12", _lognormal(12.0), _RES, "cert"),
    Case("collapse40", _lognormal(40.0), _RES, "exact"),
    Case("leading_zeros", _leading_zeros, _RES, "exact"),
    Case("trailing_zeros", _trailing_zeros, _RES, "exact"),
    Case("single_first", _single("first"), _RES, "exact"),
    Case("single_mid", _single("mid"), _RES, "exact"),
    Case("single_last", _single("last"), _RES, "exact"),
    Case("neg_zero", _neg_zero, _RES, "exact"),
    Case("subnormal", lambda n, s, r, L=None, family="fs": _uniform_rand(n, s, 12) * 1e-310, _HALF, "border"),
    Case("huge", lambda n, s, r, L=None, family="fs": _uniform_rand(n, s, 13) * 1e200, _HALF, "border"),
    Case("S_lo_in", _scaled_to(1e-120), _RES, "cert"),
    Case("S_lo_out", _scaled_to(float(np.nextafter(1e-120, 0.0))), _RES, "border"),
    Case("S_hi_in", _scaled_to(1e120), _RES, "cert"),
    Case("S_hi_out", _scaled_to(float(np.nextafter(1e120, math.inf))), _RES, "border"),
    Case("serial_walk", _serial, _RES, "serial", small=True),
    Case("border_eq", _bd0, _bn0, "border"),
    Case("border_up", _bdu, _bnu, "border"),
    Case("border_down", _bdd, _bnd, "border"),
    Case("comb_eq", _comb(0), _RES, "refused", min_n=16),
    Case("comb_lo", _comb(-1), _RES, "refused", min_n=16),
    Case("comb_hi", _comb(1), _RES, "refused", min_n=16),
    Case("best_tiles", _best_tiles, _ZERO, "none"),
    Case("best_edges", _best_edges, _ZERO, "none"),
    Case("all_minus_two", lambda n, s, r, L=None, family="fs": np.full(n, -2.0), _ZERO, "none", finite=False),
    Case("all_minus_inf", lambda n, s, r, L=None, family="fs": np.full(n, -math.inf), _ZERO, "none", finite=False),
    Case("one_inf", _one_inf, _RES, "exact", finite=False),
    Case("one_nan", _one_nan, _RES, "exact", finite=False),
    Case("negative", _negative, _RES, "exact", finite=False),
]
BY_NAME = {c.name: c for c in CASES}
# no best particle in the reference for these (max_by(partial_cmp).unwrap() panics on NaN; inf / NaN weights make one)
NO_BEST = {"one_inf", "one_nan"}
