"""Raw weight vectors for the PF / MCL step tail (normalise, N_eff gate, CDF, search, clone, moments) and its oracle.

The fused tail (pf3_post_kernel) runs one tile of NT x K weights per CTA; pf3_shape() restates how pf3_setup picks the tile
count and K for a particle count.  The cases below add to _weight_cases.CASES what a likelihood can produce that the catalogue
does not: +inf among zeros (S = inf, so every normalised weight is NaN or 0 and the CDF turns NaN at the first inf), inf with
NaN (S = NaN, the uniform fallback), finite weights whose sum overflows, and a subnormal S.  Each case names the class it is
built to hit (test_pf_tail_cases_oracle.py checks that it does).  Pure numpy; the oracle is only loaded to run the tail."""
import ctypes as C
import math
import os
import subprocess
import tempfile
from dataclasses import dataclass
from typing import Callable

import numpy as np

import _assoc_oracle
import _oracle
import _weight_cases as wc
from _oracle import OraclePF

NT = 256
FS3_MAX_TILES = 160


def pf3_shape(n, sms):
    """(tiles, K) of the fused tail at n particles on a device with `sms` multiprocessors (pf3_setup)"""
    tiles = min(min(sms, FS3_MAX_TILES), (n + NT - 1) // NT)
    k = (n + tiles * NT - 1) // (tiles * NT)
    return (n + NT * k - 1) // (NT * k), k


@dataclass(frozen=True)
class TailCase:
    name: str
    build: Callable                  # (n, T) -> w_raw; T = NT x K, the tile length at n
    cls: str                         # "S_inf", "S_nan", "S_overflow", "S_subnormal"
    first_bad: Callable = None       # (n, T) -> the slot of the first non-finite weight (None: there is none)


def _inf_at(pos):
    def build(n, T):
        w = np.zeros(n)
        p = pos(n, T)
        w[p] = math.inf
        if p + 5 < n:
            w[p + 5] = math.inf                  # a second inf after the first: the CDF stays NaN
        if p > 3:
            w[p - 3] = 0.25                      # a finite weight in front (normalised to 0 by S = inf)
        return w
    return build


def _first_tile(n, T):
    return min(5, n - 1)


def _tile_edge(n, T):
    return T if T < n else n // 2


def _last_tile(n, T):
    return n - 2


def _last_slot(n, T):
    return n - 1


def _inf_nan(n, T):
    w = wc._uniform_rand(n, 1, 21)
    w[n // 3] = math.inf
    w[(2 * n) // 3] = math.nan
    return w


def _overflow(n, T):
    """finite weights, the running sum overflows at slot n / 2 (every prefix after it is inf)"""
    w = np.full(n, 1.0)
    w[n // 2:] = 1.5e308
    w[-1] = 1.7e308
    return w


def _subnormal(n, T):
    """S = sum of small multiples of 2^-1074 (exact, subnormal): normalisation divides by a subnormal"""
    return (1.0 + (np.arange(n) % 7)) * 2.0 ** -1074


TAIL_CASES = [
    TailCase("inf_first_tile", _inf_at(_first_tile), "S_inf", _first_tile),
    TailCase("inf_tile_edge", _inf_at(_tile_edge), "S_inf", _tile_edge),
    TailCase("inf_last_tile", _inf_at(_last_tile), "S_inf", _last_tile),
    TailCase("inf_last_slot", _inf_at(_last_slot), "S_inf", _last_slot),
    TailCase("all_inf", lambda n, T: np.full(n, math.inf), "S_inf", lambda n, T: 0),
    TailCase("inf_and_nan", _inf_nan, "S_nan", lambda n, T: n // 3),
    TailCase("sum_overflow", _overflow, "S_overflow"),
    TailCase("S_subnormal", _subnormal, "S_subnormal"),
]
TAIL_BY_NAME = {c.name: c for c in TAIL_CASES}


def classify(w_raw):
    """the class of S = sum w_raw (sequential)"""
    S = wc.seq_sum(w_raw)
    if math.isnan(S):
        return "S_nan"
    if math.isinf(S):
        return "S_overflow" if np.all(np.isfinite(w_raw)) else "S_inf"
    if 0.0 < S < 2.2250738585072014e-308:
        return "S_subnormal"
    return "finite"


def normalised(w_raw):
    """normalize_weights (pf.rs:426-439): w / S with the sequential S, or 1 / n when !(S > 0)"""
    w = np.asarray(w_raw, dtype=np.float64)
    S = wc.seq_sum(w)
    with np.errstate(all="ignore"):
        return w / S if S > 0.0 else np.full(w.size, 1.0 / w.size)


def monotone_cdf(w_raw, mode):
    """the reference's cumulative weights (MCL: last := 1) are NaN-free and non-decreasing: a lower bound finds its index"""
    c = np.add.accumulate(normalised(w_raw))
    if mode == 1:
        c[-1] = 1.0
    return not np.any(np.isnan(c)) and bool(np.all(np.diff(c) >= 0.0))


def cloud(w_raw):
    """poses the tail clones (distinct per slot, finite) with the raw weights in the weight column"""
    n = len(w_raw)
    a = np.empty((n, 5))
    a[:, 0] = np.arange(n) * 0.5 + 3.0
    a[:, 1] = -np.arange(n) * 0.25 - 2.0
    a[:, 2] = np.linspace(-3.0, 3.0, n)
    a[:, 3] = 1.0
    a[:, 4] = w_raw
    return a


SRC = os.path.join(_oracle.ROOT, "tests", "host", "pf_tail_oracle.c")
_LIB = []


def load():
    """tests/host/pf_tail_oracle.c (oracle/pf_oracle.c and the tail's two entry points), built once per process in a
    temporary directory"""
    if not _LIB:
        out = os.path.join(tempfile.mkdtemp(prefix="pf_tail_oracle_"), "libpf_tail_oracle.so")
        subprocess.run(["/usr/bin/gcc"] + _assoc_oracle.CFLAGS + ["-shared", "-o", out, SRC, "-lm"], check=True)
        L = C.CDLL(out)
        vp = C.c_void_p
        L.orc_pf_new.restype = vp
        L.orc_pf_new.argtypes = [C.POINTER(_oracle.PfConfig), C.c_uint64]
        L.orc_pf_neff.restype = C.c_double
        L.orc_pf_count.restype = L.orc_pf_last_indices.restype = C.c_size_t
        for name, args in (("orc_pf_free", [vp]), ("orc_pf_count", [vp]), ("orc_pf_set_particles", [vp, _oracle.c_dp, C.c_size_t]),
                           ("orc_pf_get_particles", [vp, _oracle.c_dp]), ("orc_pf_resample", [vp]), ("orc_pf_neff", [vp]),
                           ("orc_pf_estimate", [vp, _oracle.c_dp, _oracle.c_dp]),
                           ("orc_pf_last_indices", [vp, _oracle.c_u32p, C.c_size_t]), ("orc_pf_set_fast_search", [vp, C.c_int]),
                           ("orc_pf_set_threads", [vp, C.c_int]), ("orc_tail_normalize", [vp]), ("orc_tail_resample_runmax", [vp])):
            getattr(L, name).argtypes = args
        _LIB.append(L)
    return _LIB[0]


def search_mode(w_raw, mode, linear_max=16384):
    """the oracle's search: 1 (lower bound) on a monotone CDF; else 0 (the linear scan as written) up to linear_max particles,
    and beyond that "runmax" (the lower bound on the running maximum, pinned to the linear scan by test_pf_tail_cases_oracle.py)"""
    if monotone_cdf(w_raw, mode):
        return 1
    return 0 if len(w_raw) <= linear_max else "runmax"


def oracle_tail(w_raw, mode, threshold, seed, search=None):
    """the oracle's step tail on w_raw: (gate, N_eff after normalisation, indices or None, particles, estimate, covariance)"""
    n = len(w_raw)
    L = load()
    o = OraclePF(L, n, threshold=threshold, seed=seed, mode=mode, max_particles=n)
    search = search_mode(w_raw, mode) if search is None else search
    o.L.orc_pf_set_threads(o.h, os.cpu_count() or 1)
    o.set_particles(cloud(w_raw))
    L.orc_tail_normalize(o.h)
    neff = o.neff()
    if search == "runmax":
        rc = L.orc_tail_resample_runmax(o.h)
        assert rc >= 0
        did = rc == 1
    else:
        o.L.orc_pf_set_fast_search(o.h, search)
        did = bool(o.resample())
    est, cov = o.estimate()
    return did, neff, (o.last_indices() if did else None), o.particles(), est, cov


# particle counts of the GPU test; their tail shapes on an H100 SXM (132 multiprocessors) in the comments
SIZES = {
    "one_tile": 256,          # 1 tile, K = 1
    "k1_tiles": 16384,        # 64 tiles, K = 1
    "k3_partial": 100003,     # 131 tiles, K = 3, the last tile holds 163 weights
    "2^18": 1 << 18,          # 128 tiles, K = 8
}
