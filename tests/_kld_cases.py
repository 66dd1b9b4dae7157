"""Adversarial particle clouds for the KLD-adaptive MCL resample (resample_adaptive, mcl.rs:322-365; pf_kld.cuh on the device).

Each case is a cloud of exactly n_min particles (rows x, y, yaw, v, w; the filter's count when it is created), the filter's
(n_min, n_max, eps, z) and its seed.  The first resample of a fresh filter draws r_t = U53(seed, PF_RESAMPLE stream, call 0, t),
so the stopping length is fixed by the case alone.  `expect` is the length the case was built to hit; the tests assert it
against the oracle, so a case cannot drift off its target unnoticed.

  stop_*      the stop lands at 1023, 1024, 1025 (the first 1024-draw chunk of the stop kernel and the one after it), 2048,
              2049, and one draw before the end of a partial last chunk.  Clouds of distinct bins; (seed, eps) found offline
              with the plain-Python rule (search_eps) on the real draws.
  zcarry_*    z = 60: kld_required(k) FALLS with k, so the running maximum `required` is set by k = 2 in the first chunk and
              decides a stop one or two chunks later (eps solved so that kld_required(2) is the target)
  never_*     kld_required(2) far above n_max: the generation runs to n_max (1023, 1024, 1025, 3 * 1024 + 7, 2^20 + 3, with
              small n_min and with n_min = n_max - 1).  n_max = 2 with n_min = 1 stops after one draw: k = 1 there, and
              kld_required(1) = n_min = 1.
  quantiser_* bin keys at the edges of `floor(v / bin) as i32`: saturation at |x|, |y| >= 2^30 m, NaN (key 0, the bin of
              [0, 0.5)), +-inf, -0.0, values on and one ulp off bin edges, yaw far outside [-pi, pi)
  hash_*      bin keys whose pf_bin_hash shares a slot modulo the handle's table size: 64 keys that differ only in yaw and 64
              others with home slot tcap - 1 (the probe chain wraps past the end of the table), 64 more with home slot 5
  distinct_*  2^16 particles in distinct bins, n_max = 2^18: the stop kernel walks 147 and 256 chunks
  w_*         weights: all mass on one particle, zero weights at both ends with a sum below 1 (draws above it fall to the last,
              zero-weight particle), CDF values equal to draws with zero weights after them (ties), -0.0, and weights the
              reference's linear scan handles differently from a lower bound: negative, NaN, inf
"""
import bisect
import math
from dataclasses import dataclass
from typing import Callable, Optional

import numpy as np

X_BIN, Y_BIN, YAW_BIN = 0.5, 0.5, 15.0 * math.pi / 180.0      # mcl.rs:26-28
PFC_STREAM_PF_RESAMPLE = 1
U53 = 2.0 ** -53
H1, H2, H3 = 0x9E3779B97F4A7C15, 0xC2B2AE3D27D4EB4F, 0x165667B19E3779F9


@dataclass(frozen=True)
class Case:
    name: str
    n_min: int
    n_max: int
    eps: float
    z: float
    seed: int
    build: Callable                  # (case, L) -> (n_min, 5) cloud; L: the oracle library (for its uniforms)
    expect: Optional[int] = None     # the stopping length the case was built to hit
    big: bool = False                # too large for the reference's linear scan: tests use an equivalent lower bound

    @property
    def monotone(self):
        """the cloud's weights are finite and non-negative, so its CDF never goes down (a lower bound equals the linear scan)"""
        return not self.name.startswith(("w_negative", "w_nan"))

    def cloud(self, L=None):
        a = np.ascontiguousarray(self.build(self, L), dtype=np.float64)
        assert a.shape == (self.n_min, 5), (self.name, a.shape)
        return a


# ---- the rule, restated (mcl.rs:343-355, 367-385) --------------------------------------------------------------------------
def floor_i32(v):
    """`v.floor() as i32`"""
    if v != v:
        return 0
    if v >= 2147483647.0:
        return 2147483647
    if v <= -2147483648.0:
        return -2147483648
    return int(math.floor(v))


def key(x, y, yaw):
    return floor_i32(x / X_BIN), floor_i32(y / Y_BIN), floor_i32(yaw / YAW_BIN)


def draws(L, seed, n, call=0):
    return np.array([L.orc_uniform53(seed, PFC_STREAM_PF_RESAMPLE, call, t) for t in range(n)])


def kld_required(k, n_min, n_max, eps, z):
    if k <= 1:
        return n_min
    km1 = float(k - 1)
    term = 1.0 - 2.0 / (9.0 * km1) + z * math.sqrt(2.0 / (9.0 * km1))
    nn = (km1 / (2.0 * eps)) * (term * term * term)
    v = (math.ceil(nn) if nn < math.inf else n_max) if nn > 0 else 0
    return max(n_min, min(n_max, v))


def bins_after_each_draw(cloud, r):
    """k after each draw, for a cloud with a non-decreasing CDF"""
    cum = list(np.add.accumulate(cloud[:, 4]))
    cum[-1] = 1.0
    n = len(cum)
    seen, ks = set(), []
    for x in r:
        i = bisect.bisect_left(cum, x, 0, n - 1)
        seen.add(key(*cloud[i, :3]))
        ks.append(len(seen))
    return ks


def stop_length(ks, n_min, n_max, eps, z):
    required = n_min
    memo = {}
    for t, k in enumerate(ks):
        if k not in memo:
            memo[k] = kld_required(k, n_min, n_max, eps, z)
        required = max(required, memo[k])
        if t + 1 >= n_min and t + 1 >= required:
            return t + 1
    return n_max


def search_eps(L, cloud, seed, n_max, target, z=2.326):
    """the offline search behind the stop_* cases: an eps whose stopping length is `target` (None if it skips the target)"""
    ks = bins_after_each_draw(cloud, draws(L, seed, n_max))
    n_min = cloud.shape[0]
    lo, hi = 1e-6, 10.0
    if stop_length(ks, n_min, n_max, lo, z) < target or stop_length(ks, n_min, n_max, hi, z) > target:
        return None
    for _ in range(200):
        mid = math.sqrt(lo * hi)
        s = stop_length(ks, n_min, n_max, mid, z)
        if s == target:
            return mid
        lo, hi = (mid, hi) if s > target else (lo, mid)
    return None


# ---- the device's bin hash set (pf_kld.cuh) ---------------------------------------------------------------------------------
def table_size(n_max):
    """PfKld::tcap: the power of two >= 2 n_max + 16, at least 64"""
    t = 64
    while t < 2 * n_max + 16:
        t <<= 1
    return t


def bin_hash(a, b, c):
    """pf_bin_hash, vectorised"""
    u = lambda v: np.asarray(v, dtype=np.int64).astype(np.uint32).astype(np.uint64)   # noqa: E731
    h = (u(a) * np.uint64(H1)) ^ (u(b) * np.uint64(H2)) ^ (u(c) * np.uint64(H3))
    return (h >> np.uint64(17)).astype(np.uint32)


def pose_of(a, b, c):
    """a pose in the middle of bin (a, b, c)"""
    p = (X_BIN * a + 0.25, Y_BIN * b + 0.25, YAW_BIN * (c + 0.5))
    assert key(*p) == (a, b, c), (a, b, c)
    return p


def colliding_keys(tcap, slot, count, rng, vary="all"):
    """`count` distinct keys with pf_bin_hash(key) & (tcap - 1) == slot"""
    out = []
    while len(out) < count:
        m = 1 << 20
        c = rng.integers(-(1 << 20), 1 << 20, m)
        if vary == "yaw":
            a, b = np.full(m, 1234), np.full(m, -77)
        else:
            a, b = rng.integers(-(1 << 20), 1 << 20, m), rng.integers(-(1 << 20), 1 << 20, m)
        hit = np.flatnonzero((bin_hash(a, b, c) & np.uint32(tcap - 1)) == slot)
        out += [(int(a[i]), int(b[i]), int(c[i])) for i in hit]
        out = list(dict.fromkeys(out))
    return out[:count]


# ---- clouds -----------------------------------------------------------------------------------------------------------------
def rows(poses, w=None):
    p = np.asarray(poses, dtype=np.float64).reshape(-1, 3)
    a = np.empty((p.shape[0], 5))
    a[:, :3] = p
    a[:, 3] = 1.0
    a[:, 4] = 1.0 / p.shape[0] if w is None else w
    return a


def distinct(case, L=None):
    """n_min particles, particle i alone in bin (i, 0, 0), uniform weights"""
    i = np.arange(case.n_min)
    return rows(np.stack([X_BIN * i + 0.25, np.full(i.size, 0.25), np.full(i.size, 0.1)], axis=1))


def quantiser(case, L=None):
    big = 2.0 ** 30                                     # |x| / 0.5 >= 2^31 from here on: the key saturates
    e = math.nextafter
    xs = [big, e(big, 0.0), big - 0.5, e(big - 0.5, 0.0), 1e300, math.inf, -big, e(-big, 0.0), -big + 0.5, -big - 0.5, -1e300,
          -math.inf, math.nan, -math.nan, 0.0, -0.0, 5e-324, -5e-324, 0.25, 0.5, e(0.5, 0.0), -0.5, e(-0.5, 0.0), e(-0.5, -1.0),
          1.0, -1.0, 3.5, -3.5, 1e-300, -1e-300]
    yaws = [0.0, -0.0, 1e3, -1e3, 1e300, -1e300, math.inf, -math.inf, math.nan, YAW_BIN, e(YAW_BIN, 0.0), -YAW_BIN,
            e(-YAW_BIN, 0.0), math.pi, -math.pi, 2.0 * math.pi, 7.0 * YAW_BIN, -7.0 * YAW_BIN, 1e15, -1e15]
    p = []
    for j, x in enumerate(xs):                          # x along the row, y along the column, yaw ordinary, and the reverse
        p.append((x, 0.25, 0.1))
        p.append((0.25, x, 0.1))
        p.append((x, x, yaws[j % len(yaws)]))
    for yw in yaws:
        p.append((0.25, 0.25, yw))
    p = p[:case.n_min]
    assert len(p) == case.n_min
    return rows(p)


def hash_cloud(case, L=None):
    """keys in three probe chains of the device's table at n_max: 64 differing only in yaw and 64 arbitrary ones, all with
    home slot tcap - 1 (the chain wraps to slot 0), and 64 with home slot 5 (they queue behind the wrapped chain); the rest of
    the cloud is ordinary distinct bins"""
    tcap = table_size(case.n_max)
    rng = np.random.default_rng(case.seed)
    keys = colliding_keys(tcap, tcap - 1, 64, rng, vary="yaw") + colliding_keys(tcap, tcap - 1, 64, rng) + \
        colliding_keys(tcap, 5, 64, rng)
    keys = list(dict.fromkeys(keys))
    assert len(keys) == 192
    filler = [(i, 7, 0) for i in range(case.n_min - len(keys))]
    a = rows([pose_of(*k) for k in keys + filler])
    order = rng.permutation(case.n_min)                 # colliding keys spread over the cloud, not in a block
    return a[order]


def w_single(pos, mass=1.0):
    def build(case, L=None):
        a = distinct(case)
        a[:, 4] = 0.0
        a[{"first": 0, "mid": case.n_min // 2, "last": case.n_min - 1}[pos], 4] = mass
        return a
    return build


def w_zero_ends(case, L=None):
    """zero weights in the first and last 50 slots; the rest sums to 1 - 2^-10: draws above that fall through to the forced
    last CDF value 1.0, the last (zero-weight) particle"""
    a = distinct(case)
    rng = np.random.default_rng(case.seed)
    w = rng.uniform(0.5, 1.0, case.n_min)
    w[:50] = 0.0
    w[-50:] = 0.0
    a[:, 4] = w / w.sum() * (1.0 - 2.0 ** -10)
    return a


def w_cdf_ties(case, L):
    """CDF values equal to draws r_t (r_t in [1/2, 1): multiples of 2^-53, so every weight and prefix sum is exact), each
    followed by zero weights (the CDF repeats the value): the draw must pick the FIRST particle whose CDF value reaches it"""
    n = case.n_min
    r = draws(L, case.seed, case.n_max)
    vals = np.unique(r[(r >= 0.5)][:64])
    slots = np.linspace(2, n - 8, vals.size).astype(int)
    c = np.empty(n)
    prev, k = 0.5, 0
    for j in range(n):
        if k < vals.size and j == slots[k]:
            prev = vals[k]
            k += 1
        elif k < vals.size and j % 3 == 0:
            prev = max(prev, np.round(0.5 * (prev + vals[k]) / U53) * U53)      # between the targets: a non-decreasing CDF
        c[j] = prev
    c[-1] = 1.0
    assert np.all(np.diff(c) >= 0.0)
    a = distinct(case)
    a[:, 4] = np.diff(np.concatenate([[0.0], c]))
    assert np.array_equal(np.add.accumulate(a[:, 4]), c)
    return a


def w_special(kind):
    def build(case, L=None):
        a = distinct(case)
        rng = np.random.default_rng(case.seed)
        w = rng.uniform(0.1, 1.0, case.n_min)
        if kind == "negative":
            w[3::7] *= -1.5                             # the CDF goes down at these slots
        elif kind == "nan":
            w[(3 * case.n_min) // 4] = math.nan         # every CDF value after it is NaN (the forced last one is 1.0)
        elif kind == "inf":
            w[case.n_min // 3] = math.inf
        elif kind == "neg_zero":
            w[::3] = -0.0
        a[:, 4] = w / np.nansum(np.where(np.isfinite(w), w, 0.0))
        if kind == "nan":
            a[(3 * case.n_min) // 4, 4] = math.nan
        if kind == "inf":
            a[case.n_min // 3, 4] = math.inf
        return a
    return build


Z = 2.326
NEVER = 1e-6                                            # kld_required(2) ~ 3.3e6: clamped to n_max
_ZC = 60.0


def _zcarry_eps(target):
    term = 1.0 - 2.0 / 9.0 + _ZC * math.sqrt(2.0 / 9.0)
    return term ** 3 / (2.0 * (target - 0.5))


CASES = [
    # stop_*: (seed, eps) from search_eps over the clouds' real draws
    Case("stop_1023", 512, 4096, 0.2556547160784366, Z, 1, distinct, 1023),
    Case("stop_1024", 512, 4096, 0.250673766586313, Z, 2, distinct, 1024),
    Case("stop_1025", 512, 4096, 0.250427282394819, Z, 2, distinct, 1025),
    Case("stop_2048", 512, 4096, 0.1410533954269064, Z, 1, distinct, 2048),
    Case("stop_2049", 512, 4096, 0.14098403040439905, Z, 1, distinct, 2049),
    Case("stop_3078_of_3079", 1000, 3079, 0.1724866037705876, Z, 1, distinct, 3078),
    Case("zcarry_1025", 256, 4096, _zcarry_eps(1025), _ZC, 3, distinct, 1025),
    Case("zcarry_1800", 256, 4096, _zcarry_eps(1800), _ZC, 3, distinct, 1800),
    Case("zcarry_2049", 256, 4096, _zcarry_eps(2049), _ZC, 3, distinct, 2049),
    Case("never_2", 1, 2, NEVER, Z, 4, distinct, 1),
    Case("never_1023", 64, 1023, NEVER, Z, 4, distinct, 1023),
    Case("never_1023_min1022", 1022, 1023, NEVER, Z, 4, distinct, 1023),
    Case("never_1024", 64, 1024, NEVER, Z, 4, distinct, 1024),
    Case("never_1024_min1023", 1023, 1024, NEVER, Z, 4, distinct, 1024),
    Case("never_1025", 64, 1025, NEVER, Z, 4, distinct, 1025),
    Case("never_1025_min1024", 1024, 1025, NEVER, Z, 4, distinct, 1025),
    Case("never_3079", 64, 3 * 1024 + 7, NEVER, Z, 4, distinct, 3079),
    Case("never_3079_min3078", 3078, 3079, NEVER, Z, 4, distinct, 3079),
    Case("never_1048579", 4096, (1 << 20) + 3, NEVER, Z, 4, distinct, (1 << 20) + 3, big=True),
    Case("never_1048579_min1048578", (1 << 20) + 2, (1 << 20) + 3, NEVER, Z, 4, distinct, (1 << 20) + 3, big=True),
    Case("quantiser_edges", 110, 1024, 0.05, Z, 5, quantiser),
    Case("quantiser_edges_never", 110, 1500, NEVER, Z, 5, quantiser, 1500),
    Case("hash_collisions", 256, 1024, 0.2, Z, 6, hash_cloud),
    Case("hash_collisions_never", 256, 1024, NEVER, Z, 6, hash_cloud, 1024),
    Case("distinct_65536_stop_150001", 1 << 16, 1 << 18, 0.19910395870565875, Z, 1, distinct, 150001, big=True),
    Case("distinct_65536_never", 1 << 16, 1 << 18, 0.05, Z, 1, distinct, 1 << 18, big=True),
    Case("w_single_first", 300, 2000, 0.002, Z, 7, w_single("first"), 300),
    Case("w_single_mid", 300, 2000, 0.002, Z, 7, w_single("mid"), 300),
    Case("w_single_last", 300, 2000, 0.002, Z, 7, w_single("last"), 300),
    Case("w_single_mid_0.7", 300, 2000, 0.002, Z, 7, w_single("mid", 0.7)),
    Case("w_zero_ends", 300, 2000, 0.2, Z, 7, w_zero_ends),
    Case("w_cdf_ties", 300, 2000, 0.2, Z, 8, w_cdf_ties),
    Case("w_neg_zero", 300, 2000, 0.2, Z, 7, w_special("neg_zero")),
    Case("w_inf", 300, 2000, 0.2, Z, 7, w_special("inf")),
    Case("w_negative", 300, 2000, 0.2, Z, 7, w_special("negative")),
    Case("w_nan", 300, 2000, 0.2, Z, 7, w_special("nan")),
]
BY_NAME = {c.name: c for c in CASES}
