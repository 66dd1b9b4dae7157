"""The PF / MCL estimate and covariance (refresh_cache, pf.rs:382-413) against an exact reference: adversarial clouds, the
exact two-pass values and the bar.  Shared by tests/test_pf_moments_host.py (the device's reduction order replayed on the CPU)
and tests/test_gpu_pf_moments.py (the device).

Bar:
  * estimate: |est - exact| <= 1e-12 (|exact| + 1) per component;
  * covariance: |cov_ij - exact_ij| <= 1e-6 sqrt(exact_ii exact_jj) + atol, atol = (n 2^-53 max|p|)^2, the size of the
    reference's own rounding on a cloud without spread; every diagonal entry >= 0;
  * non-finite poses: non-finite entries exactly where the reference's sums are non-finite, the others within the bar.
"""
import math

import numpy as np

UTM = (5.0e5, 5.0e6)
OFFSETS = {"origin": (0.0, 0.0), "1e2": (1.0e2, 1.0e2), "1e4": (1.0e4, 1.0e4), "utm": UTM}
SPREADS = {"1mm": 1e-3, "1cm": 1e-2, "1m": 1.0, "zero": 0.0}
WEIGHTS = ("uniform", "random", "dominant", "ones", "zero")
SIZES = (1, 17, 1000, 4096, 1 << 16, 1 << 18)
NT = 256


def geometry(n, sms):
    """(blocks of pf_moments_kernel, tiles and particles per thread of pf3_post_kernel) at n particles on `sms` SMs"""
    b0 = max(1, min(sms * 4, -(-n // NT)))
    tiles = min(min(sms, 160), -(-n // NT))
    k = -(-n // (tiles * NT))
    return b0, -(-n // (NT * k)), k


def weights(kind, n, rng):
    if kind == "uniform":
        return np.full(n, 1.0 / n)
    if kind == "random":
        w = rng.uniform(size=n)
        return w / w.sum()
    if kind == "dominant":
        w = np.full(n, 1e-9 / max(n - 1, 1))
        w[n // 3] = 1.0 - 1e-9 if n > 1 else 1.0
        return w
    if kind == "ones":
        return np.ones(n)                           # W = n: the reference's estimate is n * mean
    if kind == "zero":
        return np.zeros(n)
    raise ValueError(kind)


def cloud(n, offset, spread, wkind, seed=0):
    """n rows (x, y, yaw, v, w) around `offset` with standard deviation `spread`; yaw near 40 rad and v near -7.5 (the PF never
    wraps yaw), so no coordinate is small"""
    rng = np.random.default_rng(seed)
    a = np.empty((n, 5))
    a[:, 0] = offset[0] + spread * rng.standard_normal(n)
    a[:, 1] = offset[1] + spread * rng.standard_normal(n)
    a[:, 2] = 40.0 + 0.5 * spread * rng.standard_normal(n)
    a[:, 3] = -7.5 + 2.0 * spread * rng.standard_normal(n)
    a[:, 4] = weights(wkind, n, rng)
    return a


def with_zero_weight_outliers(a, slots, dist=1.0e4):
    """zero-weight particles `dist` metres away at the given slots"""
    a = a.copy()
    a[slots, 0] += dist
    a[slots, 1] -= dist
    a[slots, 4] = 0.0
    return a


def thread_first_slots(n, sms):
    """every slot that is the first particle of a thread in either reduction form (and slot 0)"""
    b0, _tiles, k = geometry(n, sms)
    m = np.zeros(n, dtype=bool)
    if n > b0 * NT:
        m[:b0 * NT] = True                          # pf_moments_kernel: thread t starts at slot t
    m[::k] = True                                   # pf3_post_kernel: thread tid of tile b starts at (b NT + tid) K
    if m.all():                                     # one particle per thread: every other slot, so some weight is left
        m[1::2] = False
    m[0] = True
    return m


def injected(n, half_width, seed=0):
    """a 1 cm cloud at the UTM offset with 5 % of its particles at weight 1e-100 spread over +-half_width: what augmented-MCL
    injection leaves on a large map"""
    rng = np.random.default_rng(seed)
    a = cloud(n, UTM, 1e-2, "uniform", seed)
    k = rng.random(n) < 0.05
    a[k, 0] = UTM[0] + rng.uniform(-half_width, half_width, k.sum())
    a[k, 1] = UTM[1] + rng.uniform(-half_width, half_width, k.sum())
    a[:, 4] = np.where(k, 1e-100, 1.0)
    a[:, 4] /= a[:, 4].sum()
    return a


def exact(a):
    """the reference's definition, est = sum w p (not divided by sum w), cov = sum w (p - est)(p - est)^T, each sum with
    math.fsum (exactly rounded); for non-finite input, numpy's plain sums (which are non-finite where the reference's are)"""
    w, p = a[:, 4], a[:, :4]
    with np.errstate(all="ignore"):
        if not np.all(np.isfinite(a)):
            est = (w[:, None] * p).sum(axis=0)
            d = p - est
            return est, np.einsum("i,ij,ik->jk", w, d, d)
        est = np.array([math.fsum(w * p[:, k]) for k in range(4)])
        d = p - est
        cov = np.empty((4, 4))
        for i in range(4):
            for j in range(i, 4):
                cov[i, j] = cov[j, i] = math.fsum(w * d[:, i] * d[:, j])
    return est, cov


def violations(est, cov, a, ref=None, est_slack=0.0):
    """[] when (est, cov) meets the bar against the exact reference of cloud a (or against ref = (est, cov), with est_slack
    added to the estimate's bar), else what fails"""
    re, rc = exact(a) if ref is None else ref
    est, cov = np.asarray(est, dtype=np.float64), np.asarray(cov, dtype=np.float64).reshape(4, 4)
    bad = []
    fe, fc = np.isfinite(re), np.isfinite(rc)
    if not np.array_equal(np.isfinite(est), fe) or not np.array_equal(np.isfinite(cov), fc):
        bad.append(f"non-finite pattern: est {np.isfinite(est)} vs {fe}; cov {np.isfinite(cov).ravel()} vs {fc.ravel()}")
    de = np.abs(est - re)[fe]
    if np.any(de > 1e-12 * (np.abs(re[fe]) + 1.0) + np.broadcast_to(est_slack, re.shape)[fe]):
        bad.append(f"estimate {est} vs exact {re}")
    finite = a[:, :4][np.isfinite(a[:, :4])]
    atol = (a.shape[0] * 2.0 ** -53 * (np.max(np.abs(finite)) if finite.size else 0.0)) ** 2
    dg = np.abs(np.diag(rc))
    with np.errstate(invalid="ignore"):
        tol = 1e-6 * np.sqrt(np.outer(dg, dg)) + atol
        over = (np.abs(cov - rc) > tol) & fc
    if np.any(over):
        i, j = np.argwhere(over)[0]
        bad.append(f"cov[{i},{j}] = {cov[i, j]!r} vs exact {rc[i, j]!r} (bar {tol[i, j]:.3g}); "
                   f"worst relative {np.nanmax(np.where(fc, np.abs(cov - rc) / np.where(tol > 0, tol, 1.0), 0.0)):.3g} of the bar")
    if np.any(np.diag(cov)[np.diag(fc)] < 0.0):
        bad.append(f"negative variance {np.diag(cov)}")
    return bad
