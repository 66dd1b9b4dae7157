"""include/pf_moments.h on the CPU: the PF / MCL estimate and covariance replayed in the device's reduction order
(tests/host/pf_moments_test.c, compiled without contraction like the kernels) on adversarial clouds, against the exact
two-pass reference of tests/_pf_moments_cases.py.  The replay is bit-identical to the device (tests/test_gpu_pf_moments.py
checks that), so the error claims of DESIGN §1 hold without a GPU.

Forms: the separate kernels (pf_moments_kernel + pf_moments_reduce_kernel, also per rank of a sharded engine) and the fused
step tail (pf3_post_kernel), at the geometry an H100 SXM (132 SMs) gives them."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import _pf_moments_cases as pm

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "host", "pf_moments_test.c")
SMS = 132
dp = C.POINTER(C.c_double)


@pytest.fixture(scope="module")
def lib(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("pf_moments") / "libpf_moments_test.so")
    subprocess.run(["/usr/bin/gcc", "-O2", "-ffp-contract=off", "-fPIC", "-shared", "-o", so, SRC, "-lm"], check=True)
    L = C.CDLL(so)
    L.pf_moments_replay.argtypes = [dp, C.c_size_t, C.c_int, C.c_uint, C.c_uint, C.c_uint, dp, dp]
    return L


def replay(L, a, form, shards=1):
    a = np.ascontiguousarray(a, dtype=np.float64)
    n = a.shape[0]
    b0, tiles, k = pm.geometry(n // shards, SMS)
    est, cov = np.empty(4), np.empty(16)
    rc = L.pf_moments_replay(a.ctypes.data_as(dp), n, form, b0 if form == 0 else tiles, k, shards, est.ctypes.data_as(dp),
                             cov.ctypes.data_as(dp))
    assert rc == 0
    return est, cov.reshape(4, 4)


def check_both_forms(L, a, what):
    ref = pm.exact(a)
    for form in (0, 1):
        est, cov = replay(L, a, form)
        bad = pm.violations(est, cov, a, ref)
        assert not bad, f"{what}, form {form}: {bad}"


def _grid():
    out = []
    for n in pm.SIZES:
        for off in pm.OFFSETS:
            for sp in pm.SPREADS:
                for wk in pm.WEIGHTS:
                    if n >= 1 << 16 and (wk in ("random", "zero") or sp == "1m"):
                        continue                           # the large sizes keep the cases that stress the arithmetic
                    out.append(pytest.param(n, off, sp, wk, id=f"{n}-{off}-{sp}-{wk}"))
    return out


@pytest.mark.parametrize("n,off,sp,wk", _grid())
def test_clouds(lib, n, off, sp, wk):
    check_both_forms(lib, pm.cloud(n, pm.OFFSETS[off], pm.SPREADS[sp], wk, seed=n), f"n {n} offset {off} spread {sp} weights {wk}")


@pytest.mark.parametrize("n", [17, 1000, 4096, 1 << 16, 1 << 18])
@pytest.mark.parametrize("where", ["slot0", "thread_firsts"])
def test_zero_weight_outliers(lib, n, where):
    """a zero-weight particle 10 km away must not become anybody's centre"""
    a = pm.cloud(n, pm.UTM, 1e-2, "random", seed=3)
    slots = np.array([0]) if where == "slot0" else np.flatnonzero(pm.thread_first_slots(n, SMS))
    a = pm.with_zero_weight_outliers(a, slots)
    a[:, 4] /= a[:, 4].sum()
    check_both_forms(lib, a, where)


@pytest.mark.parametrize("n", [4096, 1 << 16, 1 << 18])
@pytest.mark.parametrize("half_width", [1.0e3, 1.0e4])
def test_injected_outliers(lib, n, half_width):
    """5 % of the particles at weight 1e-100 over +-1 km / +-10 km around a 1 cm cloud at UTM coordinates"""
    check_both_forms(lib, pm.injected(n, half_width, seed=n), f"+-{half_width} m")


@pytest.mark.parametrize("shards", [2, 4, 8])
def test_sharded_rank_order_merge(lib, shards):
    n = 1 << 16
    for off, sp, wk in [("utm", "1mm", "random"), ("utm", "zero", "uniform"), ("1e4", "1cm", "ones")]:
        a = pm.cloud(n, pm.OFFSETS[off], pm.SPREADS[sp], wk, seed=shards)
        est, cov = replay(lib, a, 0, shards)
        assert not pm.violations(est, cov, a), f"{shards} shards, {off} {sp} {wk}"
    a = pm.injected(n, 1.0e4, seed=1)
    est, cov = replay(lib, a, 0, shards)
    assert not pm.violations(est, cov, a)


@pytest.mark.parametrize("n", [17, 4096, 1 << 16])
def test_non_finite_poses(lib, n):
    """inf / NaN in one coordinate of one particle (weighted, or of weight zero): non-finite exactly where the reference's sums
    are, everything else within the bar"""
    for col, val, w0 in [(0, np.inf, False), (1, -np.inf, False), (2, np.nan, False), (3, np.inf, True), (0, np.nan, True)]:
        a = pm.cloud(n, pm.UTM, 1e-2, "random", seed=7)
        i = n // 2
        a[i, col] = val
        if w0:
            a[i, 4] = 0.0
        ref = pm.exact(a)
        assert not np.isfinite(ref[0][col]) and np.isfinite(ref[0][(col + 1) % 4])
        for form in (0, 1):
            est, cov = replay(lib, a, form)
            bad = pm.violations(est, cov, a, ref)
            assert not bad, f"col {col} = {val}, zero weight {w0}, form {form}: {bad}"


def test_the_old_formula_fails_where_the_new_one_holds(lib):
    """the one-pass raw moments about a stale centre (the previous estimate, here 0) that the device used before: the same
    clouds break the bar, so the cases above can tell the two apart"""
    def raw_about(a, c):
        w, e = a[:, 4], a[:, :4] - c
        W, M1, M2 = w.sum(), (w[:, None] * e).sum(axis=0), np.einsum("i,ij,ik->jk", w, e, e)
        ea = c * (W - 1.0) + M1
        return c * W + M1, M2 - np.outer(M1, ea) - np.outer(ea, M1) + W * np.outer(ea, ea)

    for a in (pm.cloud(4096, pm.UTM, 1.0, "random"), pm.cloud(4096, pm.UTM, 0.0, "random"), pm.cloud(4096, pm.OFFSETS["1e4"], 1e-2, "random"),
              pm.cloud(4096, pm.UTM, 1e-2, "random")):
        assert pm.violations(*raw_about(a, np.zeros(4)), a)
        assert not pm.violations(*replay(lib, a, 0), a)
