"""Certified CDF of the fused FastSLAM post kernel (DESIGN §1), on the CPU: wherever the certificate of c~_j = fl(P_j / S)
passes, the resample indices searched in c~ equal those of the reference's plain loop (normalise, re-normalise, cum_sum,
r += 1/n); comb values placed within a few ulps of a CDF value are refused.  The model is tests/host/cdf_cert_emul.cpp on the
kernel's own certificate (x3_cdf_near_comb in rust_robotics_b200/csrc/x3_core.h)."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "host", "cdf_cert_emul.cpp")
LIB = os.path.join(ROOT, "tests", "host", "libcdf_cert_emul.so")
dp = C.POINTER(C.c_double)
up = C.POINTER(C.c_uint)


@pytest.fixture(scope="module")
def emul():
    subprocess.run(["/usr/bin/g++", "-O2", "-ffp-contract=off", "-fPIC", "-shared", "-o", LIB, SRC], check=True)
    L = C.CDLL(LIB)
    L.cdf_cert_emul.argtypes = [dp, C.c_int, C.c_double, up, up, dp, dp]
    L.cdf_cert_emul.restype = C.c_int
    return L


def run(L, w, p, r0, want_cdf=False):
    n = 1 << p
    w = np.ascontiguousarray(w, dtype=np.float64)
    ia, ib = np.empty(n, np.uint32), np.empty(n, np.uint32)
    ca, cb = (np.empty(n), np.empty(n)) if want_cdf else (None, None)
    near = L.cdf_cert_emul(w.ctypes.data_as(dp), p, r0, ia.ctypes.data_as(up), ib.ctypes.data_as(up),
                           ca.ctypes.data_as(dp) if want_cdf else None, cb.ctypes.data_as(dp) if want_cdf else None)
    return near, ia, ib, ca, cb


def weights(kind, n, rng):
    if kind == "random":
        return rng.uniform(size=n)
    if kind == "near_uniform":
        return 1.0 + rng.uniform(-1e-9, 1e-9, n)
    if kind == "uniform":
        return np.full(n, 0.37)
    if kind == "degenerate":
        w = np.full(n, 1e-300); w[rng.integers(n)] = 1.0; return w
    if kind == "sparse":
        w = np.zeros(n); w[rng.integers(0, n, max(1, n // 64))] = rng.uniform(size=max(1, n // 64)); return w
    if kind == "heavy_tailed":
        return np.exp(rng.normal(0, 8, n))
    if kind == "pareto":
        return rng.pareto(0.7, n) + 1e-12
    raise ValueError(kind)


KINDS = ["random", "near_uniform", "uniform", "degenerate", "sparse", "heavy_tailed", "pareto"]


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("p", [6, 9, 12, 16, 19])
def test_certified_indices_equal_the_reference(emul, kind, p):
    rng = np.random.default_rng(1000 * p + KINDS.index(kind))
    n = 1 << p
    passed = 0
    for trial in range(6 if p < 19 else 2):
        w = weights(kind, n, rng)
        r0 = float(np.floor(rng.uniform() * 2.0 ** 52) / 2.0 ** 52) / n        # Uniform(0, 1/n) as the kernel draws it
        near, ia, ib, _, _ = run(emul, w, p, r0)
        if not near:
            passed += 1
            assert np.array_equal(ia, ib), f"{kind} p={p}: certificate passed but {int((ia != ib).sum())} indices differ"
    if kind in ("random", "heavy_tailed", "degenerate") and p <= 16:
        assert passed > 0, "the certificate never passed"


@pytest.mark.parametrize("kind", ["random", "near_uniform", "heavy_tailed"])
@pytest.mark.parametrize("p", [6, 10, 16])
@pytest.mark.parametrize("ulps", [-3, -1, 0, 1, 3])
def test_comb_within_a_few_ulps_is_refused(emul, kind, p, ulps):
    """r0 chosen so that a comb value lands within a few ulps of one of the reference's CDF values"""
    rng = np.random.default_rng(7 * p + ulps + 100)
    n = 1 << p
    w = weights(kind, n, rng)
    _, _, _, _, c = run(emul, w, p, 0.0, want_cdf=True)
    for j in rng.integers(0, n - 1, 4):
        target = float(c[j])
        t = int(np.floor(target * n))
        r0 = target - t / n
        if not (0.0 <= r0 < 1.0 / n):
            continue
        r0 = float(np.nextafter(r0, np.inf if ulps > 0 else -np.inf)) if ulps else r0
        for _ in range(abs(ulps) - 1):
            r0 = float(np.nextafter(r0, np.inf if ulps > 0 else -np.inf))
        if not (0.0 <= r0 < 1.0 / n):
            continue
        near, ia, ib, _, _ = run(emul, w, p, r0)
        assert near == 1, f"{kind} p={p} j={j}: comb value {ulps} ulps from c_j was not refused"


def test_refusals_cover_every_mismatch(emul):
    """many comb offsets right at the CDF values: whenever the searched indices differ, the certificate has refused"""
    rng = np.random.default_rng(5)
    p = 12
    n = 1 << p
    w = weights("random", n, rng)
    _, _, _, ct, c = run(emul, w, p, 0.0, want_cdf=True)
    mism = 0
    for j in rng.integers(0, n - 1, 200):
        for src in (c, ct):
            t = int(np.floor(src[j] * n))
            base = float(src[j]) - t / n
            for k in range(-4, 5):
                r0 = base
                for _ in range(abs(k)):
                    r0 = float(np.nextafter(r0, np.inf if k > 0 else -np.inf))
                if not (0.0 <= r0 < 1.0 / n):
                    continue
                near, ia, ib, _, _ = run(emul, w, p, r0)
                if not np.array_equal(ia, ib):
                    mism += 1
                    assert near == 1
    assert mism > 0, "no offset reproduced a rounding difference: the test does not exercise the certificate"
