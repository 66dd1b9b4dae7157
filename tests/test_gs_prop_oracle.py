"""The scan-matched proposal's CPU oracle (tests/host/gs_prop_oracle.c, DESIGN §3.17) against tests/golden/gs_prop_golden.json, which
the plain-Python restatement in tests/_gs_prop_oracle.py wrote: that restatement still reproduces it, the glibc oracle reproduces
every particle case and whole step (poses, weights, x^, eta, took, ancestors, N_eff, copies, fuse events and the SHA-256 of every
step's grids) bit for bit, and the contract-math oracle reproduces everything discrete exactly and poses, weights and eta to 1e-9
relative.  That bar is wider than §3.16's 1e-12 because the prior's inverse A carries the last-bit differences of the contract sin
and cos into pi_j = exp(-d^T A d / 2) amplified by its condition number (up to Sigma's largest variance over eps = 1e-8)."""
import hashlib
import json
import math
import os

import numpy as np
import pytest

import _gs_oracle as GO
import _gs_prop_oracle as PO

TOL = 1e-9
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "gs_prop_golden.json")


@pytest.fixture(scope="module")
def gold():
    with open(GOLDEN) as f:
        return json.load(f)


def f64(bits):
    return np.array(bits, dtype=np.uint64).view(np.float64)


def u64(a):
    return np.ascontiguousarray(a, dtype=np.float64).view(np.uint64).ravel()


def digest(grids):
    return hashlib.sha256(np.ascontiguousarray(grids, dtype=np.float64).tobytes()).hexdigest()


def particle_args(c, ogm):
    r = f64(c["ranges"])
    return (f64(c["grid"]).reshape(ogm["width"], ogm["height"]), f64(c["pose"]), f64(c["odom"]), r, -math.pi, 2 * math.pi / len(r),
            f64(c["z4"]))


def close(a, b):
    a, b = np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64)
    return np.array_equal(np.isnan(a), np.isnan(b)) and np.allclose(a[~np.isnan(a)], b[~np.isnan(b)], rtol=TOL, atol=1e-12)


def test_restatement_reproduces_golden(gold):
    ogm = gold["ogm"]
    for c in gold["particles"]:
        p, f, xh, eta, took = PO.np_one(*particle_args(c, ogm), prop=c["prop"], ogm=ogm, alpha=c["alpha"], **c["model"])
        assert u64(p).tolist() == c["out_pose"] and u64([f])[0] == c["factor"] and u64(xh).tolist() == c["xh"], c["name"]
        assert (u64([eta])[0], took) == (c["eta"], c["took"]), c["name"]
    for case in gold["cases"]:
        n = case["n"]
        st = dict(poses=np.tile(np.array(case["start"], dtype=np.float64), (n, 1)), w=np.full(n, 1.0 / n),
                  grids=np.zeros((n, ogm["width"], ogm["height"])))
        for s in case["steps"]:
            r = f64(s["ranges"])
            did, idx, neff, copies, events, xh, eta, took = PO.np_step(st, f64(s["odom"]), r, -math.pi, 2 * math.pi / len(r),
                                                                       f64(s["nz"]).reshape(n, 4), f64([s["u01"]])[0], case["nth"],
                                                                       prop=case["prop"], ogm=ogm, **case["model"])
            assert (did, idx, u64([neff])[0], copies, events) == (s["resampled"], s["idx"], s["neff"], s["copies"], s["events"])
            assert u64(st["poses"]).tolist() == s["poses"] and u64(st["w"]).tolist() == s["w"] and digest(st["grids"]) == s["grids"]
            assert u64(xh).tolist() == s["xh"] and u64(eta).tolist() == s["eta"] and took.tolist() == s["took"]


@pytest.mark.parametrize("libm", [False, True])
def test_oracle_particles(gold, libm):
    """glibc: bit for bit.  Contract math: its sin, cos, atan2 and exp may differ from glibc's in the last bit"""
    ogm = gold["ogm"]
    for c in gold["particles"]:
        p, f, xh, eta, took = PO.one(*particle_args(c, ogm), prop=c["prop"], libm=libm, ogm=ogm, alpha=c["alpha"], **c["model"])
        assert took == c["took"], c["name"]
        if libm:
            assert u64(p).tolist() == c["out_pose"] and u64([f])[0] == c["factor"], c["name"]
            assert u64(xh).tolist() == c["xh"] and u64([eta])[0] == c["eta"], c["name"]
        else:
            assert close(p, f64(c["out_pose"])) and close(xh, f64(c["xh"])), c["name"]
            assert math.isclose(f, f64([c["factor"]])[0], rel_tol=TOL) and close([eta], f64([c["eta"]])), c["name"]


@pytest.mark.parametrize("libm", [False, True])
def test_oracle_steps(gold, libm):
    ogm = gold["ogm"]
    for case in gold["cases"]:
        n = case["n"]
        o = PO.OracleGsProp(n, case["start"], nth=case["nth"], libm=libm, ogm=ogm, prop=case["prop"], **case["model"])
        for t, s in enumerate(case["steps"]):
            od, r = f64(s["odom"]), f64(s["ranges"])
            did = o.step(od[:3], od[3:], r, -math.pi, 2 * math.pi / len(r), nz=f64(s["nz"]), u01=f64([s["u01"]])[0])
            i = o.info()
            xh, eta, took = o.last_proposal()
            assert did == s["resampled"] and took.tolist() == s["took"], (case["name"], t)
            assert o.last_indices().tolist() == (s["idx"] or [])
            assert (i.copies, i.events, i.steps) == (s["copies"], s["events"], t + 1)
            if libm:
                assert u64([i.neff])[0] == s["neff"] and u64(o.particles()).tolist() == s["poses"] and u64(o.weights()).tolist() == s["w"]
                assert u64(xh).tolist() == s["xh"] and u64(eta).tolist() == s["eta"]
                assert digest([o.grid(k) for k in range(n)]) == s["grids"]
            else:
                assert math.isclose(i.neff, f64([s["neff"]])[0], rel_tol=TOL)
                assert close(o.particles().ravel(), f64(s["poses"])) and close(o.weights(), f64(s["w"]))
                assert close(xh.ravel(), f64(s["xh"])) and close(eta, f64(s["eta"]))


@pytest.mark.parametrize("libm", [False, True])
def test_min_hits_above_beams_is_the_plain_oracle(libm):
    """every particle falls back: the proposal oracle's steps equal gs_oracle.c's plain steps bit for bit"""
    ogm = dict(resolution=0.1, width=16, height=12)
    rng = np.random.default_rng(3)
    a = PO.OracleGsProp(4, (0.1, 0.0, 0.2), seed=4, libm=libm, ogm=ogm, prop=dict(PO.PROP, min_hits=1000), max_range=5.0)
    b = GO.OracleGs(4, (0.1, 0.0, 0.2), seed=4, libm=libm, ogm=ogm, max_range=5.0)
    for t in range(5):
        od, r = (0.03 * t, 0.0, 0.01 * t), rng.uniform(0.3, 0.7, 24)
        od2 = (0.03 * t + 0.04, 0.01, 0.01 * t + 0.02)
        assert a.step(od, od2, r, -math.pi, 2 * math.pi / 24) == b.step(od, od2, r, -math.pi, 2 * math.pi / 24)
        assert not a.last_proposal()[2].any()
        assert np.array_equal(u64(a.particles()), u64(b.particles())) and np.array_equal(u64(a.weights()), u64(b.weights()))
        assert all(np.array_equal(u64(a.grid(k)), u64(b.grid(k))) for k in range(4))
