"""Grid-based FastSLAM's CPU oracle (tests/host/gs_oracle.c, DESIGN §3.16) against tests/golden/gs_golden.json, which the plain-Python
restatement in tests/_gs_oracle.py wrote: that restatement still reproduces it, the glibc oracle reproduces its weights and whole steps
(poses, weights, ancestors, N_eff, copies, fuse events and the SHA-256 of every step's grids) bit for bit, and the contract-math oracle
reproduces them with poses and weights to 1e-12."""
import hashlib
import json
import math
import os

import numpy as np
import pytest

import _gs_oracle as GO

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "gs_golden.json")


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


def weight_args(c, ogm):
    g = f64(c["grid"]).reshape(ogm["width"], ogm["height"])
    return g, f64(c["pose"]), f64(c["ranges"]), f64(c["angle_min"])[0], f64(c["angle_inc"])[0]


def test_restatement_reproduces_golden(gold):
    for c in gold["weights"]:
        w, used = GO.np_weight(*weight_args(c, gold["weight_ogm"]), gold["weight_ogm"], **c["model"])
        assert (u64([w])[0], used) == (c["w"], c["used"])
    ogm = gold["ogm"]
    for case in gold["cases"]:
        n = case["n"]
        st = dict(poses=np.tile(np.array(case["start"], dtype=np.float64), (n, 1)), w=np.full(n, 1.0 / n),
                  grids=np.zeros((n, ogm["width"], ogm["height"])))
        for s in case["steps"]:
            did, idx, neff, copies, events = GO.np_step(st, f64(s["odom"]), f64(s["ranges"]), -math.pi, 2 * math.pi / len(s["ranges"]),
                                                        f64(s["nz"]).reshape(n, 3), f64([s["u01"]])[0], case["nth"], ogm=ogm, **case["model"])
            assert (did, idx, u64([neff])[0], copies, events) == (s["resampled"], s["idx"], s["neff"], s["copies"], s["events"])
            assert u64(st["poses"]).tolist() == s["poses"] and u64(st["w"]).tolist() == s["w"] and digest(st["grids"]) == s["grids"]


@pytest.mark.parametrize("libm", [False, True])
def test_oracle_weights(gold, libm):
    for c in gold["weights"]:
        w, used = GO.weight(*weight_args(c, gold["weight_ogm"]), libm=libm, ogm=gold["weight_ogm"], **c["model"])
        assert used == c["used"]
        assert u64([w])[0] == c["w"], c["model"]


@pytest.mark.parametrize("libm", [False, True])
def test_oracle_steps(gold, libm):
    """glibc: bit for bit.  Contract math: its sin, cos, atan2 and exp may differ from glibc's in the last bit, so poses and weights
    are compared to 1e-12; ancestry, copies, events and the grids (whose cells these cases do not move) are still exact."""
    ogm = gold["ogm"]
    for case in gold["cases"]:
        n = case["n"]
        o = GO.OracleGs(n, case["start"], nth=case["nth"], libm=libm, ogm=ogm, **case["model"])
        for t, s in enumerate(case["steps"]):
            od = f64(s["odom"])
            did = o.step(od[:3], od[3:], f64(s["ranges"]), -math.pi, 2 * math.pi / len(s["ranges"]), nz=f64(s["nz"]), u01=f64([s["u01"]])[0])
            i = o.info()
            assert did == s["resampled"] and i.resampled == s["resampled"], (case["name"], t)
            assert o.last_indices().tolist() == (s["idx"] or [])
            assert (i.copies, i.events, i.steps) == (s["copies"], s["events"], t + 1)
            assert digest([o.grid(k) for k in range(n)]) == s["grids"]
            if libm:
                assert u64([i.neff])[0] == s["neff"]
                assert u64(o.particles()).tolist() == s["poses"], (case["name"], t)
                assert u64(o.weights()).tolist() == s["w"]
            else:
                assert math.isclose(i.neff, f64([s["neff"]])[0], rel_tol=1e-12)
                assert np.allclose(o.particles().ravel(), f64(s["poses"]), rtol=1e-12, atol=1e-12)
                assert np.allclose(o.weights(), f64(s["w"]), rtol=1e-12, atol=0.0)


def test_copies_match_ancestry(gold):
    for case in gold["cases"]:
        for s in case["steps"]:
            if s["resampled"]:
                assert s["copies"] == case["n"] - len(set(s["idx"]))


@pytest.mark.parametrize("libm", [False, True])
def test_refusals(libm):
    o = GO.OracleGs(4, (0.0, 0.0, 0.0), libm=libm, ogm=dict(resolution=0.5, width=12, height=10))
    assert o.step((math.nan, 0, 0), (0, 0, 0), np.ones(8), 0.0, 0.1) is None
    assert o.step((0, 0, 0), (0, 0, 0), np.ones(8), math.inf, 0.1) is None
    L = o.info().L
    assert L == GO.load(libm).orc_gs_limit(0.05 / 30.0, 0.95 + 0.05 / 30.0) and L > 1
    o2 = GO.OracleGs(4, (0.0, 0.0, 0.0), libm=libm, ogm=dict(resolution=0.5, width=12, height=10), max_beams=4096)
    assert o2.step((0, 0, 0), (0.1, 0, 0), np.full(L + 1, 2.0), 0.0, 0.01) is None
    assert o2.info().steps == 0
    assert o2.step((0, 0, 0), (0.1, 0, 0), np.full(L, 2.0), 0.0, 0.01) is not None
    assert o2.info().used == L
