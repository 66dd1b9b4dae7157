"""CPU tests of the likelihood-field scan model (DESIGN §3.9) on the oracle (tests/host/pf_lfield_oracle.c):
  - the glibc build reproduces tests/golden/lfield_golden.json (the Python restatement) bit for bit: the beam limit L, the distance
    field D, the factor table q, the used beams and the raw weight of every pose under every scan, and the refusal at L + 1 beams;
  - its distance field equals scipy.ndimage.distance_transform_edt on masks with an obstacle (to 1e-12 relative), an independent
    check of the restatement;
  - behaviour, with Philox draws: global localisation in ScanScenario's floor plan at 2^14 particles from init_region over the plan,
    recovery on, 60 steps: the estimate ends within 0.5 m and 0.1 rad of the truth."""
import json
import os

import numpy as np
import pytest
from scipy import ndimage

import _lfield_oracle as LF
import rust_robotics_b200 as rr
from rust_robotics_b200 import scenarios

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "lfield_golden.json")


def fx(v):
    if isinstance(v, list):
        return np.array([fx(a) for a in v])
    return float.fromhex(v)


def _cases():
    with open(GOLDEN) as f:
        return json.load(f)["cases"]


def _mask(c):
    return np.array([[ch == "1" for ch in row] for row in c["mask"]], dtype=bool).reshape(c["W"], c["H"])


@pytest.mark.parametrize("case", _cases(), ids=lambda c: c["name"])
def test_oracle_reproduces_golden(case):
    o = LF.OracleLField(4, libm=True)
    assert o.set_map(_mask(case), *fx(case["cfg"][:5]).tolist(), case["cfg"][5]) == 0
    assert o.info() == (case["W"], case["H"], case["L"])
    D, q = o.tables()
    assert np.array_equal(D, fx(case["D"])) and np.array_equal(q, fx(case["q"]))
    poses = fx(case["poses"])
    for j, s in enumerate(case["scans"]):
        args = (fx(s["ranges"]), fx(s["angle_min"]), fx(s["angle_inc"]))
        b, w = o.beams(*args), o.weights(poses, *args)
        if s["used"] < 0:
            assert b is None and w is None, f"scan {j}: not refused"
        else:
            assert b.shape[0] == s["used"] and np.array_equal(b.reshape(-1), fx(s["beams"]).reshape(-1)), f"scan {j}: beams"
            assert np.array_equal(w, fx(s["w"])), f"scan {j}: weights"


def test_golden_covers_the_cases():
    cases = {c["name"]: c for c in _cases()}
    assert all(float.fromhex(v) == 1e10 for row in cases["empty"]["D"] for v in row)
    assert all(float.fromhex(v) == 0.0 for row in cases["full"]["D"] for v in row)
    assert cases["row_1xN"]["W"] == 1 and cases["col_Nx1"]["H"] == 1
    bound = cases["beam_bound"]
    assert [s["used"] for s in bound["scans"]] == [bound["L"], -1]
    edge = cases["cell_edges"]["scans"][0]
    assert len(edge["w"]) == 5 and any(float.fromhex(v) > 0.0 for v in edge["w"])
    strides = {n: c["scans"][0]["used"] for n, c in cases.items() if n.startswith("stride_")}
    assert strides["stride_B361_mb60"] == 61 and strides["stride_B7_mb2"] == 2 and strides["stride_B1_mb60"] == 1
    nonsq = cases["nonsquare"]["scans"][0]
    ranges = fx(nonsq["ranges"])
    assert np.isnan(ranges).any() and np.isinf(ranges).any() and (ranges == 30.0).any()


@pytest.mark.parametrize("seed", range(6))
def test_distance_field_against_scipy(seed):
    rng = np.random.default_rng(seed)
    W, H = [(1, 40), (37, 1), (23, 31), (64, 48), (50, 50), (7, 90)][seed]
    m = rng.random((W, H)) < [0.02, 0.1, 0.05, 0.01, 0.3, 0.08][seed]
    m.flat[rng.integers(m.size)] = True
    for libm in (False, True):
        D = LF.compute_udf(m, libm)
        want = ndimage.distance_transform_edt(~m)
        assert np.allclose(D, want, rtol=1e-12, atol=0.0)
    for c in _cases():                                       # the golden masks with an obstacle
        mm = _mask(c)
        if mm.any():
            assert np.allclose(fx(c["D"]), ndimage.distance_transform_edt(~mm), rtol=1e-12, atol=0.0), c["name"]


def test_floor_plan_distance_field_against_scipy():
    m = scenarios.ScanScenario.plan()
    assert np.allclose(LF.compute_udf(m), ndimage.distance_transform_edt(~m), rtol=1e-12, atol=0.0)


def test_refusals():
    o = LF.OracleLField(8, mode=1, max_particles=8)
    m = np.zeros((4, 4), dtype=bool)
    assert o.update_scan([1.0], 0.0, 0.1) == -1                       # no map
    for bad in ((0.0,), (-1.0,), (np.nan,), (0.05, 0.0), (0.05, 0.2, -0.1), (0.05, 0.2, 0.95, 0.0), (0.05, 0.2, 0.95, 0.05, np.inf),
                (0.05, 0.2, 0.95, 0.05, 30.0, 1), (0.05, 0.2, 0.95, 1e-300, 1e10)):
        assert o.set_map(m, *bad) == -1, bad
    assert o.set_map(np.zeros((0, 4)), 0.05) == -1
    assert o.set_map(m, 0.05) == 0 and o.info()[2] == 109               # AMCL's defaults
    assert o.update_scan([1.0], np.nan, 0.1) == -1 and o.update_scan([1.0], 0.0, np.inf) == -1
    assert o.update_scan([], 0.0, 0.1) == 0 and np.all(o.particles()[:, 4] == 1.0 / 8)


def test_obstacles_from_log_odds():
    l = np.array([[-2.0, 0.0, 0.1], [800.0, -800.0, 2.0]])
    p = 1.0 - 1.0 / (1.0 + np.exp(np.clip(l, -700, 700)))
    assert np.array_equal(rr.obstacles_from_log_odds(l, 0.5), p > 0.5)
    assert np.array_equal(rr.obstacles_from_log_odds(l, 0.6), [[False, False, False], [True, False, True]])


@pytest.mark.parametrize("seed", [5, 6])
def test_global_localisation_in_floor_plan(seed):
    sc = scenarios.ScanScenario()
    n = 1 << 14
    o = LF.OracleLField(n, mode=1, max_particles=n, velocity_noise=0.2, yaw_rate_noise=0.1, seed=seed, threads=min(8, os.cpu_count() or 1))
    assert o.set_map(sc.obstacles, sc.RES) == 0
    o.enable(0.001, 0.1, sc.REGION)
    o.init_region(sc.REGION)
    err = [sc.error(k, o.step_scan(sc.controls[k], *sc.scan_args(k))[0]) for k in range(len(sc.controls))]
    assert err[-1][0] < 0.5 and err[-1][1] < 0.1, err[-1]
