"""CPU tests of the odometry motion model (DESIGN §3.14) on the oracle (tests/host/pf_odom_oracle.c):
  - the glibc build reproduces tests/golden/odom_golden.json (the Python restatement) bit for bit, with injected draws: the
    host-side increment and sigmas, single predicts (translation at the 0.01 guard and one ulp either side, pure rotation, pure
    translation, reversing, odometry yaw across +-pi, all alphas 0, no motion, particle yaw far outside +-pi), and filter runs (PF
    steps with the gate closed, KLD-adaptive MCL, recovery on, odometry steps mixed with velocity steps);
  - on random pairs the glibc build's increment and sigmas equal a numpy restatement bit for bit, and the contract build's agree
    with them to 1e-14;
  - with o == o' a predict leaves every pose equal as values;
  - behaviour, with Philox draws: OdomScenario (drive, stop, turn in place, reverse, drive; odometry with drift, seed 13) tracked by
    2^14 particles (MCL, filter seed 5) under the likelihood field from the start pose: position within 0.1 m and heading within
    0.02 rad of the truth in every phase (this run: 0.036 m and 0.0051 rad at most)."""
import json
import math
import os

import numpy as np
import pytest

import _odom_oracle as O
from rust_robotics_b200 import scenarios

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "odom_golden.json")


def fx(v):
    if isinstance(v, list):
        return np.array([fx(a) for a in v])
    return float.fromhex(v)


def _golden():
    with open(GOLDEN) as f:
        return json.load(f)


@pytest.mark.parametrize("case", _golden()["predicts"], ids=lambda c: c["name"])
def test_oracle_reproduces_golden_predict(case):
    o6, alpha = fx(case["odom"]), fx(case["alpha"])
    assert np.array_equal(O.increment(o6[:3], o6[3:], alpha, libm=True), fx(case["inc"]))
    init = fx(case["init"])
    o = O.OracleOdom(len(init), libm=True)
    o.upload(init)
    assert o.set_odom_noise(alpha) == 0
    assert o.predict_odom(o6[:3], o6[3:], fx(case["z3"])) == 0
    assert np.array_equal(o.particles(), fx(case["particles"]))


@pytest.mark.parametrize("case", _golden()["cases"], ids=lambda c: c["name"])
def test_oracle_reproduces_golden_filter(case):
    o = O.OracleOdom(case["n"], threshold=fx(case["threshold"]), range_noise=fx(case["sigma"]), velocity_noise=fx(case["sv"]),
                     yaw_rate_noise=fx(case["sw"]), dt=fx(case["dt"]), mode=case["mode"], max_particles=case["nmax"],
                     kld_epsilon=fx(case["eps"]), kld_z=fx(case["z"]), libm=True, fast_search=False)
    assert o.set_odom_noise(fx(case["alpha"])) == 0
    if "region" in case:
        assert o.enable(fx(case["a_slow"]), fx(case["a_fast"]), fx(case["region"])) == 0
    o.upload(fx(case["init"]))
    for t, s in enumerate(case["steps"]):
        cur = o.count()
        inj4 = fx(s["inj4"]) if s["inj4"] else np.zeros((cur, 4))
        if "odom" in s:
            o6 = fx(s["odom"])
            assert o.predict_odom(o6[:3], o6[3:], fx(s["z3"]), inj4) == 0
        else:
            assert o.predict(fx(s["u"]), fx(s["zv"]), fx(s["zw"]), inj4) == 0
        assert o.update(fx(s["obs"]).reshape(-1, 3)) == 0
        did = o.resample(fx(s["r"]))
        assert did == s["did_resample"], f"step {t}"
        if did:
            assert np.array_equal(o.last_indices(), np.array(s["indices"], dtype=np.uint32)), f"step {t}"
        assert o.count() == s["count"] and np.array_equal(o.estimate(), fx(s["est"])), f"step {t}"
    assert np.array_equal(o.particles(), fx(case["particles"]))


def test_golden_exercises_the_semantics():
    g = _golden()
    names = {c["name"]: c for c in g["predicts"]}
    assert fx(names["trans_below_min"]["inc"])[0] == 0.0 and fx(names["trans_at_min"]["inc"])[0] != 0.0
    assert abs(abs(fx(names["reversing"]["inc"])[0]) - math.pi) < 0.1
    z = names["alphas_zero"]
    assert np.all(fx(z["inc"])[3:] == 0.0)
    cases = {c["name"]: c for c in g["cases"]}
    pf = cases["pf_gate_closed_steps"]["steps"]
    assert any(not s["did_resample"] for s in pf) and any(s["did_resample"] for s in pf)
    assert len({s["count"] for s in cases["mcl_kld"]["steps"]}) > 1
    assert any(s["inj4"] for s in cases["mcl_recovery"]["steps"])
    mixed = cases["pf_mixed_velocity"]["steps"]
    assert any("u" in s for s in mixed) and any("odom" in s for s in mixed)


def _numpy_increment(o, a):
    """the rule of include/pf_odom_math.h, vectorised (angles wrapped by the same one-turn-at-a-time loop; atan2 is math.atan2, glibc's,
    since numpy's may be a vectorised one of its own)"""
    def norm(x):
        x = x.copy()
        while np.any(x > math.pi):
            x = np.where(x > math.pi, x - 2.0 * math.pi, x)
        while np.any(x < -math.pi):
            x = np.where(x < -math.pi, x + 2.0 * math.pi, x)
        return x
    dx, dy = o[:, 3] - o[:, 0], o[:, 4] - o[:, 1]
    trans = np.sqrt(dx * dx + dy * dy)
    rot1 = np.where(trans < 0.01, 0.0, norm(np.array([math.atan2(y, x) for y, x in zip(dy, dx)]) - o[:, 2]))
    rot2 = norm(norm(o[:, 5] - o[:, 2]) - rot1)
    n1 = np.minimum(np.abs(norm(rot1)), np.abs(norm(rot1 - math.pi)))
    n2 = np.minimum(np.abs(norm(rot2)), np.abs(norm(rot2 - math.pi)))
    tt = trans * trans
    return np.stack([rot1, trans, rot2, np.sqrt(a[0] * (n1 * n1) + a[1] * tt), np.sqrt((a[2] * tt + a[3] * (n1 * n1)) + a[3] * (n2 * n2)),
                     np.sqrt(a[0] * (n2 * n2) + a[1] * tt)], axis=1)


def test_increment_matches_numpy():
    rng = np.random.default_rng(4)
    o = np.concatenate([rng.uniform(-50, 50, (400, 2)), rng.uniform(-10, 10, (400, 1)), np.zeros((400, 3))], axis=1)
    step = rng.choice([1e-3, 5e-3, 0.05, 0.5, 3.0], 400)[:, None] * rng.normal(size=(400, 2))
    o[:, 3:5] = o[:, 0:2] + step
    o[:, 5] = o[:, 2] + rng.normal(0, 1.0, 400)
    a = np.array([0.1, 0.03, 0.2, 0.05])
    got = np.array([O.increment(r[:3], r[3:], a, libm=True) for r in o])
    assert np.array_equal(got, _numpy_increment(o, a))
    ctr = np.array([O.increment(r[:3], r[3:], a) for r in o])            # the contract libm: within a few ulp of glibc
    assert np.allclose(ctr, got, rtol=1e-14, atol=1e-15)


def test_refusals():
    assert O.increment((0.0, 0.0, np.nan), (1.0, 0.0, 0.0)) is None
    assert O.increment((0.0, 0.0, 0.0), (np.inf, 0.0, 0.0)) is None
    o = O.OracleOdom(8)
    for a in ((-0.1, 0.2, 0.2, 0.2), (0.2, np.nan, 0.2, 0.2), (0.2, 0.2, np.inf, 0.2)):
        assert o.set_odom_noise(a) == -1
    assert o.set_odom_noise((0.0, 0.0, 0.0, 0.0)) == 0


def test_no_motion_leaves_poses():
    o = O.OracleOdom(512, seed=9)
    assert o.init_state([3.0, -2.0, 7.0, 0.4]) == 0
    p0 = o.particles()
    for pose in ((0.0, 0.0, 0.0), (1e4, -3e3, -40.0), (2.5, 1.5, math.pi)):
        assert o.predict_odom(pose, pose) == 0
        assert np.array_equal(o.particles()[:, :4] == p0[:, :4], np.ones_like(p0[:, :4], dtype=bool))


def test_tracks_odom_scenario():
    sc = scenarios.OdomScenario()
    o = O.OracleOdom(1 << 14, mode=1, seed=5, threads=8)
    assert o.set_map(sc.obstacles, sc.RES) == 0
    assert o.init_state(list(sc.start) + [0.0]) == 0
    err = np.array([sc.error(t, o.step_scan_odom(*sc.odom_pair(t), *sc.scan_args(t))[0]) for t in range(sc.steps)])
    for name, (a, b) in sc.phases.items():
        assert err[a:b, 0].max() < 0.1 and err[a:b, 1].max() < 0.02, name
    # the stop: the odometry reads no motion, so no particle moves
    a, b = sc.phases["stop"]
    assert all(sc.odom[t] == sc.odom[a] for t in range(a, b + 1))
