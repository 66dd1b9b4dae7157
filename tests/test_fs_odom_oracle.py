"""CPU checks of FastSLAM's odometry motion model (include/fs_odom_math.h, DESIGN §3.15) on its oracle (tests/host/fs_odom_oracle.c):
the glibc build against the independent Python restatement (tests/golden/fs_odom_golden.json) bit for bit, the prior's covariance
against a finite-difference Jacobian, standstill, and the proposal on a turn in place and a reverse (the eps floor)."""
import json
import math
import os
import sys

import numpy as np
import pytest

import _fs_odom_oracle as F

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "fs_odom_golden.json")


def _golden():
    with open(GOLDEN) as f:
        return json.load(f)["cases"]


@pytest.mark.parametrize("libm", [True])
def test_oracle_matches_golden(libm):
    cases = _golden()
    assert len(cases) == 270 and {c["case"] for c in cases} == {0, 1, 2}
    for j, c in enumerate(cases):
        a, b = c["odom"][:3], c["odom"][3:]
        assert list(F.increment(a, b, c["alpha"], libm=libm)) == c["increment"], j
        mu, cov = F.prior(a, b, c["pose"], c["alpha"], libm=libm)
        assert list(mu) == c["mu"] and list(cov.ravel()) == c["cov"], j
        assert list(F.move(a, b, c["pose"], c["n3"], c["alpha"], libm=libm)) == c["move"], j
        kase, p = F.pose2(a, b, c["pose"], c["lm"], c["z"], c["n3"], c["alpha"], libm=libm)
        assert kase == c["case"] and list(p) == c["pose2"], j


def test_contract_build_close_to_glibc():
    for c in _golden()[:60]:
        a, b = c["odom"][:3], c["odom"][3:]
        kase, p = F.pose2(a, b, c["pose"], c["lm"], c["z"], c["n3"], c["alpha"])
        assert kase == c["case"] and np.allclose(p, c["pose2"], rtol=0, atol=1e-9)


@pytest.mark.parametrize("odom", [[0.0, 0.0, 0.0, 1.0, 0.2, 0.1], [3.0, -2.0, 0.3, 2.6, -2.1, 0.35], [1.0, 1.0, 2.0, 1.5, 1.7, -2.5]])
@pytest.mark.parametrize("pose", [[1.0, 2.0, 0.3], [-4.0, 7.5, 3.0]])
def test_prior_covariance_matches_finite_difference(odom, pose):
    """Sigma = V D V^T with V = d(x, y, yaw) / d(rot1, trans, rot2) of the move, checked against central differences of the move"""
    inc = F.increment(odom[:3], odom[3:])
    rot1, trans, rot2, s1, st, s2 = inc

    def f(r1, t, r2):
        s, c = math.sin(pose[2] + r1), math.cos(pose[2] + r1)
        return np.array([pose[0] + t * c, pose[1] + t * s, pose[2] + r1 + r2])

    h = 1e-6
    x0 = np.array([rot1, trans, rot2])
    V = np.column_stack([(f(*(x0 + h * e)) - f(*(x0 - h * e))) / (2 * h) for e in np.eye(3)])
    want = V @ np.diag([s1 * s1, st * st, s2 * s2]) @ V.T + 1e-8 * np.eye(3)
    _, cov = F.prior(odom[:3], odom[3:], pose)
    assert np.allclose(cov, want, rtol=1e-6, atol=1e-9)


@pytest.mark.parametrize("lm", [[6.0, 4.0, 1.5, 0.1, 0.1, 2.0], [0.0, 0.0, 1000.0, 0.0, 0.0, 1000.0]])
def test_standstill_returns_the_pose_bit_for_bit(lm):
    still = [3.0, -2.0, 1.2]
    for pose in ([1.0, 2.0, 0.3], [-4.0, 7.5, 3.0], [0.5, -0.25, -2.9]):
        assert list(F.move(still, still, pose, [1.3, -0.7, 2.1])) == pose
        kase, p = F.pose2(still, still, pose, lm, [5.0, 0.2], [1.3, -0.7, 2.1])
        assert kase == 0 and list(p) == pose


@pytest.mark.parametrize("odom, rank", [([3.0, -2.0, 1.2, 3.0, -2.0, 2.9], 2),                 # turn in place: V has rank 2
                                        ([3.0, -2.0, 1.2, 3.0, -2.0, -1.5], 2),
                                        ([3.0, -2.0, 0.3, 3.0 - 0.4 * math.cos(0.3), -2.0 - 0.4 * math.sin(0.3), 0.35], 3)])   # reverse
def test_proposal_on_rotation_and_reverse_stays_near_mu(odom, rank):
    """With the eps floor the proposal is finite and stays within 2 m of mu (the observation's pull included) on turns in place,
    where the prior without the floor is singular, and on reverses (rot1 near pi)."""
    pose = [1.0, 2.0, 0.3]
    lm = [6.0, 4.0, 1.5, 0.1, 0.1, 2.0]
    rng = np.random.default_rng(3)
    mu, cov = F.prior(odom[:3], odom[3:], pose)
    assert np.linalg.matrix_rank(cov - 1e-8 * np.eye(3), tol=1e-9) == rank
    dx, dy = lm[0] - mu[0], lm[1] - mu[1]
    z = [math.hypot(dx, dy), math.atan2(dy, dx) - mu[2]]
    for _ in range(50):
        kase, p = F.pose2(odom[:3], odom[3:], pose, lm, z, rng.standard_normal(3))
        assert kase == 2 and np.all(np.isfinite(p))
        assert math.hypot(p[0] - mu[0], p[1] - mu[1]) < 2.0
        assert abs(math.remainder(p[2] - mu[2], 2 * math.pi)) < 1.0


def test_eps_floor_is_needed_on_a_turn_in_place():
    """Why eps: the same turn in place without the floor.  The prior is then exactly singular, try_inverse fails and the reference's
    fallback (prior precision 1e-6, fs2.rs:205) throws the sample hundreds of metres from mu; with
    eps = 1e-8 every draw stays within 1 m.  The plain-Python restatement (tests/golden/make_fs_odom_golden.py, which the oracle
    reproduces bit for bit at eps = 1e-8) stands in for the model with its floor switched off."""
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden"))
    import make_fs_odom_golden as G
    m = G.increment([3.0, -2.0, 1.2, 3.0, -2.0, -1.5], [0.2] * 4)
    pose, lm = [1.0, 2.0, 0.3], [6.0, 4.0, 1.5, 0.1, 0.1, 2.0]
    dist = {}
    try:
        for eps in (1e-8, 0.0):
            G.EPS = eps
            mu, cov = G.prior(m, pose)
            dx, dy = lm[0] - mu[0], lm[1] - mu[1]
            z = [math.hypot(dx, dy), math.atan2(dy, dx) - mu[2]]
            rng = np.random.default_rng(3)
            dist[eps] = [math.hypot(p[0] - mu[0], p[1] - mu[1]) for p in (G.pose2(m, pose, lm, z, rng.standard_normal(3))[1] for _ in range(50))]
            if eps == 0.0:
                assert G.inv33(cov) is None
    finally:
        G.EPS = 1e-8
    assert max(dist[1e-8]) < 1.0
    assert np.median(dist[0.0]) > 100.0


def test_refusals():
    assert F.increment([0, 0, float("nan")], [1, 0, 0]) is None
    assert F.increment([0, 0, 0], [1, 0, 0], alpha=(-0.1, 0, 0, 0)) is None
