"""pfgpu_fs_estimate_merge (host only, no GPU): moments of several ranks' particles, formed here in numpy the way
pfgpu_fs_moments defines them, merged in rank order and finalised = the numpy restatement of the estimate over all particles."""
import math

import numpy as np
import pytest

import rust_robotics_b200 as rr
from test_gpu_estimate import _wrap, check, ref_estimate


def _moments(pw, lm, c, cov00_max):
    pm = rr.api._FsPoseMoments()
    w = pw[:, 0]
    d = np.stack([pw[:, 1] - c[0], pw[:, 2] - c[1], _wrap(pw[:, 3] - c[2])], axis=1)
    pm.w = w.sum()
    pm.c[:] = list(c)
    mean = (w[:, None] * d).sum(axis=0) / pm.w if pm.w else np.zeros(3)
    pm.mean[:] = list(mean)
    m2 = np.einsum("i,ij,ik->jk", w, d - mean, d - mean)
    pm.m2[:] = [m2[0, 0], m2[0, 1], m2[0, 2], m2[1, 1], m2[1, 2], m2[2, 2]]
    out = np.zeros((lm.shape[1], 7))
    for l in range(lm.shape[1]):
        sel = lm[:, l, 2] < cov00_max
        ws = w[sel]
        if ws.sum() == 0:
            continue
        mu = lm[sel, l, :2]
        mean = (ws[:, None] * mu).sum(axis=0) / ws.sum()
        e = mu - mean
        m2 = (ws[:, None] * lm[sel, l, 2:6]).sum(axis=0) + (ws[:, None] * np.stack([e[:, 0] * e[:, 0], e[:, 0] * e[:, 1], e[:, 0] * e[:, 1], e[:, 1] * e[:, 1]], axis=1)).sum(axis=0)
        out[l] = [ws.sum(), mean[0], mean[1], *m2]
    return pm, out


@pytest.mark.parametrize("cov00_max", [100.0, math.inf, 0.0])
@pytest.mark.parametrize("world", [1, 3])
def test_merge_equals_definition(cov00_max, world):
    rng = np.random.default_rng(world)
    n, m = 600, 7
    pw = np.stack([rng.uniform(0.0, 1.0, n), rng.normal(5.0, 2.0, n), rng.normal(-3.0, 1.0, n), _wrap(3.1 + rng.normal(0.0, 0.1, n))], axis=1)
    lm = np.concatenate([rng.normal(10.0, 1.0, (n, m, 2)), rng.uniform(0.0, 200.0, (n, m, 1)), rng.normal(0.0, 0.1, (n, m, 2)),
                         rng.uniform(0.5, 2.0, (n, m, 1))], axis=2)
    lm[:, 3, 2] = 500.0                                    # one landmark nobody passes at the default filter
    c = pw[-1, 1:4]
    est = rr.FastSlam1.merge_moments([_moments(p, l, c, cov00_max) for p, l in zip(np.array_split(pw, world), np.array_split(lm, world))])
    check(est, ref_estimate(pw, lm, c, cov00_max), f"world {world}")
    assert abs(abs(est.pose[2]) - math.pi) < 0.1


def test_merge_degenerate_and_invalid():
    pw = np.zeros((4, 4))
    lm = np.zeros((4, 2, 6))
    est = rr.FastSlam1.merge_moments([_moments(pw, lm, pw[-1, 1:4], 100.0)])
    assert np.isnan(est.pose).all() and np.isnan(est.pose_cov).all() and np.all(est.mass == 0.0) and np.isnan(est.mean).all()
    a, b = _moments(pw, lm, [0.0, 0.0, 0.0], 100.0), _moments(pw, lm, [1.0, 0.0, 0.0], 100.0)
    with pytest.raises(rr.InvalidParameter):          # moments about different centres
        rr.FastSlam1.merge_moments([a, b])
    pose_only = rr.FastSlam1.merge_moments([(a[0], None)])
    assert pose_only.mass is None
