"""CPU tests of the pose-hypothesis contract (include/pfgpu.h pfgpu_pf_hypotheses, DESIGN §3.10) on its numpy restatement
(tests/_cluster_oracle.py):
  - the components of the restatement (scipy connected_components over listed pairs) equal a plain-Python BFS on random clouds;
  - hand-checked cases: bin edges and -0.0, yaw at +-pi, multiples of 2 pi and |yaw| ~ 1e3, a cluster across the yaw seam,
    saturated keys, non-members, yaw_bins 1 and 2;
  - behaviour, with the lfield oracle's Philox draws: on the point-symmetric floor plan, a cloud started as two blobs at the truth
    and at its mirror keeps both after 30 scan steps, and the two heaviest hypotheses find them where the weighted estimate does
    not."""
import math
import os

import numpy as np
import pytest

import _cluster_oracle as O
import _lfield_oracle as LF
from rust_robotics_b200 import scenarios

SYM_START = (-14.0, -8.0, 0.3)        # clear of the mirrored obstacles, and more than 4 m from the centre all the way


def cloud(rows):
    return np.array(rows, dtype=np.float64).reshape(-1, 5)


@pytest.mark.parametrize("seed", range(8))
def test_components_match_bfs(seed):
    rng = np.random.default_rng(seed)
    n = [1, 2, 50, 300, 1000, 1500, 2000, 800][seed]
    p = np.zeros((n, 5))
    p[:, 0], p[:, 1] = rng.normal(0.0, 1.0 + seed, n), rng.normal(0.0, 1.0 + seed, n)
    p[:, 2] = rng.uniform(-10.0, 10.0, n)
    p[:, 3] = rng.normal(1.0, 0.1, n)
    p[:, 4] = rng.random(n)
    p[rng.random(n) < 0.05, 4] = 0.0
    K = [24, 1, 2, 36, 24, 7, 24, 3][seed]
    res = [0.5, 0.5, 0.3, 0.5, 0.25, 1.0, 0.5, 0.1][seed]
    hs, rank = O.hypotheses(p, res, K)
    bfs = O.bfs_components(p, res, K)
    assert sorted(h.label for h in hs) == sorted(bfs)
    for r, h in enumerate(hs):
        assert np.flatnonzero(rank == r).tolist() == bfs[h.label]
        assert h.count == len(bfs[h.label]) and h.label == bfs[h.label][0]
    assert (rank < 0).sum() == n - sum(h.count for h in hs)
    masses = [h.mass for h in hs]
    assert all(a > b or (a == b and hs[i].label < hs[i + 1].label) for i, (a, b) in enumerate(zip(masses, masses[1:])))


def test_bin_edges_and_negative_zero():
    p = cloud([[0.5, 0.0, 0.0, 0.0, 1.0], [-0.0, -0.0, -0.0, 0.0, 1.0], [-1e-300, 0.49999999999999994, 0.0, 0.0, 1.0]])
    k = O.bin_keys(p, 0.5, 24)
    assert k.tolist() == [[1, 0, 0], [0, 0, 0], [-1, 0, 0]]
    hs, _ = O.hypotheses(p, 0.5, 24)
    assert len(hs) == 1 and hs[0].bins == 3 and hs[0].label == 0          # adjacent bins: one cluster


def test_yaw_bins_of_special_angles():
    T = O.TWO_PI
    yaws = [math.pi, -math.pi, T, -T, 2 * T, 1e3, -1e3, -1e-300, 3 * math.pi]
    k = O.bin_keys(cloud([[0.0, 0.0, y, 0.0, 1.0] for y in yaws]), 0.5, 24)[:, 2]
    assert k[0] == 12 and k[1] == 12                                     # +-pi: the same bin, half way round
    assert k[2] == 0 and k[3] == 0 and k[4] == 0
    th = 1e3 - T * math.floor(1e3 / T)
    assert k[5] == math.floor(th / (T / 24)) and 0 <= k[6] < 24
    assert k[7] == 23                                                    # theta rounds to T: clamped to K - 1
    assert k[8] == 12


def test_cluster_across_the_yaw_seam():
    p = cloud([[0.0, 0.0, math.pi - 0.05, 1.0, 1.0], [0.0, 0.0, -math.pi + 0.05, 1.0, 1.0], [0.0, 0.0, 0.0, 1.0, 1.0]])
    hs, rank = O.hypotheses(p, 0.5, 24)
    assert len(hs) == 2 and rank.tolist() == [0, 0, 1]
    seam = hs[0]
    assert seam.count == 2 and seam.bins == 2 and abs(abs(seam.mean[2]) - math.pi) < 1e-12
    assert abs(seam.cov[2, 2] - 0.05 ** 2) < 1e-12                       # wrapped deviations, not 2 pi - 0.1


def test_saturated_keys():
    p = cloud([[1e12, 0.0, 0.0, 0.0, 1.0], [1e12 - 1.0, 0.0, 0.0, 0.0, 1.0], [-1e12, 5.0, 0.0, 0.0, 1.0], [3e9, 0.0, 0.0, 0.0, 2.0]])
    k = O.bin_keys(p, 0.5, 24)
    assert k[:, 0].tolist() == [2 ** 31 - 1, 2 ** 31 - 1, -2 ** 31, 2 ** 31 - 1]
    hs, rank = O.hypotheses(p, 0.5, 24)
    assert [h.count for h in hs] == [3, 1] and rank.tolist() == [0, 0, 1, 0]     # saturation merges the far ones into one bin


def test_non_members():
    p = cloud([[np.nan, 0, 0, 0, 1], [0, np.inf, 0, 0, 1], [0, 0, -np.inf, 0, 1], [0, 0, 0, np.nan, 1], [0, 0, 0, 0, 0.0],
               [0, 0, 0, 0, -1.0], [0, 0, 0, 0, np.nan], [0, 0, 0, 0, np.inf], [0.1, 0.1, 0.1, 0.0, 0.25]])
    hs, rank = O.hypotheses(p, 0.5, 24)
    assert rank.tolist() == [-1] * 8 + [0] and len(hs) == 1 and hs[0].label == 8 and hs[0].mass == 0.25
    assert np.all(np.abs(hs[0].cov) < 1e-30)                             # a single pose: no spread (atan2 rounds the yaw)
    assert O.hypotheses(p[:8], 0.5, 24)[0] == []


@pytest.mark.parametrize("K", [1, 2])
def test_few_yaw_bins(K):
    p = cloud([[0.0, 0.0, y, 0.0, 1.0] for y in (0.0, 1.0, 2.0, 3.0, -1.0, -2.0)] + [[5.0, 0.0, 0.0, 0.0, 1.0]])
    hs, _ = O.hypotheses(p, 0.5, K)
    assert [h.count for h in hs] == [6, 1] and hs[0].bins == K
    assert O.bfs_components(p, 0.5, K)[0] == list(range(6))


def symmetric_blobs(sc, n, seed):
    """n particles, half around the start pose, half around its mirror (sigma 0.1 m, 0.05 rad), v = 1, w = 1/n"""
    rng = np.random.default_rng(seed)
    x0, y0, a0 = sc.start
    p = np.zeros((n, 5))
    h = n // 2
    p[:h, 0], p[:h, 1], p[:h, 2] = x0, y0, a0
    p[h:, 0], p[h:, 1], p[h:, 2] = -x0, -y0, a0 + math.pi
    p[:, 0] += rng.normal(0.0, 0.1, n)
    p[:, 1] += rng.normal(0.0, 0.1, n)
    p[:, 2] += rng.normal(0.0, 0.05, n)
    p[:, 3], p[:, 4] = 1.0, 1.0 / n
    return p


def two_mode_outcome(sc, t, hs, est):
    """(errors of the two heaviest hypotheses against the truth and its mirror, their masses, estimate distances)"""
    x, y, a = sc.truth[t]
    mirror = (-x, -y, a + math.pi)

    def err(h, q):
        return math.hypot(h.mean[0] - q[0], h.mean[1] - q[1]), abs(scenarios.normalize_angle(h.mean[2] - q[2]))
    top = hs[:2]
    near = [min(top, key=lambda h: err(h, q)[0]) for q in ((x, y, a), mirror)]
    errs = [err(near[0], (x, y, a)), err(near[1], mirror)]
    return errs, [h.mass for h in near], near[0] is not near[1], (math.hypot(est[0] - x, est[1] - y), math.hypot(est[0] + x, est[1] + y))


def test_symmetric_plan_two_blobs_oracle():
    sc = scenarios.ScanScenario(steps=30, start=SYM_START, symmetric=True)
    assert math.hypot(*SYM_START[:2]) >= 4.0
    n = 1 << 14
    o = LF.OracleLField(n, mode=1, max_particles=n, range_noise=0.25, velocity_noise=0.2, yaw_rate_noise=0.1, seed=3,
                        threads=min(8, os.cpu_count() or 1))
    assert o.set_map(sc.obstacles, sc.RES) == 0
    o.upload(symmetric_blobs(sc, n, 3))
    for t in range(30):
        est, _ = o.step_scan(sc.controls[t], *sc.scan_args(t))
    hs, _ = O.hypotheses(o.particles())
    errs, masses, distinct, est_d = two_mode_outcome(sc, 29, hs, est)
    assert distinct and all(e[0] < 0.5 and e[1] < 0.1 for e in errs), errs
    assert all(0.4 <= m <= 0.6 for m in masses), masses
    assert min(est_d) > 3.0, est_d
