"""Grid-based FastSLAM on the device (DESIGN §3.16) against the contract-math oracle (tests/host/gs_oracle.c), bit for bit: OdomScenario
at 0.1 m with N = 64 (R = 1, 0, 2, and a run that never resamples), the grid copies of every resample, the edges and refusals of the
step contract, the hand-off of a particle's grid to OccupancyGridMap and the models that take one, and the filter's behaviour at
5 cm and N = 1024 against dead reckoning."""
import math
import os
import subprocess

import numpy as np
import pytest

import _gs_oracle as GO
import rust_robotics_b200 as rr
from rust_robotics_b200 import scenarios

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def bits(a):
    return np.ascontiguousarray(a, dtype=np.float64).view(np.uint64)


@pytest.fixture(scope="module")
def sc():
    return scenarios.OdomScenario()


def coarse(sc, res=0.1):
    W, H = sc.obstacles.shape
    return dict(resolution=res, width=int(round(W * sc.RES / res)), height=int(round(H * sc.RES / res)))


def pair(sc, n, seed=5, nth=None, ogm=None, **model):
    g = rr.GridFastSlam(rr.GridFastSlamConfig(rr.OccupancyGridConfig(**ogm), n_particles=n, nth=nth, **model), start_pose=sc.start,
                        seed=seed)
    o = GO.OracleGs(n, sc.start, seed=seed, nth=nth, ogm=ogm, **model)
    return g, o


def same_state(g, o, grids=False):
    assert np.array_equal(bits(g.particles()), bits(o.particles())), "poses differ from the oracle"
    assert np.array_equal(bits(g.weights()), bits(o.weights())), "weights differ from the oracle"
    assert np.array_equal(g.last_indices(), o.last_indices()), "ancestors differ from the oracle"
    s, i = g.stats(), o.info()
    assert (s.steps, s.resampled, s.copies, s.events) == (i.steps, i.resampled, i.copies, i.events)
    assert bits([s.neff])[0] == bits([i.neff])[0]
    if grids:
        for k in range(g.n):
            assert np.array_equal(bits(g.grid(k)), bits(o.grid(k))), f"slot {k}'s grid differs from the oracle"


def run(sc, g, o, check_grids_at=()):
    res = []
    for t in range(sc.steps):
        prev, cur = sc.odom_pair(t)
        g.step(prev, cur, sc.scans[t], sc.ANGLE_MIN, sc.ANGLE_INC)
        did = o.step(prev, cur, sc.scans[t], sc.ANGLE_MIN, sc.ANGLE_INC)
        same_state(g, o, grids=t in check_grids_at or t == sc.steps - 1)
        if did:
            s = g.stats()
            assert s.copies == g.n - len(set(g.last_indices().tolist()))
        res.append(did)
    return res


@pytest.mark.parametrize("R", [1, 0, 2])
def test_odom_scenario_bits(sc, R):
    g, o = pair(sc, 64, ogm=coarse(sc), search_radius=R)
    did = run(sc, g, o, check_grids_at=(10, 40))
    assert any(did) and not all(did)


def test_never_resamples(sc):
    g, o = pair(sc, 64, nth=0.0, ogm=coarse(sc))
    assert not any(run(sc, g, o, check_grids_at=(20,)))


def test_every_step_resamples_with_copies(sc):
    g, o = pair(sc, 64, nth=math.inf, ogm=coarse(sc))
    copies = []
    for t in range(12):
        prev, cur = sc.odom_pair(t)
        g.step(prev, cur, sc.scans[t], sc.ANGLE_MIN, sc.ANGLE_INC)
        assert o.step(prev, cur, sc.scans[t], sc.ANGLE_MIN, sc.ANGLE_INC)
        same_state(g, o, grids=t in (3, 11))
        copies.append(g.stats().copies)
    assert max(copies) > 0


SMALL = dict(resolution=0.5, width=24, height=20)


def small_pair(n=16, nth=None, start=(0.3, -0.2, 0.4), **model):
    g = rr.GridFastSlam(rr.GridFastSlamConfig(rr.OccupancyGridConfig(**SMALL), n_particles=n, nth=nth, **model), start_pose=start, seed=9)
    o = GO.OracleGs(n, start, seed=9, nth=nth, ogm=SMALL, **model)
    return g, o


def both(g, o, odom, ranges, amin=-math.pi, ainc=None):
    ainc = 2.0 * math.pi / len(ranges) if ainc is None else ainc
    g.step(odom[:3], odom[3:], ranges, amin, ainc)
    return o.step(odom[:3], odom[3:], ranges, amin, ainc)


def test_edges():
    rng = np.random.default_rng(4)
    # a map first, then the edges on it
    g, o = small_pair(nth=8.0)
    for t in range(4):
        both(g, o, (0.1 * t, 0, 0, 0.1 * t + 0.1, 0.02, 0.05), rng.uniform(1, 6, 40))
    same_state(g, o, grids=True)
    # equal odometry poses move nothing (a resample only reorders the poses)
    p0 = g.particles()
    both(g, o, (1, 1, 0.2, 1, 1, 0.2), rng.uniform(1, 6, 40))
    idx = g.last_indices()
    assert np.array_equal(bits(g.particles()), bits(p0[idx] if idx.size else p0))
    same_state(g, o, grids=True)
    # every range unusable: w_raw = 1 and no fuse events
    both(g, o, (1, 1, 0.2, 1, 1, 0.2), np.array([np.inf, np.nan, 0.0, -1.0] * 10))
    assert g.stats().events == 0 and o.info().used == 0
    same_state(g, o, grids=True)
    # endpoints on the grid border with R = 2: ranges that end at and past the walls of the 12 m x 10 m grid
    g2, o2 = small_pair(nth=8.0, search_radius=2, start=(0.0, 0.0, 0.0))
    for t in range(3):
        both(g2, o2, (0, 0, 0, 0.05, 0, 0.01), np.full(64, 5.0 + 0.5 * t) + rng.uniform(-0.3, 0.3, 64))
    same_state(g2, o2, grids=True)


def test_pose_outside_grid():
    g, o = small_pair(start=(40.0, 0.0, 0.0))
    both(g, o, (0, 0, 0, 0.1, 0, 0), np.full(30, 2.0))
    assert g.stats().events == 0
    assert np.all(g.grid(0) == 0.0)
    same_state(g, o, grids=True)


def test_exactly_L_beams_and_more():
    g, o = small_pair(max_beams=4096)
    L = g.max_used_beams()
    both(g, o, (0, 0, 0, 0.1, 0, 0), np.full(L, 3.0), ainc=0.01)
    assert o.info().used == L
    same_state(g, o, grids=True)
    with pytest.raises(rr.InvalidParameter):
        g.step((0, 0, 0), (0.1, 0, 0), np.full(L + 1, 3.0), -math.pi, 0.01)
    assert o.step((0, 0, 0), (0.1, 0, 0), np.full(L + 1, 3.0), -math.pi, 0.01) is None
    assert g.stats().steps == 1


def test_refusals(sc):
    cfg = rr.OccupancyGridConfig(**SMALL)
    for bad in (dict(z_rand=0.0), dict(max_range=-1.0), dict(max_beams=1), dict(search_radius=9), dict(z_hit=math.nan),
                dict(nth=math.nan), dict(n_particles=0)):
        with pytest.raises(rr.InvalidParameter):
            rr.GridFastSlam(rr.GridFastSlamConfig(cfg, **dict(dict(n_particles=4), **bad)))
    with pytest.raises(rr.InvalidParameter):
        rr.GridFastSlam(rr.GridFastSlamConfig(rr.OccupancyGridConfig(resolution=0.0, width=4, height=4), n_particles=4))
    g = rr.GridFastSlam(rr.GridFastSlamConfig(cfg, n_particles=4))
    for odom in ((math.nan, 0, 0), (0, math.inf, 0)):
        with pytest.raises(rr.InvalidParameter):
            g.step(odom, (0, 0, 0), np.ones(8), 0.0, 0.1)
    with pytest.raises(rr.InvalidParameter):
        g.step((0, 0, 0), (0, 0, 0), np.ones(8), math.nan, 0.1)
    with pytest.raises(rr.InvalidParameter):
        g.set_odometry_noise((0.1, -0.1, 0.1, 0.1))
    g.set_odometry_noise((0.1, 0.2, 0.3, 0.4))
    assert g.odometry_noise() == (0.1, 0.2, 0.3, 0.4)
    assert g.stats().steps == 0
    other = rr.OccupancyGridMap(rr.OccupancyGridConfig(resolution=0.5, width=24, height=21))
    with pytest.raises(rr.InvalidParameter):
        g.copy_grid_to(0, other)
    with pytest.raises(rr.InvalidParameter):
        g.copy_grid_to(4, rr.OccupancyGridMap(cfg))
    # grids that cannot fit: 2^20 particles of 2^28 cells
    with pytest.raises(rr.InvalidParameter) as e:
        rr.GridFastSlam(rr.GridFastSlamConfig(rr.OccupancyGridConfig(resolution=0.05, width=16384, height=16384), n_particles=1 << 20))
    assert "not supported" in str(e.value)
    g.step((0, 0, 0), (0.1, 0, 0), np.ones(8), 0.0, 0.1)        # still usable
    g.sync()


def test_hand_off(sc):
    ogm = coarse(sc)
    g, _ = pair(sc, 32, ogm=ogm)
    for t in range(20):
        prev, cur = sc.odom_pair(t)
        g.step(prev, cur, sc.scans[t], sc.ANGLE_MIN, sc.ANGLE_INC)
    b, pose = g.best()
    w = g.weights()
    assert b == int(np.argmax(w))
    m = rr.OccupancyGridMap(rr.OccupancyGridConfig(**ogm))
    g.copy_grid_to(b, m)
    assert np.array_equal(bits(m.grid), bits(g.grid(b)))
    csm = rr.CorrelativeScanMatcher()
    csm.set_reference_from_grid(m, 0.5)
    mcl = rr.MonteCarloLocalizer(rr.MonteCarloLocalizationConfig(1024, 1024), seed=1)
    mcl.set_beam_model_from_grid(m, 0.5)


def dead_reckoning(sc, t):
    """the odometry of step t composed onto the start pose (odom[0] is the origin of the odometry frame)"""
    sx, sy, sa = sc.start
    ox, oy, oa = sc.odom[t + 1]
    return (sx + math.cos(sa) * ox - math.sin(sa) * oy, sy + math.sin(sa) * ox + math.cos(sa) * oy, sa + oa)


def near_path(sc, W, H, res, radius=10.0):
    xs = (np.arange(W) + 0.5 - W / 2.0) * res
    ys = (np.arange(H) + 0.5 - H / 2.0) * res
    X, Y = np.meshgrid(xs, ys, indexing="ij")
    m = np.zeros((W, H), dtype=bool)
    for x, y, _ in sc.truth:
        m |= (X - x) ** 2 + (Y - y) ** 2 <= radius * radius
    return m


def map_scores(mask, plan, region):
    """(agreement over the region, obstacle IoU over the region) of an obstacle mask against the plan"""
    a, b = mask[region], plan[region]
    return float(np.mean(a == b)), float(np.sum(a & b) / max(1, np.sum(a | b)))


def behaviour(sc, n=1024, seed=3):
    W, H = sc.obstacles.shape
    cfg = rr.OccupancyGridConfig(resolution=sc.RES, width=W, height=H)
    g = rr.GridFastSlam(rr.GridFastSlamConfig(cfg, n_particles=n), start_pose=sc.start, seed=seed)
    for t in range(sc.steps):
        prev, cur = sc.odom_pair(t)
        g.step(prev, cur, sc.scans[t], sc.ANGLE_MIN, sc.ANGLE_INC)
    b, pose = g.best()
    dr = [dead_reckoning(sc, t) for t in range(sc.steps)]
    m = rr.OccupancyGridMap(cfg)
    m.update_with_scans(dr, np.stack(sc.scans), sc.ANGLE_MIN, sc.ANGLE_INC)
    region = near_path(sc, W, H, sc.RES)
    truth = sc.truth[-1]
    best_map = rr.obstacles_from_log_odds(g.grid(b), 0.5)
    return dict(err_filter=math.hypot(pose[0] - truth[0], pose[1] - truth[1]), err_dr=math.hypot(dr[-1][0] - truth[0], dr[-1][1] - truth[1]),
                map_filter=map_scores(best_map, sc.obstacles, region), map_dr=map_scores(m.obstacles(0.5), sc.obstacles, region))


def test_behaviour_against_dead_reckoning(sc):
    """OdomScenario at 5 cm, N = 1024: the best particle ends closer to the truth than dead reckoning and its map (obstacle mask at
    0.5, cells within 10 m of the truth path) agrees better with the plan than the map fused at the dead-reckoning poses.  Measured
    on an H100 (DESIGN §3.16): 0.022 m against 0.087 m; agreement 0.985 against 0.977, obstacle IoU 0.378 against 0.169."""
    r = behaviour(sc)
    print("grid FastSLAM behaviour:", r)
    assert r["err_filter"] < 0.5 * r["err_dr"]
    assert r["map_filter"][0] > r["map_dr"][0]
    assert r["map_filter"][1] > 1.5 * r["map_dr"][1]


def test_cpp_mirror(tmp_path):
    """host/gslam_check.cpp through the C++ mirror: the oracle's poses, weights, ancestors, stats and best grid, bit for bit"""
    pkg, exe = os.path.join(ROOT, "rust_robotics_b200"), str(tmp_path / "gslam_check")
    subprocess.run(["/usr/bin/g++", "-std=c++17", "-O1", os.path.join(pkg, "host", "gslam_check.cpp"), "-I", os.path.join(ROOT, "include"),
                    "-I", os.path.join(pkg, "host"), "-L", pkg, "-lpfgpu", f"-Wl,-rpath,{pkg}", "-o", exe], check=True)
    r = subprocess.run([exe], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr
    lines = r.stdout.split("\n")
    o = GO.OracleGs(16, (0.2, -0.1, 0.3), seed=11, nth=12.0, ogm=dict(resolution=0.1, width=120, height=80))
    ranges = np.array([0.5 + 0.1 * ((i * 7) % 50) for i in range(90)])
    ranges[5] = np.inf
    for t in range(6):
        o.step((0.1 * t, 0.0, 0.02 * t), (0.1 * t + 0.1, 0.01, 0.02 * t + 0.02), ranges, -math.pi, 2.0 * math.pi / 90.0)
    hexes = [np.array([float.fromhex(x) for x in lines[k].split()]) for k in (0, 1, 4)]
    assert np.array_equal(bits(hexes[0]), bits(o.particles().ravel()))
    assert np.array_equal(bits(hexes[1]), bits(o.weights()))
    assert [int(x) for x in lines[2].split()] == o.last_indices().tolist()
    i = o.info()
    assert [int(x) for x in lines[3].split()] == [int(i.resampled), i.copies, i.events]
    w = o.weights()
    assert np.array_equal(bits(hexes[2]), bits(o.grid(int(np.argmax(w))).ravel()))
    assert lines[5].strip() == "1"
