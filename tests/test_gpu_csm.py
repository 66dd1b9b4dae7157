"""Correlative scan matching on the device (DESIGN §3.13) against the contract-math oracle (tests/host/csm_oracle.c), bit for bit: x,
y, yaw and score bits and converged of every result, and the lookup table's extent and every cell.  Golden cases, random clouds,
ScanScenario scans against the floor plan from host points and from the device grid, batches with uneven and invalid members, point
counts across the workspace chunks, a relocalisation-sized window in yaw chunks, resolution changes, repeated calls, refusals, the
C++ mirror, and scan-matched mapping on the device that reproduces the oracle loop and then localises with the beam model."""
import ctypes as C
import math
import os
import subprocess

import numpy as np
import pytest

import _csm_oracle as CO
import _ogm_oracle as OO
import rust_robotics_b200 as rr
from rust_robotics_b200 import api, scenarios
from test_csm_oracle import CASES, FX, FY, case_args, run_oracle_mapping

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def sc():
    return scenarios.ScanScenario()


def cfg_of(d):
    return rr.CorrelativeScanMatcherConfig(**dict(CO.DEFAULTS, **d))


def bits(v):
    return np.array(v, dtype=np.float64).view(np.uint64)


def assert_same(got, want, what=""):
    """a device ScanMatchResult against an oracle tuple, bit for bit"""
    assert np.array_equal(bits([got.x, got.y, got.yaw, got.score]), bits(want[:4])) and got.converged == want[4], (what, got, want)


def assert_table(m, rx, ry, res):
    """the device table for res equals the oracle's HashMap: same extent (the reference cells' box grown by R), same cells"""
    want, R = CO.table(rx, ry, res)
    t, (ox, oy), r = m.lookup_table(res)
    assert r == R
    if not len(rx):
        assert t.size == 0
        return
    cx = [int(v) for v in np.sign(np.asarray(rx) / res) * np.floor(np.abs(np.asarray(rx) / res) + 0.5)]
    cy = [int(v) for v in np.sign(np.asarray(ry) / res) * np.floor(np.abs(np.asarray(ry) / res) + 0.5)]
    assert (ox, oy) == (min(cx) - R, min(cy) - R) and t.shape == (max(cx) - min(cx) + 2 * R + 1, max(cy) - min(cy) + 2 * R + 1)
    nz = np.argwhere(t != 0.0)
    assert len(nz) == len(want)
    keys = np.array(sorted(want))
    got = t[keys[:, 0] - ox, keys[:, 1] - oy]
    assert np.array_equal(bits(got), bits([want[tuple(k)] for k in keys]))


@pytest.mark.parametrize("case", CASES, ids=[c["name"] for c in CASES])
def test_golden_cases_match_oracle(case):
    rx, ry, qx, qy, pose, cfg = case_args(case)
    m = rr.CorrelativeScanMatcher()
    m.set_reference(rx, ry)
    assert_same(m.match(qx, qy, pose, cfg_of(cfg)), CO.match(rx, ry, qx, qy, pose, cfg))
    if cfg["grid_resolution"] > 0.0:
        assert_table(m, rx, ry, cfg["grid_resolution"])
    # the module-level function with the reference's signature
    assert_same(rr.correlative_scan_match(rx, ry, qx, qy, pose, cfg_of(cfg)), CO.match(rx, ry, qx, qy, pose, cfg))


@pytest.mark.parametrize("seed", range(6))
def test_random_clouds(seed):
    rng = np.random.default_rng(seed)
    n = int(rng.integers(1, 400))
    rx, ry = rng.uniform(-5.0, 5.0, n), rng.uniform(-5.0, 5.0, n)
    k = int(rng.integers(1, min(n, 120) + 1))
    pose = (rng.normal(0.0, 0.2), rng.normal(0.0, 0.2), rng.normal(0.0, 0.1))
    sel = rng.choice(n, k, replace=False)
    qx, qy = rx[sel] + rng.normal(0.0, 0.03, k), ry[sel] + rng.normal(0.0, 0.03, k)
    res = [0.05, 0.1, 0.25, 0.02, 0.07, 0.5][seed]
    cfg = dict(linear_search_range=0.3, angular_search_range=0.1, linear_step=0.05, angular_step=0.01, grid_resolution=res)
    m = rr.CorrelativeScanMatcher()
    m.set_reference(rx, ry)
    assert_same(m.match(qx, qy, pose, cfg_of(cfg)), CO.match(rx, ry, qx, qy, pose, cfg))
    assert_table(m, rx, ry, res)


def plan_points(sc):
    return CO.grid_points(sc.obstacles, sc.RES)


def test_scans_against_the_plan_host_points_and_grid(sc):
    """ScanScenario's scans from noisy poses against the plan: the table from host points, and from a device grid whose obstacle
    cells are the plan's, give the same table and the same results"""
    rx, ry = plan_points(sc)
    a = rr.CorrelativeScanMatcher()
    a.set_reference(rx, ry)
    W, H = sc.obstacles.shape
    g = rr.OccupancyGridMap(rr.OccupancyGridConfig(resolution=sc.RES, width=W, height=H))
    g.set_grid(np.where(sc.obstacles, 2.0, -2.0))
    b = rr.CorrelativeScanMatcher()
    b.set_reference_from_grid(g, 0.5)
    assert b.reference_size == rx.size
    ta, ta0, _ = a.lookup_table(0.05)
    tb, tb0, _ = b.lookup_table(0.05)
    assert ta0 == tb0 and np.array_equal(bits(ta), bits(tb))
    assert_table(a, rx, ry, 0.05)
    rng = np.random.default_rng(2)
    cfg = dict(linear_search_range=0.3, angular_search_range=0.06, linear_step=0.05, angular_step=0.01, grid_resolution=0.05)
    for t in (0, 17, 41):
        qx, qy = CO.scan_points(sc.scans[t], sc.ANGLE_MIN, sc.ANGLE_INC)
        pose = np.array(sc.truth[t]) + rng.normal(0.0, 1.0, 3) * [0.1, 0.1, 0.03]
        want = CO.match(rx, ry, qx, qy, pose, cfg)
        assert_same(a.match(qx, qy, pose, cfg_of(cfg)), want, t)
        assert_same(b.match(qx, qy, pose, cfg_of(cfg)), want, t)
        assert math.hypot(want[0] - sc.truth[t][0], want[1] - sc.truth[t][1]) < 0.1


@pytest.mark.parametrize("Q", [1, 7, 60, 1000])
def test_batches(sc, Q):
    """Q queries with uneven point counts, some empty (the invalid result); each equals its own oracle call"""
    rx, ry = plan_points(sc)
    m = rr.CorrelativeScanMatcher()
    m.set_reference(rx, ry)
    rng = np.random.default_rng(Q)
    cfg = (dict(linear_search_range=0.2, angular_search_range=0.04, linear_step=0.05, angular_step=0.01, grid_resolution=0.05) if Q < 1000
           else dict(linear_search_range=0.1, angular_search_range=0.02, linear_step=0.05, angular_step=0.01, grid_resolution=0.05))
    qxs, qys, poses = [], [], []
    for q in range(Q):
        t = int(rng.integers(0, len(sc.scans)))
        x, y = CO.scan_points(sc.scans[t], sc.ANGLE_MIN, sc.ANGLE_INC)
        n = 0 if (Q > 1 and q % 5 == 3) else int(rng.integers(1, x.size + 1))
        sel = np.sort(rng.choice(x.size, n, replace=False))
        qxs.append(x[sel]), qys.append(y[sel])
        poses.append(np.array(sc.truth[t]) + rng.normal(0.0, 1.0, 3) * [0.05, 0.05, 0.01])
    got = m.match(qxs, qys, np.array(poses), cfg_of(cfg))
    assert len(got) == Q
    for q in range(Q):
        assert_same(got[q], CO.match(rx, ry, qxs[q], qys[q], poses[q], cfg), q)
    # the batch equals one call per query
    for q in range(0, Q, max(1, Q // 7)):
        assert_same(m.match(qxs[q], qys[q], poses[q], cfg_of(cfg)), CO.match(rx, ry, qxs[q], qys[q], poses[q], cfg), q)


@pytest.mark.parametrize("ws", [None, "200000", "600000"])
def test_point_counts_across_chunks(sc, monkeypatch, ws):
    """1 .. 3000 query points, with the default workspace and with small ones that split queries into groups and yaws into chunks"""
    if ws:
        monkeypatch.setenv("PFGPU_CSM_WS_CAP", ws)
    rx, ry = plan_points(sc)
    m = rr.CorrelativeScanMatcher()
    m.set_reference(rx, ry)
    rng = np.random.default_rng(11)
    cfg = dict(linear_search_range=0.15, angular_search_range=0.03, linear_step=0.05, angular_step=0.01, grid_resolution=0.05)
    counts = [1, 2, 31, 32, 33, 255, 256, 257, 1000, 3000]
    qxs = [rng.uniform(-19.0, 19.0, n) for n in counts]
    qys = [rng.uniform(-14.0, 14.0, n) for n in counts]
    poses = rng.normal(0.0, 0.1, (len(counts), 3))
    got = m.match(qxs, qys, poses, cfg_of(cfg))
    for q, n in enumerate(counts):
        assert_same(got[q], CO.match(rx, ry, qxs[q], qys[q], poses[q], cfg), n)


def test_relocalisation_window_in_yaw_chunks(sc, monkeypatch):
    """+-2 m at 2.5 cm and +-pi at 0.5 degrees (1.87e7 candidates) for a few points; the workspace forces yaw chunks"""
    monkeypatch.setenv("PFGPU_CSM_WS_CAP", "1000000")
    rx, ry = plan_points(sc)
    m = rr.CorrelativeScanMatcher()
    m.set_reference(rx, ry)
    x, y = CO.scan_points(sc.scans[30], sc.ANGLE_MIN, sc.ANGLE_INC)
    qx, qy = x[::60], y[::60]
    cfg = dict(linear_search_range=2.0, angular_search_range=math.pi, linear_step=0.025, angular_step=math.pi / 360.0, grid_resolution=0.05)
    pose = np.array(sc.truth[30]) + [1.3, -0.8, 2.0]
    want = CO.match(rx, ry, qx, qy, pose, cfg)
    assert want[5] == 161 * 161 * 721
    got = m.match(qx, qy, pose, cfg_of(cfg))
    assert_same(got, want)
    assert_same(m.match(qx, qy, pose, cfg_of(cfg)), want)


def test_resolution_change_and_repeat_calls():
    rng = np.random.default_rng(4)
    rx, ry = rng.uniform(-3.0, 3.0, 200), rng.uniform(-3.0, 3.0, 200)
    qx, qy = rx[:80] + 0.01, ry[:80] - 0.02
    m = rr.CorrelativeScanMatcher()
    m.set_reference(rx, ry)
    for res in (0.05, 0.25, 0.05, 0.1, 0.1):
        cfg = dict(linear_search_range=0.2, angular_search_range=0.04, linear_step=0.05, angular_step=0.02, grid_resolution=res)
        want = CO.match(rx, ry, qx, qy, (0.0, 0.0, 0.0), cfg)
        for _ in range(2):
            assert_same(m.match(qx, qy, (0.0, 0.0, 0.0), cfg_of(cfg)), want, res)
        assert_table(m, rx, ry, res)
    # a new reference replaces the table
    m.set_reference(rx[:50], ry[:50])
    assert_table(m, rx[:50], ry[:50], 0.1)


def raw_match(m, cfg, qx, qy, pose):
    """the C ABI's status of one query"""
    qx, qy, p = (np.ascontiguousarray(np.asarray(v, dtype=np.float64)) for v in (qx, qy, pose))
    off = np.array([0, qx.size], dtype=np.uint64)
    out = (api._CsmResult * 1)()
    return m.L.pfgpu_csm_match(m.h, C.byref(cfg._c()), api._dp(p), 1, api._dp(qx), api._dp(qy), off.ctypes.data_as(C.POINTER(C.c_uint64)),
                               out)


def test_refusals_and_usable_after_unsupported():
    m = rr.CorrelativeScanMatcher()
    with pytest.raises(rr.InvalidParameter):
        m.set_reference([0.0, np.nan], [0.0, 1.0])
    with pytest.raises(rr.InvalidParameter):
        m.set_reference([0.0, 1.0], [0.0])
    m.set_reference(FX, FY)
    for bad in (dict(linear_step=np.nan), dict(angular_search_range=np.inf), dict(grid_resolution=-np.inf)):
        with pytest.raises(rr.InvalidParameter):
            m.match(FX, FY, (0.0, 0.0, 0.0), cfg_of(bad))
    for pose in ((np.nan, 0.0, 0.0), (0.0, 0.0, np.inf)):
        with pytest.raises(rr.InvalidParameter):
            m.match(FX, FY, pose)
    with pytest.raises(rr.InvalidParameter):
        m.match([0.0, np.inf], [0.0, 0.0], (0.0, 0.0, 0.0))
    with pytest.raises(rr.InvalidParameter):
        m.match(FX, FY[:3], (0.0, 0.0, 0.0))
    # a reference cell beyond 2^30
    far = rr.CorrelativeScanMatcher()
    far.set_reference([0.0, 2.0 ** 31 * 0.05], [0.0, 0.0])
    assert raw_match(far, cfg_of({}), FX, FY, (0.0, 0.0, 0.0)) == -1
    # UNSUPPORTED: a table above the cap, a window above the candidate caps, a resolution outside [2^-500, 2^500]
    wide = rr.CorrelativeScanMatcher()
    wide.set_reference([-5000.0, 5000.0], [-5000.0, 5000.0])
    assert raw_match(wide, cfg_of({}), FX, FY, (0.0, 0.0, 0.0)) == -2
    for bad in (dict(linear_search_range=1e6), dict(angular_search_range=1e6, angular_step=1e-3), dict(grid_resolution=1e-160)):
        assert raw_match(m, cfg_of(bad), FX, FY, (0.0, 0.0, 0.0)) == -2, bad
    with pytest.raises(rr.InvalidParameter):
        m.match(FX, FY, (0.0, 0.0, 0.0), cfg_of(dict(linear_search_range=1e6)))
    # still usable, and the cheap refusals still give the reference's results
    want = CO.match(FX, FY, FX, FY, (0.0, 0.0, 0.0))
    for h in (m, wide):
        h.set_reference(FX, FY)
        assert_same(h.match(FX, FY, (0.0, 0.0, 0.0)), want)
    assert_same(m.match(FX, FY, (0.0, 0.0, 9.0), cfg_of(dict(grid_resolution=0.0))), (0.0, 0.0, 9.0, 0.0, False))
    assert m.match([], [], (1.0, 2.0, 3.0)) == rr.ScanMatchResult(1.0, 2.0, 3.0, 0.0, False)
    empty = rr.CorrelativeScanMatcher()
    assert empty.match(FX, FY, (1.0, 2.0, 3.0)) == rr.ScanMatchResult(1.0, 2.0, 3.0, 0.0, False)


def test_grid_refusals():
    g = rr.OccupancyGridMap(rr.OccupancyGridConfig(resolution=0.1, width=40, height=30))
    m = rr.CorrelativeScanMatcher()
    with pytest.raises(rr.InvalidParameter):
        m.set_reference_from_grid(g, np.nan)
    m.set_reference_from_grid(g, 0.5)                  # a prior grid: no obstacle, so every match is invalid
    assert m.reference_size == 0 and m.match(FX, FY, (0.0, 0.0, 5.0)) == rr.ScanMatchResult(0.0, 0.0, 5.0, 0.0, False)
    n = C.c_int()
    m.L.pfgpu_device_count(C.byref(n))
    if n.value < 2:
        pytest.skip("the wrong-device refusal needs two GPUs")
    other = rr.OccupancyGridMap(rr.OccupancyGridConfig(resolution=0.1, width=40, height=30), device=1)
    with pytest.raises(rr.InvalidParameter):
        m.set_reference_from_grid(other, 0.5)


def test_grid_is_copied_at_set_time(sc):
    W, H = sc.obstacles.shape
    g = rr.OccupancyGridMap(rr.OccupancyGridConfig(resolution=sc.RES, width=W, height=H))
    g.update_with_scans(sc.truth[:10], np.stack(sc.scans[:10]), sc.ANGLE_MIN, sc.ANGLE_INC)
    m = rr.CorrelativeScanMatcher()
    m.set_reference_from_grid(g, 0.5)
    before = m.lookup_table(0.05)[0].copy()
    g.update_with_scans(sc.truth[10:], np.stack(sc.scans[10:]), sc.ANGLE_MIN, sc.ANGLE_INC)
    m.lookup_table(0.1)
    assert np.array_equal(bits(m.lookup_table(0.05)[0]), bits(before))
    m.set_reference_from_grid(g, 0.5)
    assert m.lookup_table(0.05)[0].shape != before.shape or not np.array_equal(m.lookup_table(0.05)[0], before)


def test_scan_matched_mapping_on_the_device(sc):
    """the oracle loop (test_csm_oracle.py) with the device grid and matcher: the same trajectory and the same final grid, bit for
    bit; then the device map localises a robot globally with the beam model"""
    odom = CO.odometry(sc.truth)
    want_poses, want_scores, o = run_oracle_mapping(sc, odom)
    W, H = sc.obstacles.shape
    g = rr.OccupancyGridMap(rr.OccupancyGridConfig(resolution=sc.RES, width=W, height=H))
    m = rr.CorrelativeScanMatcher()
    cfg = cfg_of(CO.MAP_CFG)
    poses, scores = CO.scan_matched_mapping(
        sc, odom, lambda p, r: g.update_with_scan(p[0], p[1], p[2], r, sc.ANGLE_MIN, sc.ANGLE_INC),
        lambda: m.set_reference_from_grid(g, 0.5), lambda qx, qy, p: m.match(qx, qy, p, cfg))
    assert np.array_equal(bits(poses), bits(want_poses)) and np.array_equal(bits(scores), bits(want_scores))
    assert np.array_equal(bits(g.grid), bits(o.grid))
    n = 1 << 16
    f = rr.MonteCarloLocalizer.try_with_region(sc.REGION, rr.MonteCarloLocalizationConfig(n, n, 0.05, 2.326, 0.2, 0.2, 0.1, 0.1), seed=5)
    f.set_beam_model_from_grid(g, 0.5)
    f.enable_recovery(0.001, 0.1, sc.REGION)
    err = [sc.error(k, f.try_step_beam_scan(sc.controls[k], *sc.scan_args(k))) for k in range(len(sc.controls))]
    assert all(e[0] < 1.0 for e in err[10:]), [round(e[0], 2) for e in err]


def test_cpp_mirror_csm(tmp_path):
    """host/csm_check.cpp through the C++ mirror: the oracle's results, bit for bit"""
    pkg, exe = os.path.join(ROOT, "rust_robotics_b200"), str(tmp_path / "csm_check")
    subprocess.run(["/usr/bin/g++", "-std=c++17", "-O1", os.path.join(pkg, "host", "csm_check.cpp"), "-I", os.path.join(ROOT, "include"),
                    "-I", os.path.join(pkg, "host"), "-L", pkg, "-lpfgpu", f"-Wl,-rpath,{pkg}", "-o", exe], check=True)
    r = subprocess.run([exe], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr
    lines = [ln.split() for ln in r.stdout.strip().split("\n")]
    qx, qy = [x + 0.1 for x in FX], [y - 0.05 for y in FY]
    cfg = dict(linear_search_range=0.3, angular_search_range=0.1, linear_step=0.05, angular_step=0.02, grid_resolution=0.05)
    want = [CO.match(FX, FY, qx, qy, (0.0, 0.0, 0.0), cfg), CO.match(FX, FY, FX, FY, (0.2, -0.1, 0.05), cfg),
            CO.match(FX, FY, [], [], (0.5, 0.5, 7.0), cfg)]
    assert len(lines) == 3
    for ln, w in zip(lines, want):
        assert np.array_equal(bits([float.fromhex(v) for v in ln[:4]]), bits(w[:4])) and int(ln[4]) == int(w[4])


def expected_sparse(rx, ry, qx, qy, pose, lstep, nl, res):
    """the winner of a window with no angular offsets whose nonzero scores all lie near the candidates that put a query point on a
    reference point: those candidates are scored by the oracle one by one, every other candidate scores 0.0 (its cells are outside
    the table), and the lexicographic order of the rule picks the winner"""
    cand = set()
    for x, y in zip(rx, ry):
        for px, py in zip(qx, qy):
            i0, j0 = round((x - px - pose[0]) / lstep), round((y - py - pose[1]) / lstep)
            cand |= {(i, j) for i in range(i0 - 8, i0 + 9) for j in range(j0 - 8, j0 + 9) if -nl <= i <= nl and -nl <= j <= nl}
    best = None
    for i, j in cand:
        dx, dy = i * lstep, j * lstep
        s = CO.score(rx, ry, qx, qy, (pose[0] + dx, pose[1] + dy, pose[2]), res)
        key = (-s, (dx * dx + dy * dy) + 0.0 * 0.0, (i + nl) * (2 * nl + 1) + (j + nl))
        if best is None or key < best[0]:
            best = (key, (pose[0] + dx, pose[1] + dy, pose[2], s, s > 0.0))
    assert best[1][3] > 0.0
    return best[1]


@pytest.mark.parametrize("ref", [(3276.0, 3100.0), (0.25, 1000.0), (-3276.0, -3000.0)], ids=["t_above_2p32", "t_above_2p31", "t_small"])
def test_widest_linear_window(ref):
    """n_linear at its cap, 2^15 (NL = 65 537, 4.3e9 candidates): the candidate index within a yaw passes 2^31 and 2^32, where a
    32-bit index would wrap.  The only reference point sits where the winner's index is in the named range."""
    m = rr.CorrelativeScanMatcher()
    m.set_reference([ref[0]], [ref[1]])
    qx, qy, pose = [0.0, 0.12], [0.0, -0.07], (0.0, 0.0, 0.0)
    cfg = dict(linear_search_range=3276.8, angular_search_range=0.0, linear_step=0.1, angular_step=0.02, grid_resolution=0.05)
    want = expected_sparse([ref[0]], [ref[1]], qx, qy, pose, 0.1, 1 << 15, 0.05)
    assert_same(m.match(qx, qy, pose, cfg_of(cfg)), want)
    # one offset more is refused, and the handle stays usable
    assert raw_match(m, cfg_of(dict(cfg, linear_search_range=3276.9)), qx, qy, pose) == -2
    assert_same(m.match(qx, qy, pose, cfg_of(cfg)), want)


@pytest.mark.parametrize("ws", [None, "100000"])
def test_empty_queries_take_no_blocks_and_keep_their_result(sc, monkeypatch, ws):
    """a batch whose members alternate empty and not, in one group and in groups of three queries with points: each result equals
    its own oracle call, and an empty member keeps the invalid result"""
    if ws:
        monkeypatch.setenv("PFGPU_CSM_WS_CAP", ws)
    rx, ry = plan_points(sc)
    m = rr.CorrelativeScanMatcher()
    m.set_reference(rx, ry)
    cfg = dict(linear_search_range=0.2, angular_search_range=0.04, linear_step=0.05, angular_step=0.01, grid_resolution=0.05)
    qxs, qys, poses = [], [], []
    for q in range(9):
        x, y = CO.scan_points(sc.scans[q], sc.ANGLE_MIN, sc.ANGLE_INC)
        n = 0 if q in (0, 2, 3, 8) else x.size
        qxs.append(x[:n]), qys.append(y[:n]), poses.append(np.array(sc.truth[q]) + [0.03, -0.02, 0.01 + 7.0 * (n == 0)])
    got = m.match(qxs, qys, np.array(poses), cfg_of(cfg))
    for q in range(9):
        assert_same(got[q], CO.match(rx, ry, qxs[q], qys[q], poses[q], cfg), q)
    assert got[0] == rr.ScanMatchResult(*poses[0], 0.0, False)
