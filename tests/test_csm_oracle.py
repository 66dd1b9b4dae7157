"""CPU checks of the correlative scan matching oracle (tests/host/csm_oracle.c, DESIGN §3.13):
  - the glibc build reproduces tests/golden/csm_golden.json (the independent Python restatement) bit for bit, tables included; the
    contract build agrees with it to 4 ulp of the score and exactly in the pose;
  - the reference's own four tests (correlative_scan_matching.rs:234-345) hold on the oracle;
  - the cutoff radius quirk, the invalid and zero-candidate results, all-zero scores, exact ties, saturated cells, duplicate and
    single reference points, |yaw| >> pi;
  - scan-matched mapping on ScanScenario beats dead reckoning, within bounds measured on this oracle;
  - CorrelativeScanMatcher refuses bad input before it looks for a device."""
import ctypes as C
import json
import math
import os

import numpy as np
import pytest

import _csm_oracle as CO
import _ogm_oracle as OO
import rust_robotics_b200 as rr
from rust_robotics_b200 import scenarios

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "csm_golden.json")
CASES = json.load(open(GOLDEN))["cases"]
FIXTURE = [(0.0, 0.0), (1.0, 0.0), (2.0, 0.0), (0.0, 1.0), (0.0, 2.0), (1.0, 1.0), (1.5, 2.0)]
FX, FY = [p[0] for p in FIXTURE], [p[1] for p in FIXTURE]


def unhex(v):
    return [unhex(a) for a in v] if isinstance(v, list) else float.fromhex(v)


def case_args(c):
    """(rx, ry, qx, qy, pose, cfg dict) of a golden case"""
    cfg = dict(zip(CO.FIELDS, unhex(c["cfg"])))
    return unhex(c["rx"]), unhex(c["ry"]), unhex(c["qx"]), unhex(c["qy"]), unhex(c["pose"]), cfg


def expected(c):
    r = c["result"]
    return float.fromhex(r["x"]), float.fromhex(r["y"]), float.fromhex(r["yaw"]), float.fromhex(r["score"]), r["converged"]


def same_bits(a, b):
    return np.array_equal(np.array(a, dtype=np.float64).view(np.uint64), np.array(b, dtype=np.float64).view(np.uint64))


def inverse_transform(points, pose):
    c, s = math.cos(pose[2]), math.sin(pose[2])
    return ([c * (x - pose[0]) + s * (y - pose[1]) for x, y in points], [-s * (x - pose[0]) + c * (y - pose[1]) for x, y in points])


@pytest.mark.parametrize("case", CASES, ids=[c["name"] for c in CASES])
def test_glibc_oracle_reproduces_golden(case):
    rx, ry, qx, qy, pose, cfg = case_args(case)
    got = CO.match(rx, ry, qx, qy, pose, cfg, libm=True)
    want = expected(case)
    assert same_bits(got[:4], want[:4]) and got[4] == want[4], (got, want)
    if "table" in case:
        tab, R = CO.table(rx, ry, cfg["grid_resolution"], libm=True)
        assert R == case["table"]["R"]
        assert sorted([k[0], k[1], v.hex()] for k, v in tab.items()) == case["table"]["cells"]


@pytest.mark.parametrize("case", CASES, ids=[c["name"] for c in CASES])
def test_contract_oracle_agrees_with_glibc(case):
    """the contract's exp / sincos are within 2 ulp of glibc's (DESIGN §8 deviation 2): on these cases the winner is the same
    pose, and the score within 4 ulp per point"""
    rx, ry, qx, qy, pose, cfg = case_args(case)
    a = CO.match(rx, ry, qx, qy, pose, cfg, libm=False)
    b = CO.match(rx, ry, qx, qy, pose, cfg, libm=True)
    assert same_bits(a[:3], b[:3]) and a[4] == b[4]
    assert abs(a[3] - b[3]) <= 4 * max(1, len(qx)) * np.spacing(max(abs(b[3]), 1.0))


def test_golden_covers_the_cases():
    names = {c["name"] for c in CASES}
    for must in ("identity", "translation", "rotation", "table_res_0.05", "table_res_0.25", "invalid_empty_reference", "invalid_empty_query",
                 "invalid_linear_step", "invalid_angular_step", "invalid_resolution", "no_linear_offsets", "no_angular_offsets",
                 "all_zero_scores", "tie_equal_penalty", "saturated_query_cells", "duplicate_reference", "single_reference", "large_yaw",
                 "random_cloud"):
        assert must in names


# ---- the reference's own tests (correlative_scan_matching.rs:234-345) ----
@pytest.mark.parametrize("libm", [False, True])
def test_identity_match(libm):
    x, y, yaw, score, conv, n = CO.match(FX, FY, FX, FY, (0.0, 0.0, 0.0), libm=libm)
    assert conv and x == 0.0 and y == 0.0 and yaw == 0.0 and score == 7.0
    assert n == 21 * 21 * 21                     # the defaults' 9 261 candidates


@pytest.mark.parametrize("libm", [False, True])
def test_known_translation_recovery(libm):
    qx, qy = inverse_transform(FIXTURE, (0.4, -0.3, 0.0))
    cfg = dict(linear_search_range=0.6, angular_search_range=0.1, linear_step=0.1, angular_step=0.05, grid_resolution=0.05)
    x, y, yaw, _, conv, _ = CO.match(FX, FY, qx, qy, (0.0, 0.0, 0.0), cfg, libm=libm)
    assert conv and abs(x - 0.4) < 1e-9 and abs(y + 0.3) < 1e-9 and abs(yaw) < 1e-9


@pytest.mark.parametrize("libm", [False, True])
def test_known_rotation_recovery(libm):
    qx, qy = inverse_transform(FIXTURE, (0.0, 0.0, 0.16))
    cfg = dict(linear_search_range=0.2, angular_search_range=0.3, linear_step=0.1, angular_step=0.02, grid_resolution=0.05)
    x, y, yaw, _, conv, _ = CO.match(FX, FY, qx, qy, (0.0, 0.0, 0.0), cfg, libm=libm)
    assert conv and abs(x) < 1e-9 and abs(y) < 1e-9 and abs(yaw - 0.16) < 1e-9


@pytest.mark.parametrize("libm", [False, True])
def test_lookup_table_prefers_exact_alignment(libm):
    aligned = CO.score(FX, FY, FX, FY, (0.0, 0.0, 0.0), 0.05, libm)
    assert aligned > CO.score(FX, FY, FX, FY, (0.15, 0.0, 0.0), 0.05, libm)
    assert aligned > CO.score(FX, FY, FX, FY, (0.0, 0.0, 0.15), 0.05, libm)


# ---- the rule's corners ----
def test_cutoff_radius_quirk():
    """R = ceil(3 sigma / res) with sigma = res: 3 * res / res is 3.0000000000000004 at 0.05 and 0.1, so R = 4; exactly 3 at 0.25"""
    for res, R in ((0.05, 4), (0.1, 4), (0.025, 4), (0.2, 4), (0.25, 3), (0.02, 3), (0.5, 3), (1.0, 3)):
        assert math.ceil(3.0 * res / res) == R
        assert CO.table([0.0], [0.0], res)[1] == R
    # an entry that exists only because R = 4: four cells from the centre along an axis, weight exp(-8) > 1e-6
    tab, _ = CO.table([0.0], [0.0], 0.05, libm=True)
    assert (4, 0) in tab and (0, -4) in tab and abs(tab[(4, 0)] - math.exp(-8.0)) < 1e-15
    assert max(max(abs(k[0]), abs(k[1])) for k in tab) == 4
    tab3, _ = CO.table([0.0], [0.0], 0.25, libm=True)
    assert (4, 0) not in tab3 and (3, 0) in tab3
    by = {c["name"]: c for c in CASES}
    for name, R in (("table_res_0.05", 4), ("table_res_0.25", 3)):
        cells = by[name]["table"]["cells"]
        assert by[name]["table"]["R"] == R
        rx, ry = unhex(by[name]["rx"]), unhex(by[name]["ry"])
        res = float(name.split("_")[-1])
        centres = {(int(round(x / res)), int(round(y / res))) for x, y in zip(rx, ry)}
        reach = max(min(max(abs(c[0] - a), abs(c[1] - b)) for a, b in centres) for c in cells)
        assert reach == R


def test_invalid_and_zero_candidate_results():
    by = {c["name"]: expected(c) for c in CASES}
    for name in ("invalid_empty_reference", "invalid_empty_query", "invalid_linear_step", "invalid_angular_step", "invalid_resolution"):
        x, y, yaw, score, conv = by[name]
        assert (x, y, abs(yaw), score, conv) == (1.0, 2.0, 7.0, 0.0, False), name          # the yaw as given
    for name in ("no_linear_offsets", "no_angular_offsets"):
        x, y, yaw, score, conv = by[name]
        assert (x, y, score, conv) == (1.0, 2.0, -1.0, False) and abs(yaw) < math.pi and abs(abs(yaw) - (7.0 - 2.0 * math.pi)) < 1e-15


def test_all_zero_scores_pick_the_zero_penalty_candidate():
    x, y, yaw, score, conv = expected({c["name"]: c for c in CASES}["all_zero_scores"])
    assert score == 0.0 and not conv and (x, y) == (0.3, -0.2) and yaw == 4.0 - 2.0 * math.pi


def test_ties_at_equal_penalty_go_to_the_earlier_candidate():
    by = {c["name"]: expected(c) for c in CASES}
    assert by["tie_equal_penalty"][:2] == (-0.2, 0.0)          # dx = -0.2 comes before dx = +0.2 in the loop
    assert by["tie_equal_penalty_y"][:2] == (0.0, -0.3)
    # and the candidates really tie: the same score at the same penalty
    assert CO.score([-0.2, 0.2], [0.0, 0.0], [0.0], [0.0], (-0.2, 0.0, 0.0), 0.05) == CO.score([-0.2, 0.2], [0.0, 0.0], [0.0], [0.0],
                                                                                                (0.2, 0.0, 0.0), 0.05)


def test_saturated_duplicate_single_and_large_yaw():
    by = {c["name"]: expected(c) for c in CASES}
    assert by["saturated_query_cells"][3] == 7.0                  # the two far points read 0.0
    assert by["duplicate_reference"][3] == 7.0 and by["duplicate_reference"][:3] == (0.0, 0.0, 0.0)
    assert by["single_reference"][4] and by["single_reference"][3] < 1.0
    for name, yaw0 in (("large_yaw", 1000.0), ("large_negative_yaw", -1234.5)):
        assert abs(by[name][2]) <= math.pi and by[name][3] == 1.0


# ---- scan-matched mapping ----
def run_oracle_mapping(sc, odom):
    W, H = sc.obstacles.shape
    o = OO.OracleOgm(resolution=sc.RES, width=W, height=H)
    ref = {}

    def fuse(p, r):
        o.update_with_scans([p], [r], sc.ANGLE_MIN, sc.ANGLE_INC)

    def set_reference():
        ref["p"] = CO.grid_points(o.obstacles(0.5).astype(bool), sc.RES)

    def match(qx, qy, pose):
        return CO.match(ref["p"][0], ref["p"][1], qx, qy, pose, CO.MAP_CFG)

    poses, scores = CO.scan_matched_mapping(sc, odom, fuse, set_reference, match)
    return poses, scores, o


# measured on this oracle (contract math) with CO.MAP_CFG and CO.ODOM_SIGMA, seed 3: matched 0.047 m / 0.0084 rad at worst, dead
# reckoning 0.196 m / 0.055 rad
MATCHED_POS_BOUND, MATCHED_YAW_BOUND = 0.06, 0.012


def test_scan_matched_mapping_beats_dead_reckoning():
    sc = scenarios.ScanScenario(steps=60)
    odom = CO.odometry(sc.truth)
    poses, scores, _ = run_oracle_mapping(sc, odom)
    pos, yaw = CO.pose_errors(sc, poses)
    dpos, dyaw = CO.pose_errors(sc, CO.dead_reckoning(sc.truth, odom))
    assert pos < dpos and yaw < dyaw
    assert pos < MATCHED_POS_BOUND and yaw < MATCHED_YAW_BOUND, (pos, yaw)
    assert dpos > 2 * MATCHED_POS_BOUND and dyaw > 2 * MATCHED_YAW_BOUND
    assert scores.min() > 100.0


# ---- refusals before any device ----
def test_invalid_shapes_are_refused_before_the_device():
    with pytest.raises(rr.InvalidParameter):
        rr.CorrelativeScanMatcher.match(object.__new__(rr.CorrelativeScanMatcher), [0.0, 1.0], [0.0], (0.0, 0.0, 0.0))


def test_matcher_needs_a_device():
    """no CPU fallback: without a device the matcher cannot be made"""
    cnt = C.c_int()
    if rr.load_library().pfgpu_device_count(C.byref(cnt)) == 0 and cnt.value > 0:
        pytest.skip("a CUDA device is present")
    with pytest.raises(rr.PfgpuError):
        rr.CorrelativeScanMatcher()
    with pytest.raises(rr.PfgpuError):
        rr.correlative_scan_match(FX, FY, FX, FY, (0.0, 0.0, 0.0), rr.CorrelativeScanMatcherConfig())
