"""CPU checks of the occupancy grid mapping oracle (tests/host/ogm_oracle.c, DESIGN §3.12) and of the config refusals:
  - the glibc build reproduces tests/golden/ogm_golden.json (the independent Python restatement) bit for bit: every cell, the
    obstacle masks and the census (events, most updates of one cell, beams with a repeated cell, longest ray);
  - a batch equals the same scans one call at a time;
  - no beam updates a cell twice (the property the device's order-by-cell fold relies on), on every golden case and on a whole
    ScanScenario trajectory, plain and tiled;
  - the closed form of bresenham_line the device walks equals the loop;
  - OccupancyGridMap refuses bad configs before it looks for a device."""
import ctypes as C
import json
import math
import os

import numpy as np
import pytest

import _ogm_oracle as OO
import rust_robotics_b200 as rr
from rust_robotics_b200 import scenarios

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ogm_golden.json")
CASES = json.load(open(GOLDEN))["cases"]


def unhex(v):
    return [unhex(a) for a in v] if isinstance(v, list) else float.fromhex(v)


def golden_cfg(c):
    return {k: (float.fromhex(v) if isinstance(v, str) else v) for k, v in c["cfg"].items()}


def run_case(c, libm, one_call=False):
    o = OO.OracleOgm(libm=libm, **golden_cfg(c))
    for call in c["calls"]:
        if one_call:
            for p, r in zip(unhex(call["poses"]), unhex(call["ranges"])):
                o.update_with_scan(p[0], p[1], p[2], r, float.fromhex(call["angle_min"]), float.fromhex(call["angle_inc"]))
        else:
            o.update_with_scans(unhex(call["poses"]), unhex(call["ranges"]), float.fromhex(call["angle_min"]), float.fromhex(call["angle_inc"]))
    return o


def expected_grid(c):
    cfg = golden_cfg(c)
    g = np.full(cfg["width"] * cfg["height"], cfg["prior_log_odds"])
    for idx, v in c["changed"]:
        g[idx] = float.fromhex(v)
    return g.reshape(cfg["width"], cfg["height"])


def bits(a):
    return np.ascontiguousarray(a, dtype=np.float64).view(np.uint64)


@pytest.mark.parametrize("case", CASES, ids=[c["name"] for c in CASES])
def test_oracle_reproduces_golden(case):
    o = run_case(case, libm=True)
    assert np.array_equal(bits(o.grid), bits(expected_grid(case)))
    for t, m in case["masks"].items():
        assert "".join(map(str, o.obstacles(float.fromhex(t)).ravel())) == m
    tot = [0, 0, 0, 0]                 # events, -, beams with a repeated cell, longest ray: summed over the calls
    for call in case["calls"]:
        e, _, rep, longest = o.census(unhex(call["poses"]), unhex(call["ranges"]), float.fromhex(call["angle_min"]), float.fromhex(call["angle_inc"]))
        tot[0] += e
        tot[2] += rep
        tot[3] = max(tot[3], longest)
    assert tot[0] == case["census"][0] and tot[3] == case["census"][3]
    assert tot[2] == 0 and case["census"][2] == 0, "a beam updated a cell twice"


@pytest.mark.parametrize("libm", [False, True])
@pytest.mark.parametrize("case", CASES, ids=[c["name"] for c in CASES])
def test_batch_equals_single_scans(case, libm):
    assert np.array_equal(bits(run_case(case, libm).grid), bits(run_case(case, libm, one_call=True).grid))


def test_golden_covers_the_cases():
    names = {c["name"] for c in CASES}
    for must in ("one_by_n", "n_by_one", "non_square", "origin_on_edges", "origin_outside", "special_ranges", "nan_yaw", "end_outside",
                 "zero_length", "saturate_occ_then_free", "saturate_free_then_occ", "saturate_min", "min_equals_max",
                 "zero_deltas_prior_outside", "prior_below_min", "same_cells_one_scan", "repeated_scans"):
        assert must in names


def test_saturation_order_matters():
    """From l = 4.9 with limits +-5: +0.85 then -0.4 gives 4.6, -0.4 then +0.85 gives 5.0 (the cell both rays share)"""
    by = {c["name"]: expected_grid(c) for c in CASES}
    g1, g2 = by["saturate_occ_then_free"], by["saturate_free_then_occ"]
    assert g1[7, 5] == 5.0 - 0.4 and abs(g1[7, 5] - 4.6) < 1e-12
    assert g2[7, 5] == 5.0
    assert by["saturate_one_batch"][7, 5] == 5.0 - 0.4


@pytest.mark.parametrize("cells", [0, 8192])
def test_no_cell_twice_per_beam_on_a_trajectory(cells):
    sc = scenarios.ScanScenario(steps=60, cells=cells)
    W, H = sc.obstacles.shape
    o = OO.OracleOgm(resolution=sc.RES, width=W, height=H)
    events, most, repeats, longest = o.census(sc.truth, np.stack(sc.scans), sc.ANGLE_MIN, sc.ANGLE_INC)
    assert repeats == 0
    assert events > 60 * 300 and most >= 60 and 1 < longest <= 2 + int(sc.MAX_RANGE / sc.RES) * 2


def closed_form(x0, y0, x1, y1):
    """the device's walk (ogm.cuh pf_ogm_emit_kernel): step k moves k along the major axis and floor((2 k dm + dM - 1) / (2 dM))
    along the minor one"""
    dx, dy = x1 - x0, y1 - y0
    adx, ady = abs(dx), abs(dy)
    xmaj = adx >= ady
    dM, dm = (adx, ady) if xmaj else (ady, adx)
    sx, sy = (1 if x0 < x1 else -1), (1 if y0 < y1 else -1)
    out = []
    for k in range(dM + 1):
        mi = (2 * k * dm + dM - 1) // (2 * dM) if dm else 0
        ox, oy = (k, mi) if xmaj else (mi, k)
        out.append((x0 + sx * ox, y0 + sy * oy))
    return out


def test_closed_form_equals_the_loop():
    for dx in range(-40, 41):
        for dy in range(-40, 41):
            assert [tuple(c) for c in OO.line(3, -7, 3 + dx, -7 + dy)] == closed_form(3, -7, 3 + dx, -7 + dy), (dx, dy)
    rng = np.random.default_rng(5)
    for _ in range(300):
        x0, y0 = (int(v) for v in rng.integers(0, 65536, 2))
        x1, y1 = (int(v) for v in rng.integers(0, 65536, 2))
        assert [tuple(c) for c in OO.line(x0, y0, x1, y1)] == closed_form(x0, y0, x1, y1)


@pytest.mark.parametrize("bad", [dict(width=0), dict(height=0), dict(width=65537), dict(width=20000, height=20000),
                                 dict(resolution=0.0), dict(resolution=-0.5), dict(resolution=math.inf), dict(resolution=math.nan),
                                 dict(prior_log_odds=math.nan), dict(occupied_log_odds=math.inf), dict(free_log_odds=-math.inf),
                                 dict(max_log_odds=math.nan), dict(min_log_odds=math.nan), dict(min_log_odds=1.0, max_log_odds=0.5)])
def test_config_refusals(bad):
    with pytest.raises(rr.InvalidParameter):
        rr.OccupancyGridMap(rr.OccupancyGridConfig(**bad))


def test_valid_config_needs_a_device():
    """a valid config is refused only for want of a device: no CPU fallback (the prior may lie outside [min, max])"""
    cnt = C.c_int()
    if rr.load_library().pfgpu_device_count(C.byref(cnt)) == 0 and cnt.value > 0:
        pytest.skip("a CUDA device is present")
    with pytest.raises(rr.PfgpuError):
        rr.OccupancyGridMap(rr.OccupancyGridConfig(prior_log_odds=9.0, min_log_odds=2.0, max_log_odds=2.0))
