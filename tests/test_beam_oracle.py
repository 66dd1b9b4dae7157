"""CPU tests of the beam measurement model (DESIGN §3.11) on the oracle (tests/host/pf_beam_oracle.c):
  - the glibc build reproduces tests/golden/beam_golden.json (the Python restatement) bit for bit: the beam limit L, the clearance
    table, the expected ranges, the used beams and the raw weight of every pose under every scan, and the refusal at L + 1 beams;
  - the closed form of bresenham_line the device's skipping caster walks equals the loop: exhaustively for |dx|, |dy| <= 256 in every
    direction, and on random lines with deltas up to 2^20 for the first 2^17 steps;
  - the clearance table equals scipy.ndimage.distance_transform_cdt (chessboard) of the mask padded with a ring of obstacles;
  - occlusion: a pose across a 0.2 m wall from the truth loses more weight under the beam model than under the likelihood field;
  - behaviour, with Philox draws: global localisation in ScanScenario's floor plan from init_region with recovery on ends within
    0.5 m and 0.1 rad of the truth."""
import json
import math
import os

import numpy as np
import pytest
from scipy import ndimage

import _beam_oracle as BO
from rust_robotics_b200 import scenarios

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "beam_golden.json")


def fx(v):
    if isinstance(v, list):
        return np.array([fx(a) for a in v])
    return float.fromhex(v)


def _cases():
    with open(GOLDEN) as f:
        return json.load(f)["cases"]


def _mask(c):
    return np.array([[ch == "1" for ch in row] for row in c["mask"]], dtype=bool).reshape(c["W"], c["H"])


def _kw(c):
    v = fx(c["cfg"][:8]).tolist()
    return v[0], dict(sigma_hit=v[1], z_hit=v[2], z_short=v[3], z_max=v[4], z_rand=v[5], lambda_short=v[6], max_range=v[7],
                      max_beams=c["cfg"][8])


@pytest.mark.parametrize("case", _cases(), ids=lambda c: c["name"])
def test_oracle_reproduces_golden(case):
    o = BO.OracleBeam(4, libm=True)
    res, kw = _kw(case)
    assert o.set_beam_map(_mask(case), res, **kw) == 0
    assert o.beam_info() == (case["W"], case["H"], case["L"])
    assert np.array_equal(o.clearance(), np.array(case["clearance"], dtype=np.uint8).reshape(case["W"], case["H"]))
    poses = fx(case["poses"])
    for c in case["casts"]:
        got = o.raycast(poses, c["B"], fx(c["angle_min"]), fx(c["angle_inc"]))
        assert np.array_equal(got, fx(c["rhat"]).reshape(len(poses), c["B"]))
    for j, s in enumerate(case["scans"]):
        args = (fx(s["ranges"]), fx(s["angle_min"]), fx(s["angle_inc"]))
        b, w = o.beam_beams(*args), o.beam_weights(poses, *args)
        if s["used"] < 0:
            assert b is None and w is None, f"scan {j}: not refused"
        else:
            assert b.shape[0] == s["used"] and np.array_equal(b.reshape(-1), fx(s["beams"]).reshape(-1)), f"scan {j}: beams"
            assert np.array_equal(w, fx(s["w"])), f"scan {j}: weights"


def test_golden_covers_the_cases():
    cases = {c["name"]: c for c in _cases()}
    assert cases["row_1xN"]["W"] == 1 and cases["col_Nx1"]["H"] == 1
    assert all(v == 0 for row in cases["full"]["clearance"] for v in row)
    rh = [fx(c["rhat"]) for c in cases["full"]["casts"]]
    assert all((r == 0.0).all() for r in rh)                                     # every start cell occupied
    walls = fx(cases["walls"]["casts"][0]["rhat"])
    assert (walls == 0.0).any() and ((walls > 0.0) & (walls < 6.0)).any()
    assert (fx(cases["empty"]["casts"][0]["rhat"]) == 3.0).any()                  # no obstacle up to c1: max_range
    bound = cases["beam_bound"]
    assert [s["used"] for s in bound["scans"]] == [bound["L"], -1]
    assert cases["z_max_0"]["scans"][0]["used"] < cases["walls"]["scans"][1]["used"]   # the same ranges without their max readings
    strides = {n: c["scans"][0]["used"] for n, c in cases.items() if n.startswith("stride_")}
    assert strides["stride_B7_mb2"] == 2 and strides["stride_B1_mb60"] == 1
    ranges = fx(cases["walls"]["scans"][1]["ranges"])
    assert np.isnan(ranges).any() and np.isinf(ranges).any() and (ranges == 6.0).any() and (ranges == 0.0).any() and (ranges < 0).any()


# ---- the closed form of bresenham_line that the device walks (pf_beam.cuh) ----
def _closed(i, dM, dm):
    return np.where(dm == 0, 0, (2 * i * dm + dM - 1) // np.maximum(2 * dM, 1))


def _check_lines(dx, dy, steps):
    """run bresenham_line's loop on every line (0, 0) -> (dx, dy) at once; at each step compare the cell with the closed form"""
    dx, dy = np.asarray(dx, np.int64), np.asarray(dy, np.int64)
    adx, ady = np.abs(dx), np.abs(dy)
    sx, sy = np.where(0 < dx, 1, -1), np.where(0 < dy, 1, -1)
    xmaj = adx >= ady
    dM, dm = np.where(xmaj, adx, ady), np.where(xmaj, ady, adx)
    x, y, err = np.zeros_like(dx), np.zeros_like(dy), adx - ady
    live = np.ones(dx.shape, bool)
    for i in range(steps + 1):
        mi = _closed(i, dM, dm)
        ex, ey = np.where(xmaj, sx * i, sx * mi), np.where(xmaj, sy * mi, sy * i)
        ok = ~live | ((x == ex) & (y == ey))
        assert ok.all(), (dx[~ok][:5], dy[~ok][:5], i)
        done = (x == dx) & (y == dy)
        assert not (live & done & (i != dM)).any()                              # the loop ends exactly at step d_major
        live &= ~done
        if not live.any():
            return
        e2 = 2 * err
        a, b = e2 > -ady, e2 < adx
        err = np.where(live & a, err - ady, err)
        x = np.where(live & a, x + sx, x)
        err = np.where(live & b, err + adx, err)
        y = np.where(live & b, y + sy, y)


def test_closed_form_exhaustive_256():
    d = np.arange(-256, 257)
    dx, dy = np.meshgrid(d, d, indexing="ij")
    _check_lines(dx.ravel(), dy.ravel(), 256)


def test_closed_form_random_long_lines():
    rng = np.random.default_rng(17)
    n = 96
    big = rng.integers(-(1 << 20), (1 << 20) + 1, size=(n, 2))
    big[:8, 1] = big[:8, 0]                                                     # ties
    big[8:16, 1] = -big[8:16, 0]
    big[16:20, 1] = 0                                                           # axis-aligned
    big[20:24, 0] = rng.integers(-3, 4, 4)                                      # nearly vertical
    _check_lines(big[:, 0], big[:, 1], 1 << 17)


# ---- the clearance table ----
def _scipy_clearance(mask):
    free = np.pad(~np.asarray(mask, bool), 1, constant_values=False)
    return np.minimum(ndimage.distance_transform_cdt(free, metric="chessboard"), 255)[1:-1, 1:-1].astype(np.uint8)


@pytest.mark.parametrize("seed", range(6))
def test_clearance_against_scipy(seed):
    rng = np.random.default_rng(seed)
    W, H = [(1, 40), (37, 1), (23, 31), (64, 48), (600, 580), (7, 90)][seed]
    m = rng.random((W, H)) < [0.02, 0.1, 0.05, 0.01, 0.000005, 0.0][seed]
    for libm in (False, True):
        assert np.array_equal(BO.chessboard(m, libm), _scipy_clearance(m))
    for c in _cases():
        assert np.array_equal(np.array(c["clearance"], dtype=np.uint8).reshape(c["W"], c["H"]), _scipy_clearance(_mask(c))), c["name"]


def test_floor_plan_clearance_against_scipy():
    m = scenarios.ScanScenario.plan()
    assert np.array_equal(BO.chessboard(m), _scipy_clearance(m))
    assert np.array_equal(BO.chessboard(np.zeros((700, 650), bool)), _scipy_clearance(np.zeros((700, 650), bool)))   # capped at 255


def test_refusals():
    o = BO.OracleBeam(8, mode=1, max_particles=8)
    m = np.zeros((4, 4), dtype=bool)
    assert o.update_beam([1.0], 0.0, 0.1) == -1                                 # no map
    for bad in (dict(resolution=0.0), dict(resolution=np.nan), dict(sigma_hit=-1.0), dict(z_hit=-0.1), dict(z_short=-0.1),
                dict(z_short=np.inf), dict(z_max=-1.0), dict(z_rand=0.0), dict(lambda_short=0.0), dict(max_range=np.inf),
                dict(max_beams=1), dict(resolution=1e-6, max_range=2.0), dict(z_rand=1e-300, z_max=0.0, max_range=1e10)):
        a = dict(resolution=0.05)
        a.update(bad)
        assert o.set_beam_map(m, a.pop("resolution"), **a) == -1, bad
    assert o.set_beam_map(m, 0.05) == 0
    assert o.update_beam([1.0], np.nan, 0.1) == -1 and o.update_beam([1.0], 0.0, np.inf) == -1
    assert o.update_beam([], 0.0, 0.1) == 0 and np.all(o.particles()[:, 4] == 1.0 / 8)


def _march(mask, res, pose, B=360, amin=-math.pi, ainc=math.pi / 180.0, max_range=30.0):
    """ScanScenario's ray-marching (every res / 4) from one pose; no obstacle within max_range: inf"""
    W, H = mask.shape
    ang = pose[2] + amin + np.arange(B) * ainc
    ds = np.arange(1, int(max_range / (res / 4.0)) + 1) * (res / 4.0)
    ex, ey = pose[0] + np.cos(ang)[:, None] * ds, pose[1] + np.sin(ang)[:, None] * ds
    ix, iy = np.floor(ex / res + W / 2.0).astype(np.int64), np.floor(ey / res + H / 2.0).astype(np.int64)
    inside = (ix >= 0) & (ix < W) & (iy >= 0) & (iy < H)
    hit = inside & mask[np.clip(ix, 0, W - 1), np.clip(iy, 0, H - 1)]
    first = np.where(hit.any(axis=1), hit.argmax(axis=1), -1)
    return np.where(first >= 0, ds[first], np.inf), amin, ainc


def test_occlusion_beam_against_likelihood_field():
    """the truth at (-5.4, 0, 0) just east of the west rooms' 0.2 m wall (x = -6 .. -5.8); the candidate at (-6.2, 0, 0) just west
    of it, in the room behind.  Its beam endpoints land next to the same wall, so the likelihood field barely tells them apart;
    the beam model sees that its beams are stopped by the wall.  The gaps are recorded in DESIGN §3.11."""
    sc = scenarios.ScanScenario(steps=1)
    truth, other = (-5.4, 0.0, 0.0), (-6.2, 0.0, 0.0)
    scan = _march(sc.obstacles, sc.RES, truth)
    o = BO.OracleBeam(4)
    assert o.set_beam_map(sc.obstacles, sc.RES) == 0 and o.set_map(sc.obstacles, sc.RES) == 0
    wb = o.beam_weights([truth, other], *scan)
    wl = o.weights([truth, other], *scan)
    gap_b, gap_l = math.log(wb[0]) - math.log(wb[1]), math.log(wl[0]) - math.log(wl[1])
    print(f"log-weight gap truth - across the wall: beam {gap_b:.2f}, likelihood field {gap_l:.2f}")
    assert gap_b > gap_l and gap_b > 0.0


@pytest.mark.parametrize("seed", [5, 6])
def test_global_localisation_in_floor_plan(seed):
    sc = scenarios.ScanScenario()
    n = 1 << 14
    o = BO.OracleBeam(n, mode=1, max_particles=n, velocity_noise=0.2, yaw_rate_noise=0.1, seed=seed, threads=min(16, os.cpu_count() or 1))
    assert o.set_beam_map(sc.obstacles, sc.RES) == 0
    o.enable(0.001, 0.1, sc.REGION)
    o.init_region(sc.REGION)
    err = [sc.error(k, o.step_beam(sc.controls[k], *sc.scan_args(k))[0]) for k in range(len(sc.controls))]
    assert err[-1][0] < 0.5 and err[-1][1] < 0.1, err[-1]
