"""Occupancy grid mapping on the device (DESIGN §3.12) against the contract-math oracle (tests/host/ogm_oracle.c), bit for bit:
every golden case, ScanScenario's trajectory in every batching on the floor plan and the tiled 8192^2 grid, chunked batches, repeated
runs, the device obstacle mask; the hand-off of a grid to the likelihood field and the beam model; a map made on the device that
localises a robot; the C++ mirror and the sharded hand-off."""
import os
import subprocess
import sys

import numpy as np
import pytest

import _ogm_oracle as OO
import rust_robotics_b200 as rr
from rust_robotics_b200 import scenarios
from test_ogm_oracle import CASES, golden_cfg, unhex

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SV, SW = 0.2, 0.1


def bits(a):
    return np.ascontiguousarray(a, dtype=np.float64).view(np.uint64)


@pytest.fixture(scope="module")
def sc():
    return scenarios.ScanScenario()


def plan_cfg(sc, cells=0):
    W, H = (sc.obstacles.shape if not cells else (cells, cells))
    return dict(resolution=sc.RES, width=W, height=H)


def plan_map(sc, cells=0, **kw):
    return rr.OccupancyGridMap(rr.OccupancyGridConfig(**plan_cfg(sc, cells)), **kw)


def plan_maps(sc, cells=0):
    return plan_map(sc, cells), OO.OracleOgm(**plan_cfg(sc, cells))


@pytest.mark.parametrize("case", CASES, ids=[c["name"] for c in CASES])
def test_golden_cases_match_oracle(case):
    cfg = golden_cfg(case)
    g = rr.OccupancyGridMap(rr.OccupancyGridConfig(**cfg))
    o = OO.OracleOgm(**cfg)
    assert np.array_equal(bits(g.grid), bits(o.grid))
    for call in case["calls"]:
        args = unhex(call["poses"]), unhex(call["ranges"]), float.fromhex(call["angle_min"]), float.fromhex(call["angle_inc"])
        g.update_with_scans(*args)
        o.update_with_scans(*args)
        assert np.array_equal(bits(g.grid), bits(o.grid))
        events, most, _, _ = o.census(*args)
        st = g.stats()
        assert st.events == events and st.chunks == (1 if events else 0) and st.longest_run == most
    for t in (0.5, 0.2, 0.9):
        m = g.obstacles(t)
        assert np.array_equal(m, o.obstacles(t).astype(bool))
        assert np.array_equal(m, rr.obstacles_from_log_odds(g.grid, t))


def test_reference_api(sc):
    g = rr.OccupancyGridMap(rr.OccupancyGridConfig())
    o = OO.OracleOgm()
    assert g.world_to_grid(0.0, 0.0) == (50, 50) and g.world_to_grid(25.0, 0.0) is None and g.world_to_grid(-25.0, -25.0) == (0, 0)
    assert g.world_to_grid(float("nan"), 1.0) == (0, 52)
    r = sc.scans[0] / 4.0
    g.update_with_scan(1.0, -2.0, 0.4, r, sc.ANGLE_MIN, sc.ANGLE_INC)
    o.update_with_scan(1.0, -2.0, 0.4, r, sc.ANGLE_MIN, sc.ANGLE_INC)
    assert np.array_equal(bits(g.grid), bits(o.grid))
    hit = np.argwhere(o.grid > 0.0)[0]
    assert g.get_probability(*hit) == 1.0 - 1.0 / (1.0 + np.exp(o.grid[tuple(hit)])) and g.is_occupied(*hit, 0.5)
    ox, oy = g.world_to_grid(1.0, -2.0)                  # the origin: a free update from every beam
    assert o.grid[ox, oy] < 0.0 and g.get_probability(ox, oy) < 0.5 and not g.is_occupied(ox, oy, 0.5)


@pytest.mark.parametrize("cells", [0, 8192])
def test_trajectory_in_any_batching(sc, cells):
    o = OO.OracleOgm(**plan_cfg(sc, cells))
    poses, scans = np.array(sc.truth), np.stack(sc.scans)
    o.update_with_scans(poses, scans, sc.ANGLE_MIN, sc.ANGLE_INC)
    want = bits(o.grid).copy()
    del o
    splits = {"one_batch": [], "one_per_call": list(range(1, len(poses))), "uneven": [1, 4, 5, 17, 30, 31]}
    for name, cut in splits.items():
        g = plan_map(sc, cells)
        for p, r in zip(np.split(poses, cut), np.split(scans, cut)):
            g.update_with_scans(p, r, sc.ANGLE_MIN, sc.ANGLE_INC)
        assert np.array_equal(bits(g.grid), want), name
        g.close()
        if cells:
            break                      # the tiled grid: one batch (the other batchings are covered on the plan)


def test_chunked_batches_and_repeat_runs(sc, monkeypatch):
    """a batch larger than the cap runs in several chunks that split between beams; the same bits every time"""
    poses, scans = np.tile(np.array(sc.truth), (10, 1)), np.tile(np.stack(sc.scans), (10, 1))      # 600 scans
    g, o = plan_maps(sc)
    o.update_with_scans(poses, scans, sc.ANGLE_MIN, sc.ANGLE_INC)
    events, most, repeats, _ = o.census(poses, scans, sc.ANGLE_MIN, sc.ANGLE_INC)
    assert repeats == 0
    g.update_with_scans(poses, scans, sc.ANGLE_MIN, sc.ANGLE_INC)
    st = g.stats()
    assert st.events == events and st.event_cap == 1 << 24 and st.chunks >= 2 and 0 < st.longest_run <= most
    assert np.array_equal(bits(g.grid), bits(o.grid))
    for cap in ("65536", "100003"):
        monkeypatch.setenv("PFGPU_OGM_EVENT_CAP", cap)
        h = plan_map(sc)
        h.update_with_scans(poses[:120], scans[:120], sc.ANGLE_MIN, sc.ANGLE_INC)
        h.update_with_scans(poses[120:], scans[120:], sc.ANGLE_MIN, sc.ANGLE_INC)
        assert h.stats().chunks > 10 and h.stats().event_cap == int(cap)
        assert np.array_equal(bits(h.grid), bits(o.grid)), cap
    monkeypatch.delenv("PFGPU_OGM_EVENT_CAP")
    again = plan_map(sc)
    again.update_with_scans(poses, scans, sc.ANGLE_MIN, sc.ANGLE_INC)
    assert np.array_equal(bits(again.grid), bits(o.grid))
    g.set_grid(np.zeros((g.W, g.H)))
    g.update_with_scans(poses, scans, sc.ANGLE_MIN, sc.ANGLE_INC)
    assert np.array_equal(bits(g.grid), bits(o.grid))


def test_set_read_and_mask(sc):
    g, o = plan_maps(sc)
    rng = np.random.default_rng(3)
    v = rng.normal(0.0, 3.0, (g.W, g.H))
    v[:3, :3] = [[np.inf, -np.inf, np.nan], [800.0, -800.0, 0.0], [5e-324, -0.0, 1e300]]
    g.set_grid(v)
    o.grid[...] = v
    assert np.array_equal(bits(g.grid), bits(v))
    for t in (0.5, 0.0, 0.99, -1.0):
        m = g.obstacles(t)
        assert np.array_equal(m, o.obstacles(t).astype(bool)), t
        assert np.array_equal(m, rr.obstacles_from_log_odds(v, t)), t
    with pytest.raises(rr.InvalidParameter):
        g.obstacles(np.nan)
    with pytest.raises(rr.InvalidParameter):
        g.set_grid(np.zeros((3, 3)))


def mapped(sc):
    g = plan_map(sc)
    g.update_with_scans(sc.truth, np.stack(sc.scans), sc.ANGLE_MIN, sc.ANGLE_INC)
    return g


@pytest.mark.parametrize("model", ["beam", "lfield"])
def test_hand_off_equals_host_mask(sc, model):
    g = mapped(sc)
    cfg = rr.MonteCarloLocalizationConfig(4096, 4096, 0.05, 2.326, 0.25, SV, SW, 0.1)
    a = rr.MonteCarloLocalizer.try_with_region(sc.REGION, cfg, seed=9)
    b = rr.MonteCarloLocalizer.try_with_region(sc.REGION, cfg, seed=9)
    if model == "beam":
        a.set_beam_model_from_grid(g, 0.5, max_range=sc.MAX_RANGE)
        b.set_beam_model(g.obstacles(0.5), sc.RES, max_range=sc.MAX_RANGE)
        assert np.array_equal(a.beam_model(), b.beam_model()) and a.beam_model_info() == b.beam_model_info()
        step = "try_step_beam_scan"
    else:
        a.set_likelihood_field_from_grid(g, 0.5, max_range=sc.MAX_RANGE)
        b.set_likelihood_field(g.obstacles(0.5), sc.RES, max_range=sc.MAX_RANGE)
        for x, y in zip(a.likelihood_field(), b.likelihood_field()):
            assert np.array_equal(np.asarray(x), np.asarray(y))
        step = "try_step_scan"
    for t in range(6):
        getattr(a, step)(sc.controls[t], *sc.scan_args(t))
        getattr(b, step)(sc.controls[t], *sc.scan_args(t))
        assert np.array_equal(a.get_particles(), b.get_particles()) and np.array_equal(a.last_indices(), b.last_indices()), t
    # the grid is copied at set time: updating it leaves the loaded model as it was
    before = a.beam_model() if model == "beam" else a.likelihood_field()[1]
    g.update_with_scans(np.tile([0.0, 0.0, 0.0], (20, 1)), np.full((20, 360), 2.0), sc.ANGLE_MIN, sc.ANGLE_INC)
    after = a.beam_model() if model == "beam" else a.likelihood_field()[1]
    assert np.array_equal(before, after)
    c = rr.MonteCarloLocalizer.try_with_region(sc.REGION, cfg, seed=9)
    (c.set_beam_model_from_grid if model == "beam" else c.set_likelihood_field_from_grid)(g, 0.5, max_range=sc.MAX_RANGE)
    assert not np.array_equal(before, c.beam_model() if model == "beam" else c.likelihood_field()[1])


def test_hand_off_refusals(sc):
    g = mapped(sc)
    f = rr.MonteCarloLocalizer.try_with_region(sc.REGION, rr.MonteCarloLocalizationConfig(1024, 1024), seed=1)
    coarse = rr.OccupancyGridMap(rr.OccupancyGridConfig(resolution=0.1, width=400, height=300))
    for call in (f.set_beam_model_from_grid, f.set_likelihood_field_from_grid):
        with pytest.raises(rr.InvalidParameter):
            call(g, np.nan)
        with pytest.raises(rr.InvalidParameter):
            call(g, 0.5, max_beams=1)
    # a model config at another resolution than the grid's: built from the coarse grid's own resolution, refused by the C ABI
    import ctypes as C
    from rust_robotics_b200 import api
    cfg = api._BmCfg(sc.RES, 0.2, 0.95, 0.1, 0.05, 0.05, 0.1, 30.0, 60, 0)
    assert f.L.pfgpu_pf_beam_set_grid(f.h, coarse.h, 0.5, C.byref(cfg)) == -1
    lcfg = api._LfCfg(sc.RES, 0.2, 0.95, 0.05, 30.0, 60, 0)
    assert f.L.pfgpu_pf_lfield_set_grid(f.h, coarse.h, 0.5, C.byref(lcfg)) == -1
    assert f.beam_model_info() == (0, 0, 0) and f.likelihood_field_info() == (0, 0, 0)
    n = C.c_int()
    f.L.pfgpu_device_count(C.byref(n))
    if n.value < 2:
        pytest.skip("the wrong-device refusal needs two GPUs")
    other = rr.OccupancyGridMap(rr.OccupancyGridConfig(resolution=sc.RES, width=800, height=600), device=1)
    with pytest.raises(rr.InvalidParameter):
        f.set_beam_model_from_grid(other)
    with pytest.raises(rr.InvalidParameter):
        f.set_likelihood_field_from_grid(other)


@pytest.mark.parametrize("n", [1 << 14, 1 << 16])
def test_map_then_localise(sc, n):
    """map the floor plan from the truth poses and scans on the device, hand the map to the beam model and localise globally from
    init_region: within 1 m from step 10 on (the oracle at 2^14 particles, seeds 5 and 7, is within 1 m from step 0)"""
    g = mapped(sc)
    f = rr.MonteCarloLocalizer.try_with_region(sc.REGION, rr.MonteCarloLocalizationConfig(n, n, 0.05, 2.326, 0.2, SV, SW, 0.1), seed=5)
    f.set_beam_model_from_grid(g, 0.5)
    f.enable_recovery(0.001, 0.1, sc.REGION)
    err = [sc.error(k, f.try_step_beam_scan(sc.controls[k], *sc.scan_args(k))) for k in range(len(sc.controls))]
    assert all(e[0] < 1.0 for e in err[10:]), [round(e[0], 2) for e in err]


def test_cpp_mirror_ogm(tmp_path):
    """host/ogm_check.cpp through the C++ mirror: the oracle's grid, bit for bit"""
    pkg, exe = os.path.join(ROOT, "rust_robotics_b200"), str(tmp_path / "ogm_check")
    subprocess.run(["/usr/bin/g++", "-std=c++17", "-O1", os.path.join(pkg, "host", "ogm_check.cpp"), "-I", os.path.join(ROOT, "include"),
                    "-I", os.path.join(pkg, "host"), "-L", pkg, "-lpfgpu", f"-Wl,-rpath,{pkg}", "-o", exe], check=True)
    r = subprocess.run([exe], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr
    lines = r.stdout.split("\n")
    o = OO.OracleOgm(resolution=0.1, width=120, height=80)
    ranges = np.array([0.5 + 0.1 * ((i * 7) % 50) for i in range(90)])
    ranges[5] = np.inf
    for s in range(4):
        o.update_with_scan(0.5 * s - 1.0, 0.2 * s, 0.3 * s, ranges, -np.pi, 2.0 * np.pi / 90.0)
    got = np.array([float.fromhex(x) for x in lines[0].split()])
    assert np.array_equal(bits(got), bits(o.grid.ravel()))
    assert int(lines[1]) == int(o.obstacles(0.5).sum())


def test_ogm_multi_process():
    """one process per GPU (tests/mgpu_ogm_worker.py): every rank maps on its own device and hands its grid to its shard"""
    import ctypes as C
    c = C.c_int()
    rr.load_library().pfgpu_device_count(C.byref(c))
    if c.value < 2:
        pytest.skip("needs two GPUs")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nproc-per-node", "2", "--master-addr", "127.0.0.1",
           "--master-port", "29563", os.path.join(ROOT, "tests", "mgpu_ogm_worker.py"), str(4096 * 2), "8"]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0 and "MGPU_OK" in r.stdout, r.stdout[-3000:] + r.stderr[-3000:]
