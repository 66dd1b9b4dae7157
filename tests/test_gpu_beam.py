"""The beam measurement model on the GPU (DESIGN §3.11) against the oracle (tests/host/pf_beam_oracle.c, contract math, the same Philox
draws), bit for bit: the clearance table; the expected ranges on adversarial poses at the floor plan and at a tiled 8192^2 map, with
and without skipping; and at every step the particles, resample indices and recovery state on every path of the step (fused tail,
separate kernels with and without the graph, beyond 2^18 particles, the phase API, KLD-adaptive MCL, a PF whose gate stays closed on
some steps, recovery with injection, landmark / likelihood-field / beam steps on one handle, the map replaced mid-run, beam counts
that change across graph replays); the estimate to 1e-6.  Plus refusals, launch counts, the global-localisation outcome, the C++
mirror and the sharded engine."""
import ctypes as C
import math
import json
import os
import subprocess
import sys

import numpy as np
import pytest

import _beam_oracle as BO
import rust_robotics_b200 as rr
from rust_robotics_b200 import scenarios

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "beam_golden.json")
SV, SW = 0.2, 0.1
AL = (0.1, 0.6)


def fx(v):
    if isinstance(v, list):
        return np.array([fx(a) for a in v])
    return float.fromhex(v)


@pytest.fixture(scope="module")
def sc():
    return scenarios.ScanScenario(steps=14)


def _pair(sc, mode, n, seed, nmax=None, region_start=False, rec=True, thr=0.5, bm=None):
    bm = bm or {}
    cfg = rr.MonteCarloLocalizationConfig(n, nmax or n, 0.05, 2.326, 0.25, SV, SW, 0.1) if mode else rr.ParticleFilterConfig(n, thr, 0.25, SV, SW, 0.1)
    cls = rr.MonteCarloLocalizer if mode else rr.ParticleFilterLocalizer
    init = [sc.truth[0][0], sc.truth[0][1], sc.truth[0][2], 1.0]
    g = cls.try_with_region(sc.REGION, cfg, seed=seed) if region_start else cls.try_with_initial_state(init, cfg, seed=seed)
    o = BO.OracleBeam(n, threshold=thr, range_noise=0.25, velocity_noise=SV, yaw_rate_noise=SW, seed=seed, mode=mode, max_particles=nmax or n,
                      threads=min(16, os.cpu_count() or 1))
    o.init_region(sc.REGION) if region_start else o.init_state(init)
    g.set_beam_model(sc.obstacles, sc.RES, **bm)
    assert o.set_beam_map(sc.obstacles, sc.RES, **bm) == 0
    if rec:
        g.enable_recovery(*AL, sc.REGION)
        o.enable(*AL, sc.REGION)
    return g, o


def _same(g, o, what, did=False):
    assert np.array_equal(g.get_particles(), o.particles()), f"{what}: particles"
    ws, wf, p, inj = g.recovery_state()
    w, oinj = o.state()
    assert np.array_equal([ws, wf, p], w) and inj == oinj, f"{what}: recovery state"
    assert not did or np.array_equal(g.last_indices(), o.last_indices()), f"{what}: indices"
    return oinj


def _beam_steps(g, o, sc, ts, scan=None):
    out = []
    for t in ts:
        args = scan(t) if scan else sc.scan_args(t)
        e = g.try_step_beam_scan(sc.controls[t], *args)
        oe, did = o.step_beam(sc.controls[t], *args)
        assert np.allclose(e, oe, rtol=1e-6, atol=1e-6), f"step {t}: estimate"
        out.append((did, _same(g, o, f"step {t}", did)))
    return out


def _adversarial_poses(W, H, res, rng, n=200):
    hw, hh = W * res / 2.0, H * res / 2.0
    p = [[rng.uniform(-hw - 1.0, hw + 1.0), rng.uniform(-hh - 1.0, hh + 1.0), rng.uniform(-4.0, 4.0)] for _ in range(n)]
    for x in (-hw, hw, -hw + res, hw - res, math.nextafter(-hw, 0.0), math.nextafter(hw, 0.0)):   # near every grid edge
        for y in (-hh, hh - 1e-9, 0.0, math.nextafter(hh, 0.0), -hh + 0.5 * res):
            p.append([x, y, rng.uniform(-4.0, 4.0)])
    p += [[k * res, j * res, a] for k, j, a in ((0, 0, 0.0), (3, -7, math.pi / 4), (-11, 5, -3 * math.pi / 4), (40, 2, math.pi / 2))]
    p += [[math.nan, 0.0, 0.3], [0.5, math.nan, 0.0], [0.1, 0.2, math.nan], [1e300, 0.0, 0.0], [-1e300, 1e300, 1.0], [0.0, 0.0, 1e300],
          [0.0, 0.0, -1e300], [math.inf, 0.0, 0.0], [0.0, 0.0, math.inf]]
    return np.array(p, dtype=np.float64)


@pytest.mark.parametrize("case", json.load(open(GOLDEN))["cases"], ids=lambda c: c["name"])
def test_clearance_and_casts_match_oracle_golden(case):
    mask = np.array([[ch == "1" for ch in row] for row in case["mask"]], dtype=bool).reshape(case["W"], case["H"])
    v = fx(case["cfg"][:8]).tolist()
    kw = dict(sigma_hit=v[1], z_hit=v[2], z_short=v[3], z_max=v[4], z_rand=v[5], lambda_short=v[6], max_range=v[7], max_beams=case["cfg"][8])
    g = rr.MonteCarloLocalizer(rr.MonteCarloLocalizationConfig(256, 256))
    g.set_beam_model(mask, v[0], **kw)
    o = BO.OracleBeam(4)
    assert o.set_beam_map(mask, v[0], **kw) == 0
    assert g.beam_model_info() == o.beam_info() and np.array_equal(g.beam_model(), o.clearance())
    poses = fx(case["poses"])
    for c in case["casts"]:
        args = (c["B"], fx(c["angle_min"]), fx(c["angle_inc"]))
        assert np.array_equal(g.expected_scan(poses, *args), o.raycast(poses, *args))


@pytest.mark.parametrize("tiled", [False, True])
def test_expected_scan_matches_oracle(sc, tiled, monkeypatch):
    rng = np.random.default_rng(8 + tiled)
    mask = scenarios.ScanScenario.tiled(sc.obstacles, 8192) if tiled else sc.obstacles
    W, H = mask.shape
    poses = _adversarial_poses(W, H, sc.RES, rng)
    if tiled:                                                                  # and a spread of poses over the whole map
        poses = np.concatenate([poses, np.stack([rng.uniform(-W * sc.RES / 2, W * sc.RES / 2, 300), rng.uniform(-H * sc.RES / 2, H * sc.RES / 2, 300),
                                                 rng.uniform(-4, 4, 300)], axis=1)])
    o = BO.OracleBeam(4)
    assert o.set_beam_map(mask, sc.RES) == 0
    want = o.raycast(poses, 97, -math.pi, 2 * math.pi / 97)
    assert (want == 0.0).any() and (want == 30.0).any() and ((want > 0.0) & (want < 30.0)).any()
    for skip in ("1", "0"):                                                    # skipping and the one-cell-at-a-time caster
        monkeypatch.setenv("PFGPU_BEAM_SKIP", skip)
        g = rr.MonteCarloLocalizer(rr.MonteCarloLocalizationConfig(256, 256))
        g.set_beam_model(mask, sc.RES)
        if skip == "1" and tiled:
            assert np.array_equal(g.beam_model(), o.clearance())
        assert np.array_equal(g.expected_scan(poses, 97, -math.pi, 2 * math.pi / 97), want), f"skip {skip}"
        del g


def test_skip_off_gives_the_same_steps(sc, monkeypatch):
    runs = []
    for skip in ("1", "0"):
        monkeypatch.setenv("PFGPU_BEAM_SKIP", skip)
        g = rr.MonteCarloLocalizer.try_with_region(sc.REGION, rr.MonteCarloLocalizationConfig(8192, 8192, 0.05, 2.326, 0.25, SV, SW, 0.1), seed=2)
        g.set_beam_model(sc.obstacles, sc.RES)
        g.enable_recovery(*AL, sc.REGION)
        for t in range(6):
            g.try_step_beam_scan(sc.controls[t], *sc.scan_args(t))
        runs.append(g.get_particles())
    assert np.array_equal(runs[0], runs[1])


@pytest.mark.parametrize("n,path", [(4096, "fused"), (4096, "separate"), (4096, "separate_graph"), ((1 << 18) + 4096, "graph_beyond_2^18")])
def test_step_paths(sc, n, path, monkeypatch):
    monkeypatch.setenv("PFGPU_PF_FUSED", "1" if path == "fused" else "0")
    monkeypatch.setenv("PFGPU_PF_GRAPH", "0" if path == "separate" else "1")
    g, o = _pair(sc, 1, n, seed=3)
    _beam_steps(g, o, sc, range(len(sc.controls) if n < (1 << 18) else 6))


@pytest.mark.parametrize("fused", ["1", "0"])
def test_beam_counts_across_graph_replays(sc, fused, monkeypatch):
    """max_beams 90: the used count goes above and below the 64 that ride in the launch parameters from step to step, and changes
    between replays of one captured beam graph"""
    monkeypatch.setenv("PFGPU_PF_FUSED", fused)
    g, o = _pair(sc, 1, 4096, seed=12, bm=dict(max_beams=90))
    cut = [0, 200, 330, 10, 300, 0, 120, 345, 250, 0, 359, 100, 320, 5]

    def scan(t):
        r, amin, ainc = sc.scan_args(t)
        r = r.copy()
        r[:cut[t]] = np.nan
        return r, amin, ainc
    counts = [o.beam_beams(*scan(t)).shape[0] for t in range(len(sc.controls))]
    assert any(k > 64 for k in counts) and len({k for k in counts if k <= 64}) > 2
    _beam_steps(g, o, sc, range(len(sc.controls)), scan)


@pytest.mark.parametrize("rec", [False, True])
def test_pf_gate_closed_on_some_steps(sc, rec):
    g, o = _pair(sc, 0, 4096, seed=3, rec=rec, bm=dict(sigma_hit=3.0, max_beams=3, z_short=0.0))
    gates = [d for d, _ in _beam_steps(g, o, sc, range(len(sc.controls)))]
    assert any(gates) and not all(gates)


def test_phase_api(sc):
    g, o = _pair(sc, 1, 4096, seed=4)
    for t in range(len(sc.controls)):
        g.try_predict_with_control(sc.controls[t]); o.predict(sc.controls[t])
        _same(g, o, f"predict {t}")
        g.try_update_with_beam_scan(*sc.scan_args(t)); assert o.update_beam(*sc.scan_args(t)) == 0
        _same(g, o, f"update {t}")
        did = g.resample()
        assert did == o.resample()
        _same(g, o, f"resample {t}", did)


def test_kld_adaptive_global(sc):
    g, o = _pair(sc, 1, 256, seed=6, nmax=16384, region_start=True, bm=dict(sigma_hit=2.0, max_beams=3))
    counts = []
    for t in range(len(sc.controls)):
        _beam_steps(g, o, sc, [t])
        counts.append(o.count())
    assert len(set(counts)) > 1


def test_recovery_injects(sc):
    """global start with recovery on: the filter injects random particles on some steps, identically"""
    g, o = _pair(sc, 1, 4096, seed=21, region_start=True)
    injected = [inj for _, inj in _beam_steps(g, o, sc, range(len(sc.controls)))]
    assert any(i > 0 for i in injected), injected


def test_three_models_on_one_handle(sc):
    g, o = _pair(sc, 1, 4096, seed=8)
    g.set_likelihood_field(sc.obstacles, sc.RES)
    assert o.set_map(sc.obstacles, sc.RES) == 0
    lms = np.array([(1.7, -7.8), (-11.8, -9.8), (14.2, 1.2), (3.2, 10.2)])
    for t in range(len(sc.controls)):
        if t % 3 == 1:
            x, y = sc.truth[t][:2]
            obs = np.stack([np.hypot(lms[:, 0] - x, lms[:, 1] - y), lms[:, 0], lms[:, 1]], axis=1)
            e = g.try_step(sc.controls[t], obs)
            oe, did = o.step(sc.controls[t], obs)
            assert np.allclose(e, oe, rtol=1e-6, atol=1e-6)
            _same(g, o, f"landmark step {t}", did)
        elif t % 3 == 2:
            e = g.try_step_scan(sc.controls[t], *sc.scan_args(t))
            oe, did = o.step_scan(sc.controls[t], *sc.scan_args(t))
            assert np.allclose(e, oe, rtol=1e-6, atol=1e-6)
            _same(g, o, f"likelihood-field step {t}", did)
        else:
            _beam_steps(g, o, sc, [t])


def test_map_replaced_mid_run(sc):
    g, o = _pair(sc, 1, 4096, seed=9)
    other = sc.obstacles.copy()
    other[300:310, :] = True
    for t in range(len(sc.controls)):
        if t == 6:
            g.set_beam_model(other, sc.RES, sigma_hit=0.3, z_max=0.0)
            assert o.set_beam_map(other, sc.RES, sigma_hit=0.3, z_max=0.0) == 0
        if t == 10:
            g.clear_beam_model(); o.clear_beam_map()
            with pytest.raises(rr.InvalidParameter):
                g.try_step_beam_scan(sc.controls[t], *sc.scan_args(t))
            g.set_beam_model(sc.obstacles, sc.RES); o.set_beam_map(sc.obstacles, sc.RES)
        _beam_steps(g, o, sc, [t])


def test_refusals(sc):
    g = rr.MonteCarloLocalizer(rr.MonteCarloLocalizationConfig(256, 256))
    r, amin, ainc = sc.scan_args(0)
    assert g.beam_model_info() == (0, 0, 0)
    for f in (lambda: g.try_step_beam_scan([1.0, 0.0], r, amin, ainc), lambda: g.try_update_with_beam_scan(r, amin, ainc),
              lambda: g.expected_scan([[0.0, 0.0, 0.0]], 4, 0.0, 0.1), g.beam_model):
        with pytest.raises(rr.InvalidParameter):
            f()
    g.set_likelihood_field(sc.obstacles, sc.RES)                               # a likelihood field is not a beam map
    with pytest.raises(rr.InvalidParameter):
        g.try_step_beam_scan([1.0, 0.0], r, amin, ainc)
    m = np.zeros((8, 8), dtype=bool)
    for kw in (dict(resolution=0.0), dict(resolution=np.nan), dict(sigma_hit=-1.0), dict(z_hit=-0.1), dict(z_short=-0.1), dict(z_max=np.inf),
               dict(z_rand=0.0), dict(lambda_short=0.0), dict(max_range=np.inf), dict(max_beams=1), dict(resolution=1e-6, max_range=2.0),
               dict(z_rand=1e-300, z_max=0.0, max_range=1e10)):
        a = dict(resolution=0.05); a.update(kw)
        with pytest.raises(rr.InvalidParameter):
            g.set_beam_model(m, **a)
    for bad in (np.zeros((0, 4)), np.zeros((65537, 1))):
        with pytest.raises(rr.InvalidParameter):
            g.set_beam_model(bad, 0.05)
    assert g.beam_model_info() == (0, 0, 0)
    g.set_beam_model(m, 0.5, z_rand=1e-30, z_max=0.0, max_range=1.0, sigma_hit=0.3, z_hit=0.9, max_beams=100)
    o = BO.OracleBeam(4)
    assert o.set_beam_map(m, 0.5, z_rand=1e-30, z_max=0.0, max_range=1.0, sigma_hit=0.3, z_hit=0.9, max_beams=100) == 0
    L = g.beam_model_info()[2]
    assert L == o.beam_info()[2] and L > 1
    g.try_update_with_beam_scan([0.5] * L + [np.inf, np.nan, 0.0], 0.0, 0.1)   # max readings unused with z_max = 0
    with pytest.raises(rr.InvalidParameter):
        g.try_update_with_beam_scan([0.5] * (L + 1), 0.0, 0.1)
    with pytest.raises(rr.InvalidParameter):
        g.try_step_beam_scan([1.0, 0.0], [0.5], np.nan, 0.1)
    with pytest.raises(rr.InvalidParameter):
        g.try_step_beam_scan([np.inf, 0.0], [0.5], 0.0, 0.1)
    with pytest.raises(rr.InvalidParameter):
        g.expected_scan([[0.0, 0.0, 0.0]], 3, 0.0, np.inf)
    assert g.expected_scan(np.zeros((0, 3)), 5, 0.0, 0.1).shape == (0, 5)
    L_ = rr.load_library()
    assert L_.pfgpu_pf_beam_set(None, None, 1, 1, None) < 0 and L_.pfgpu_pf_update_beam(g.h, None, 3, 0.0, 0.1) < 0
    assert L_.pfgpu_pf_beam_download(g.h, None, 64) < 0 and L_.pfgpu_pf_beam_raycast(g.h, None, 2, 3, 0.0, 0.1, None) < 0


@pytest.mark.parametrize("fused", ["1", "0"])
def test_beam_step_launches_like_scan_step(sc, fused, monkeypatch):
    monkeypatch.setenv("PFGPU_PF_FUSED", fused)
    per_step = []
    for beam in (False, True):
        g = rr.MonteCarloLocalizer(rr.MonteCarloLocalizationConfig(4096, 4096), seed=1)
        g.set_likelihood_field(sc.obstacles, sc.RES)
        g.set_beam_model(sc.obstacles, sc.RES)
        launches = []
        for t in range(8):
            (g.try_step_beam_scan if beam else g.try_step_scan)(sc.controls[t], *sc.scan_args(t))
            launches.append(g.stats().kernel_launches)
        per_step.append((launches[-1] - launches[2]) / 5)
    assert per_step[0] == per_step[1], per_step


@pytest.mark.parametrize("n", [1 << 16, 1 << 18])
def test_global_localisation(n):
    sc = scenarios.ScanScenario()
    g = rr.MonteCarloLocalizer.try_with_region(sc.REGION, rr.MonteCarloLocalizationConfig(n, n, 0.05, 2.326, 0.25, SV, SW, 0.1), seed=5)
    g.set_beam_model(sc.obstacles, sc.RES)
    g.enable_recovery(0.001, 0.1, sc.REGION)
    err = [sc.error(k, g.try_step_beam_scan(sc.controls[k], *sc.scan_args(k))) for k in range(len(sc.controls))]
    assert err[-1][0] < 0.5 and err[-1][1] < 0.1, err[-1]


def test_cpp_mirror_beam(tmp_path):
    """host/beam_check.cpp through the C++ mirror: the Python mirror's numbers, bit for bit"""
    pkg, exe = os.path.join(ROOT, "rust_robotics_b200"), str(tmp_path / "beam_check")
    subprocess.run(["/usr/bin/g++", "-std=c++17", "-O1", os.path.join(pkg, "host", "beam_check.cpp"), "-I", os.path.join(ROOT, "include"),
                    "-I", os.path.join(pkg, "host"), "-L", pkg, "-lpfgpu", f"-Wl,-rpath,{pkg}", "-o", exe], check=True)
    r = subprocess.run([exe], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr
    got = np.array([float.fromhex(x) for x in r.stdout.split()])
    f = rr.MonteCarloLocalizer(rr.MonteCarloLocalizationConfig(4096, 4096, 0.05, 2.326, 0.2, 0.2, 0.1, 0.1), seed=13)
    m = np.zeros((200, 200), dtype=bool)
    m[:2, :] = m[-2:, :] = m[:, :2] = m[:, -2:] = True
    m[120:124, :130] = True
    f.set_beam_model(m, 0.1, max_range=12.0)
    f.init_region((-9.0, 9.0, -9.0, 9.0))
    want = []
    for t in range(8):
        ranges = np.array([2.0 + 0.05 * ((i * 7 + t) % 40) for i in range(90)])
        ranges[t] = np.inf
        want += list(f.try_step_beam_scan([1.0, 0.1], ranges, -np.pi, 2.0 * np.pi / 90.0)[:3])
    f.try_update_with_beam_scan(np.full(90, 3.0), -np.pi, 2.0 * np.pi / 90.0)
    want += list(f.estimate()[:3])
    want += list(f.expected_scan([[0.5, -1.0, 0.3], [3.0, 3.0, -2.0]], 5, -1.0, 0.5).ravel())
    assert got.shape == (len(want),) and np.array_equal(got, np.array(want))


def test_beam_multi_process():
    """one process per GPU (tests/mgpu_beam_worker.py): each shard equals the oracle's slice"""
    c = C.c_int()
    rr.load_library().pfgpu_device_count(C.byref(c))
    if c.value < 2:
        pytest.skip("needs 2 GPUs")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr", "127.0.0.1",
           "--master-port", "29561", os.path.join(ROOT, "tests", "mgpu_beam_worker.py"), str(4096 * 2), "10"]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0 and "MGPU_OK" in r.stdout, r.stdout[-2000:] + r.stderr[-4000:]
