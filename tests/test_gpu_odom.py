"""The odometry motion model on the GPU (DESIGN §3.14) against the oracle (tests/host/pf_odom_oracle.c, contract math, the same Philox
draws), bit for bit: at every step the particles, resample indices and recovery state on every path of the step (fused tail,
separate kernels with and without the graph, beyond 2^18 particles, the phase API, KLD-adaptive MCL, a PF whose gate stays closed on
some steps, recovery with injection, landmark / likelihood-field / beam weights, odometry and velocity steps alternating on one
handle); the estimate to 1e-6.  Plus launch counts against the velocity twin, refusals, the C++ mirror, global localisation with the
beam model on OdomScenario, and the sharded engine."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

import _odom_oracle as OO
import rust_robotics_b200 as rr
from rust_robotics_b200 import scenarios

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SV, SW = 0.2, 0.1
AL = (0.1, 0.6)
ALPHA = (0.1, 0.05, 0.1, 0.05)


@pytest.fixture(scope="module")
def sc():
    return scenarios.OdomScenario(legs=((4, 1.0, 0.05), (3, 0.0, 0.0), (3, 0.0, 1.0), (3, -0.5, 0.0), (3, 1.0, -0.05)))


def _pair(sc, mode, n, seed, nmax=None, rec=True, thr=0.5, region_start=False):
    cfg = rr.MonteCarloLocalizationConfig(n, nmax or n, 0.05, 2.326, 0.25, SV, SW, 0.1) if mode else rr.ParticleFilterConfig(n, thr, 0.25, SV, SW, 0.1)
    cls = rr.MonteCarloLocalizer if mode else rr.ParticleFilterLocalizer
    init = [sc.start[0], sc.start[1], sc.start[2], 0.0]
    g = cls.try_with_region(sc.REGION, cfg, seed=seed) if region_start else cls.try_with_initial_state(init, cfg, seed=seed)
    o = OO.OracleOdom(n, threshold=thr, range_noise=0.25, velocity_noise=SV, yaw_rate_noise=SW, seed=seed, mode=mode, max_particles=nmax or n,
                      threads=min(16, os.cpu_count() or 1))
    o.init_region(sc.REGION) if region_start else o.init_state(init)
    g.set_odometry_noise(*ALPHA)
    assert o.set_odom_noise(ALPHA) == 0
    g.set_likelihood_field(sc.obstacles, sc.RES)
    assert o.set_map(sc.obstacles, sc.RES) == 0
    g.set_beam_model(sc.obstacles, sc.RES)
    assert o.set_beam_map(sc.obstacles, sc.RES) == 0
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


def _landmarks(sc, t):
    x, y, _ = sc.truth[t]
    lms = [(-10.0, -8.0), (12.0, -9.0), (10.0, 10.0), (-14.0, 9.0), (0.0, 0.0)]
    return np.array([[np.hypot(x - a, y - b) + 0.05 * ((t * 3 + j) % 5 - 2), a, b] for j, (a, b) in enumerate(lms)])


def _step(g, o, sc, t, model):
    """one odometry step of `model` on both; 'vel' is the velocity twin with the scenario's equivalent control (likelihood field)"""
    a, b = sc.odom_pair(t)
    if model == "lm":
        e, (oe, did) = g.try_step_odometry(a, b, _landmarks(sc, t)), o.step_odom(a, b, _landmarks(sc, t))
    elif model == "lf":
        e, (oe, did) = g.try_step_scan_odometry(a, b, *sc.scan_args(t)), o.step_scan_odom(a, b, *sc.scan_args(t))
    elif model == "beam":
        e, (oe, did) = g.try_step_beam_scan_odometry(a, b, *sc.scan_args(t)), o.step_beam_odom(a, b, *sc.scan_args(t))
    else:
        e, (oe, did) = g.try_step_scan(sc.controls[t], *sc.scan_args(t)), o.step_scan(sc.controls[t], *sc.scan_args(t))
    assert np.allclose(e, oe, rtol=1e-6, atol=1e-6), f"step {t} ({model}): estimate"
    return did, _same(g, o, f"step {t} ({model})", did)


@pytest.mark.parametrize("model", ["lm", "lf", "beam"])
@pytest.mark.parametrize("n,path", [(4096, "fused"), (4096, "separate"), (4096, "separate_graph"), ((1 << 18) + 4096, "graph_beyond_2^18")])
def test_step_paths(sc, n, path, model, monkeypatch):
    monkeypatch.setenv("PFGPU_PF_FUSED", "1" if path == "fused" else "0")
    monkeypatch.setenv("PFGPU_PF_GRAPH", "0" if path == "separate" else "1")
    g, o = _pair(sc, 1, n, seed=3)
    for t in range(sc.steps if n < (1 << 18) else 5):
        _step(g, o, sc, t, model)


@pytest.mark.parametrize("fused", ["1", "0"])
def test_motion_kinds_alternate(sc, fused, monkeypatch):
    """odometry and velocity steps, and the three measurement models, alternating on one handle: the graph is re-keyed each time"""
    monkeypatch.setenv("PFGPU_PF_FUSED", fused)
    g, o = _pair(sc, 1, 4096, seed=8)
    order = ["lf", "vel", "lf", "lm", "vel", "beam", "beam", "vel", "lf", "lm"]
    for t in range(min(sc.steps, len(order))):
        _step(g, o, sc, t, order[t])


@pytest.mark.parametrize("rec", [False, True])
def test_pf_gate_closed_on_some_steps(sc, rec):
    g, o = _pair(sc, 0, 4096, seed=4, rec=rec, thr=0.05)
    dids = [_step(g, o, sc, t, "lm")[0] for t in range(sc.steps)]
    assert not all(dids)


def test_phase_api(sc):
    g, o = _pair(sc, 0, 4096, seed=6)
    for t in range(6):
        a, b = sc.odom_pair(t)
        g.try_predict_with_odometry(a, b)
        assert o.predict_odom(a, b) == 0
        _same(g, o, f"predict {t}")
        g.try_update_with_scan(*sc.scan_args(t))
        assert o.update_scan(*sc.scan_args(t)) == 0
        did = g.resample()
        assert did == o.resample()
        _same(g, o, f"resample {t}", did)


def test_kld_adaptive(sc):
    """from a global start under a flat likelihood field (sigma_hit 2 m, 3 beams), so that the cloud keeps many bins for a while"""
    g, o = _pair(sc, 1, 256, seed=9, nmax=16384, region_start=True)
    g.set_likelihood_field(sc.obstacles, sc.RES, sigma_hit=2.0, max_beams=3)
    assert o.set_map(sc.obstacles, sc.RES, sigma_hit=2.0, max_beams=3) == 0
    counts = []
    for t in range(sc.steps):
        _step(g, o, sc, t, "lf")
        counts.append(g.particle_count())
        assert counts[-1] == o.count()
    assert len(set(counts)) > 1


def test_recovery_injects(sc):
    g, o = _pair(sc, 1, 4096, seed=10, region_start=True)
    injected = [_step(g, o, sc, t, "beam")[1] for t in range(sc.steps)]
    assert any(injected)


def test_no_motion_moves_nothing(sc):
    g, _ = _pair(sc, 1, 4096, seed=2, rec=False)
    p0 = g.get_particles()
    g.try_predict_with_odometry((1.0, 2.0, 3.0), (1.0, 2.0, 3.0))
    assert np.array_equal(g.get_particles() == p0, np.ones_like(p0, dtype=bool))


@pytest.mark.parametrize("fused", ["1", "0"])
@pytest.mark.parametrize("model", ["lm", "lf", "beam"])
def test_odometry_step_launches_like_velocity_step(sc, fused, model, monkeypatch):
    monkeypatch.setenv("PFGPU_PF_FUSED", fused)
    per_step = []
    for odom in (False, True):
        g = rr.MonteCarloLocalizer(rr.MonteCarloLocalizationConfig(4096, 4096), seed=1)
        g.set_likelihood_field(sc.obstacles, sc.RES)
        g.set_beam_model(sc.obstacles, sc.RES)
        launches = []
        for t in range(8):
            a, b = sc.odom_pair(t)
            if model == "lm":
                g.try_step_odometry(a, b, _landmarks(sc, t)) if odom else g.try_step(sc.controls[t], _landmarks(sc, t))
            elif model == "lf":
                g.try_step_scan_odometry(a, b, *sc.scan_args(t)) if odom else g.try_step_scan(sc.controls[t], *sc.scan_args(t))
            else:
                g.try_step_beam_scan_odometry(a, b, *sc.scan_args(t)) if odom else g.try_step_beam_scan(sc.controls[t], *sc.scan_args(t))
            launches.append(g.stats().kernel_launches)
        per_step.append((launches[-1] - launches[2]) / 5)
    assert per_step[0] == per_step[1], per_step


def test_refusals(sc):
    g = rr.ParticleFilterLocalizer(rr.ParticleFilterConfig(256), seed=1)
    assert g.odometry_noise() == (0.2, 0.2, 0.2, 0.2)
    for bad in ((-0.1, 0.2, 0.2, 0.2), (0.2, np.nan, 0.2, 0.2), (0.2, 0.2, np.inf, 0.2)):
        with pytest.raises(rr.InvalidParameter):
            g.set_odometry_noise(*bad)
    assert g.odometry_noise() == (0.2, 0.2, 0.2, 0.2)
    g.set_odometry_noise(0.0, 0.0, 0.3, 0.0)
    assert g.odometry_noise() == (0.0, 0.0, 0.3, 0.0)
    p0 = g.get_particles()
    for a, b in (((0.0, 0.0, np.nan), (1.0, 0.0, 0.0)), ((0.0, 0.0, 0.0), (np.inf, 0.0, 0.0)), ((-np.inf, 0.0, 0.0), (0.0, 0.0, 0.0))):
        with pytest.raises(rr.InvalidParameter):
            g.try_predict_with_odometry(a, b)
        with pytest.raises(rr.InvalidParameter):
            g.try_step_odometry(a, b, [[1.0, 0.0, 0.0]])
        with pytest.raises(rr.InvalidParameter):
            g.try_step_scan_odometry(a, b, sc.scans[0], sc.ANGLE_MIN, sc.ANGLE_INC)
    with pytest.raises(rr.InvalidParameter):
        g.try_predict_with_odometry((0.0, 0.0), (1.0, 0.0, 0.0))
    with pytest.raises(rr.InvalidParameter):                          # no map loaded
        g.try_step_beam_scan_odometry((0.0, 0.0, 0.0), (0.1, 0.0, 0.0), sc.scans[0], sc.ANGLE_MIN, sc.ANGLE_INC)
    assert np.array_equal(g.get_particles(), p0)


def test_global_localisation_beam():
    sc = scenarios.OdomScenario()
    n = 1 << 16
    g = rr.MonteCarloLocalizer.try_with_region(sc.REGION, rr.MonteCarloLocalizationConfig(n, n, 0.05, 2.326, 0.25, SV, SW, 0.1), seed=5)
    g.set_beam_model(sc.obstacles, sc.RES)
    g.enable_recovery(0.001, 0.1, sc.REGION)
    err = [sc.error(t, g.try_step_beam_scan_odometry(*sc.odom_pair(t), *sc.scan_args(t))) for t in range(sc.steps)]
    assert err[-1][0] < 0.5 and err[-1][1] < 0.1, err[-1]


def test_cpp_mirror_odom(tmp_path):
    """host/odom_check.cpp through the C++ mirror: the Python mirror's numbers, bit for bit"""
    pkg, exe = os.path.join(ROOT, "rust_robotics_b200"), str(tmp_path / "odom_check")
    subprocess.run(["/usr/bin/g++", "-std=c++17", "-O1", os.path.join(pkg, "host", "odom_check.cpp"), "-I", os.path.join(ROOT, "include"),
                    "-I", os.path.join(pkg, "host"), "-L", pkg, "-lpfgpu", f"-Wl,-rpath,{pkg}", "-o", exe], check=True)
    r = subprocess.run([exe], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr
    got = np.array([float.fromhex(x) for x in r.stdout.split()])
    odom = [(0.0, 0.0, 0.0), (0.1, 0.0, 0.01), (0.1, 0.0, 0.4), (0.1, 0.0, 0.4), (0.05, -0.02, 0.41), (0.15, 0.02, 0.42), (0.25, 0.06, 0.43)]
    want = []
    p = rr.ParticleFilterLocalizer(rr.ParticleFilterConfig(4096), seed=7)
    p.set_odometry_noise(0.1, 0.05, 0.1, 0.05)
    z = [[5.0, 3.0, 4.0], [4.0, -2.0, 3.5], [6.5, 1.0, -6.0]]
    for t in range(len(odom) - 1):
        want += list(p.try_step_odometry(odom[t], odom[t + 1], z)[:3])
    want += list(p.odometry_noise())
    f = rr.MonteCarloLocalizer(rr.MonteCarloLocalizationConfig(4096, 4096), seed=13)
    m = np.zeros((200, 200), dtype=bool)
    m[:2, :] = m[-2:, :] = m[:, :2] = m[:, -2:] = True
    m[120:124, :130] = True
    f.set_beam_model(m, 0.1, max_range=12.0)
    f.init_region((-9.0, 9.0, -9.0, 9.0))
    for t in range(len(odom) - 1):
        ranges = np.array([2.0 + 0.05 * ((i * 7 + t) % 40) for i in range(90)])
        want += list(f.try_step_beam_scan_odometry(odom[t], odom[t + 1], ranges, -np.pi, 2.0 * np.pi / 90.0)[:3])
    f.try_predict_with_odometry(odom[0], odom[1])
    want += list(f.estimate()[:3])
    assert got.shape == (len(want),) and np.array_equal(got, np.array(want))


def test_odom_multi_process():
    """one process per GPU (tests/mgpu_odom_worker.py): each shard equals the oracle's slice"""
    c = C.c_int()
    rr.load_library().pfgpu_device_count(C.byref(c))
    if c.value < 2:
        pytest.skip("needs 2 GPUs")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr", "127.0.0.1",
           "--master-port", "29563", os.path.join(ROOT, "tests", "mgpu_odom_worker.py"), str(4096 * 2)]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0 and "MGPU_OK" in r.stdout, r.stdout[-2000:] + r.stderr[-4000:]
