"""The likelihood-field scan model on the GPU (DESIGN §3.9) against the oracle (tests/host/pf_lfield_oracle.c, contract math, the same
Philox draws), bit for bit: the distance field and the factor table, and at every step the particles, resample indices and the
recovery state, on every path of the step (fused tail, separate kernels with and without the graph, beyond 2^18 particles, the phase
API, KLD-adaptive MCL, a PF whose gate stays closed on some steps, recovery on, landmark steps between scan steps, the map replaced
mid-run); the estimate to 1e-6.  Plus refusals, launch counts, the global-localisation outcome, the C++ mirror and the sharded
engine."""
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np
import pytest

import _lfield_oracle as LF
import rust_robotics_b200 as rr
from rust_robotics_b200 import scenarios

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "lfield_golden.json")
SV, SW = 0.2, 0.1
AL = (0.1, 0.6)


def fx(v):
    if isinstance(v, list):
        return np.array([fx(a) for a in v])
    return float.fromhex(v)


@pytest.fixture(scope="module")
def sc():
    return scenarios.ScanScenario(steps=14)


def _pair(sc, mode, n, seed, nmax=None, region_start=False, rec=True, thr=0.5, lf=None):
    lf = lf or {}
    cfg = rr.MonteCarloLocalizationConfig(n, nmax or n, 0.05, 2.326, 0.25, SV, SW, 0.1) if mode else rr.ParticleFilterConfig(n, thr, 0.25, SV, SW, 0.1)
    cls = rr.MonteCarloLocalizer if mode else rr.ParticleFilterLocalizer
    init = [sc.truth[0][0], sc.truth[0][1], sc.truth[0][2], 1.0]
    g = cls.try_with_region(sc.REGION, cfg, seed=seed) if region_start else cls.try_with_initial_state(init, cfg, seed=seed)
    o = LF.OracleLField(n, threshold=thr, range_noise=0.25, velocity_noise=SV, yaw_rate_noise=SW, seed=seed, mode=mode, max_particles=nmax or n,
                        threads=min(8, os.cpu_count() or 1))
    o.init_region(sc.REGION) if region_start else o.init_state(init)
    g.set_likelihood_field(sc.obstacles, sc.RES, **lf)
    assert o.set_map(sc.obstacles, sc.RES, **lf) == 0
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


def _scan_steps(g, o, sc, ts):
    out = []
    for t in ts:
        e = g.try_step_scan(sc.controls[t], *sc.scan_args(t))
        oe, did = o.step_scan(sc.controls[t], *sc.scan_args(t))
        assert np.allclose(e, oe, rtol=1e-6, atol=1e-6), f"step {t}: estimate"
        out.append((did, _same(g, o, f"step {t}", did)))
    return out


@pytest.mark.parametrize("case", json.load(open(GOLDEN))["cases"], ids=lambda c: c["name"])
def test_tables_match_oracle(case):
    mask = np.array([[ch == "1" for ch in row] for row in case["mask"]], dtype=bool).reshape(case["W"], case["H"])
    cfg = fx(case["cfg"][:5]).tolist()
    kw = dict(sigma_hit=cfg[1], z_hit=cfg[2], z_rand=cfg[3], max_range=cfg[4], max_beams=case["cfg"][5])
    g = rr.MonteCarloLocalizer(rr.MonteCarloLocalizationConfig(256, 256))
    g.set_likelihood_field(mask, cfg[0], **kw)
    o = LF.OracleLField(4)
    assert o.set_map(mask, cfg[0], **kw) == 0
    D, q, L = g.likelihood_field()
    oD, oq = o.tables()
    assert L == case["L"] and np.array_equal(D, oD) and np.array_equal(q, oq)


def test_tables_match_oracle_4096():
    rng = np.random.default_rng(4)
    mask = rng.random((4096, 4096)) < 0.002
    mask[1000:1010, 200:3000] = True
    g = rr.MonteCarloLocalizer(rr.MonteCarloLocalizationConfig(256, 256))
    g.set_likelihood_field(mask, 0.05)
    o = LF.OracleLField(4)
    assert o.set_map(mask, 0.05) == 0
    D, q, L = g.likelihood_field()
    oD, oq = o.tables()
    assert L == o.info()[2] and np.array_equal(D, oD) and np.array_equal(q, oq)


@pytest.mark.parametrize("n,path", [(4096, "fused"), (4096, "separate"), (4096, "separate_graph"), ((1 << 18) + 4096, "graph_beyond_2^18")])
def test_step_paths(sc, n, path, monkeypatch):
    monkeypatch.setenv("PFGPU_PF_FUSED", "1" if path == "fused" else "0")
    monkeypatch.setenv("PFGPU_PF_GRAPH", "0" if path == "separate" else "1")
    g, o = _pair(sc, 1, n, seed=3)
    _scan_steps(g, o, sc, range(len(sc.controls)))


@pytest.mark.parametrize("fused", ["1", "0"])
def test_beam_list_beyond_the_launch_parameters(sc, fused, monkeypatch):
    """max_beams 90: about 90 used beams per scan, more than ride in the launch parameters, so they go through the device buffer"""
    monkeypatch.setenv("PFGPU_PF_FUSED", fused)
    g, o = _pair(sc, 1, 4096, seed=12, lf=dict(max_beams=90))
    assert all(o.beams(*sc.scan_args(t)).shape[0] > 64 for t in range(len(sc.controls)))
    _scan_steps(g, o, sc, range(len(sc.controls)))


@pytest.mark.parametrize("rec", [False, True])
def test_pf_gate_closed_on_some_steps(sc, rec):
    g, o = _pair(sc, 0, 4096, seed=3, rec=rec, lf=dict(sigma_hit=1.5, max_beams=3))
    gates = [d for d, _ in _scan_steps(g, o, sc, range(len(sc.controls)))]
    assert any(gates) and not all(gates)


def test_phase_api(sc):
    g, o = _pair(sc, 1, 4096, seed=4)
    for t in range(len(sc.controls)):
        g.try_predict_with_control(sc.controls[t]); o.predict(sc.controls[t])
        _same(g, o, f"predict {t}")
        g.try_update_with_scan(*sc.scan_args(t)); assert o.update_scan(*sc.scan_args(t)) == 0
        _same(g, o, f"update {t}")
        did = g.resample()
        assert did == o.resample()
        _same(g, o, f"resample {t}", did)


def test_kld_adaptive_global(sc):
    """a flat model (sigma_hit 2, 3 beams), so that the cloud keeps several KLD bins and the count changes from step to step"""
    g, o = _pair(sc, 1, 256, seed=6, nmax=16384, region_start=True, lf=dict(sigma_hit=2.0, max_beams=3))
    counts = []
    for t in range(len(sc.controls)):
        _scan_steps(g, o, sc, [t])
        counts.append(o.count())
    assert len(set(counts)) > 1


def test_landmark_steps_between_scan_steps(sc):
    g, o = _pair(sc, 1, 4096, seed=8)
    lms = np.array([(1.7, -7.8), (-11.8, -9.8), (14.2, 1.2), (3.2, 10.2)])
    for t in range(len(sc.controls)):
        if t % 3 == 1:
            x, y = sc.truth[t][:2]
            obs = np.stack([np.hypot(lms[:, 0] - x, lms[:, 1] - y), lms[:, 0], lms[:, 1]], axis=1)
            e = g.try_step(sc.controls[t], obs)
            oe, did = o.step(sc.controls[t], obs)
            assert np.allclose(e, oe, rtol=1e-6, atol=1e-6)
            _same(g, o, f"landmark step {t}", did)
        else:
            _scan_steps(g, o, sc, [t])


def test_map_replaced_mid_run(sc):
    g, o = _pair(sc, 1, 4096, seed=9)
    other = sc.obstacles.copy()
    other[300:310, :] = True
    for t in range(len(sc.controls)):
        if t == 6:
            g.set_likelihood_field(other, sc.RES, sigma_hit=0.3)
            assert o.set_map(other, sc.RES, sigma_hit=0.3) == 0
        if t == 10:
            g.clear_likelihood_field(); o.clear_map()
            with pytest.raises(rr.InvalidParameter):
                g.try_step_scan(sc.controls[t], *sc.scan_args(t))
            g.set_likelihood_field(sc.obstacles, sc.RES); o.set_map(sc.obstacles, sc.RES)
        _scan_steps(g, o, sc, [t])


def test_refusals(sc):
    g = rr.MonteCarloLocalizer(rr.MonteCarloLocalizationConfig(256, 256))
    r, amin, ainc = sc.scan_args(0)
    assert g.likelihood_field_info() == (0, 0, 0)
    with pytest.raises(rr.InvalidParameter):
        g.try_step_scan([1.0, 0.0], r, amin, ainc)                               # no map
    with pytest.raises(rr.InvalidParameter):
        g.try_update_with_scan(r, amin, ainc)
    m = np.zeros((8, 8), dtype=bool)
    for kw in (dict(resolution=0.0), dict(resolution=np.nan), dict(sigma_hit=-1.0), dict(z_hit=-0.1), dict(z_rand=0.0),
               dict(max_range=np.inf), dict(max_beams=1), dict(z_rand=1e-300, max_range=1e10)):
        a = dict(resolution=0.05); a.update(kw)
        with pytest.raises(rr.InvalidParameter):
            g.set_likelihood_field(m, **a)
    for bad in (np.zeros((0, 4)), np.zeros((65537, 1))):
        with pytest.raises(rr.InvalidParameter):
            g.set_likelihood_field(bad, 0.05)
    g.set_likelihood_field(m, 0.5, z_rand=1e-30, max_range=1.0, sigma_hit=0.3, z_hit=0.9, max_beams=100)
    L = g.likelihood_field_info()[2]
    assert L == 9
    g.try_update_with_scan([0.5] * L, 0.0, 0.1)
    with pytest.raises(rr.InvalidParameter):
        g.try_update_with_scan([0.5] * (L + 1), 0.0, 0.1)
    with pytest.raises(rr.InvalidParameter):
        g.try_step_scan([1.0, 0.0], [0.5], np.nan, 0.1)
    with pytest.raises(rr.InvalidParameter):
        g.try_step_scan([np.inf, 0.0], [0.5], 0.0, 0.1)
    L_ = rr.load_library()
    assert L_.pfgpu_pf_lfield_set(None, None, 1, 1, None) < 0 and L_.pfgpu_pf_update_scan(g.h, None, 3, 0.0, 0.1) < 0
    assert L_.pfgpu_pf_lfield_download(g.h, None, None, 5) < 0


@pytest.mark.parametrize("fused", ["1", "0"])
def test_scan_step_launches_like_landmark_step(sc, fused, monkeypatch):
    monkeypatch.setenv("PFGPU_PF_FUSED", fused)
    per_step = []
    for scan in (False, True):
        g = rr.MonteCarloLocalizer(rr.MonteCarloLocalizationConfig(4096, 4096), seed=1)
        g.set_likelihood_field(sc.obstacles, sc.RES)
        launches = []
        for t in range(8):
            if scan:
                g.try_step_scan(sc.controls[t], *sc.scan_args(t))
            else:
                g.try_step(sc.controls[t], [[5.0, 1.0, 1.0], [4.0, -2.0, 0.5]])
            launches.append(g.stats().kernel_launches)
        per_step.append((launches[-1] - launches[2]) / 5)
    assert per_step[0] == per_step[1], per_step


@pytest.mark.parametrize("n", [1 << 16, 1 << 18])
def test_global_localisation(n):
    sc = scenarios.ScanScenario()
    g = rr.MonteCarloLocalizer.try_with_region(sc.REGION, rr.MonteCarloLocalizationConfig(n, n, 0.05, 2.326, 0.25, SV, SW, 0.1), seed=5)
    g.set_likelihood_field(sc.obstacles, sc.RES)
    g.enable_recovery(0.001, 0.1, sc.REGION)
    err = [sc.error(k, g.try_step_scan(sc.controls[k], *sc.scan_args(k))) for k in range(len(sc.controls))]
    assert err[-1][0] < 0.5 and err[-1][1] < 0.1, err[-1]


def test_cpp_mirror_lfield(tmp_path):
    """host/lfield_check.cpp through the C++ mirror: the Python mirror's numbers, bit for bit"""
    pkg, exe = os.path.join(ROOT, "rust_robotics_b200"), str(tmp_path / "lfield_check")
    subprocess.run(["/usr/bin/g++", "-std=c++17", "-O1", os.path.join(pkg, "host", "lfield_check.cpp"), "-I", os.path.join(ROOT, "include"),
                    "-I", os.path.join(pkg, "host"), "-L", pkg, "-lpfgpu", f"-Wl,-rpath,{pkg}", "-o", exe], check=True)
    r = subprocess.run([exe], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr
    got = np.array([float.fromhex(x) for x in r.stdout.split()])
    f = rr.MonteCarloLocalizer(rr.MonteCarloLocalizationConfig(4096, 4096, 0.05, 2.326, 0.2, 0.2, 0.1, 0.1), seed=13)
    m = np.zeros((200, 200), dtype=bool)
    m[:2, :] = m[-2:, :] = m[:, :2] = m[:, -2:] = True
    m[120:124, :130] = True
    f.set_likelihood_field(m, 0.1)
    f.init_region((-9.0, 9.0, -9.0, 9.0))
    want = []
    for t in range(8):
        ranges = np.array([2.0 + 0.05 * ((i * 7 + t) % 40) for i in range(90)])
        ranges[t] = np.inf
        want += list(f.try_step_scan([1.0, 0.1], ranges, -np.pi, 2.0 * np.pi / 90.0)[:3])
    f.try_update_with_scan(np.full(90, 3.0), -np.pi, 2.0 * np.pi / 90.0)
    want += list(f.estimate()[:3])
    assert got.shape == (len(want),) and np.array_equal(got, np.array(want))


def test_lfield_multi_process():
    """one process per GPU (tests/mgpu_lfield_worker.py): each shard equals the oracle's slice"""
    c = C.c_int()
    rr.load_library().pfgpu_device_count(C.byref(c))
    if c.value < 2:
        pytest.skip("needs 2 GPUs")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr", "127.0.0.1",
           "--master-port", "29557", os.path.join(ROOT, "tests", "mgpu_lfield_worker.py"), str(4096 * 2), "10"]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0 and "MGPU_OK" in r.stdout, r.stdout[-2000:] + r.stderr[-4000:]
