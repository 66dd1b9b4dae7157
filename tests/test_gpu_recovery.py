"""Augmented MCL on the GPU (DESIGN §3.8) against the oracle (tests/host/pf_recovery_oracle.c, contract math, the same Philox
draws), bit for bit every step: particles, resample indices, (w_slow, w_fast, p) and the injected count, on every path of the step
(fused tail, separate kernels with and without the graph, beyond 2^18 particles, the phase API, KLD-adaptive MCL, a PF whose gate
stays closed on some steps); plus resets, refusals, launch counts, the kidnap / global-localisation outcomes, the C++ mirror and the
sharded engine."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

import _recovery_oracle as R
import rust_robotics_b200 as rr
from rust_robotics_b200 import scenarios

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
RN, SV, SW = 0.25, 0.05, 0.02              # config 2's noises
AL = (0.1, 0.6)                            # fast averages, so that a short run injects


def _setup(mode, n, seed, nmax=None, region_start=False):
    """a GPU filter and its oracle with recovery on, started from the scenario's pose (or from its region).  MCL: a 15 m kidnap
    (every likelihood underflows, S = 0); PF: a 1.5 m one (tiny, uneven weights: the gate opens)"""
    sc = scenarios.KidnapScenario(before=6, after=14, pitch_deg=12.0, jump=(12.0, -9.0, 0.5) if mode == 1 else (1.5, 0.0, 0.0))
    cfg = rr.MonteCarloLocalizationConfig(n, nmax or n, 0.05, 2.326, RN, SV, SW, 0.1) if mode else rr.ParticleFilterConfig(n, 0.5, RN, SV, SW, 0.1)
    cls = rr.MonteCarloLocalizer if mode else rr.ParticleFilterLocalizer
    g = cls.try_with_region(sc.REGION, cfg, seed=seed) if region_start else cls.try_with_initial_state(sc.init, cfg, seed=seed)
    o = R.OracleRecovery(n, range_noise=RN, velocity_noise=SV, yaw_rate_noise=SW, seed=seed, mode=mode, max_particles=nmax or n,
                         threads=min(8, os.cpu_count() or 1))
    o.init_region(sc.REGION) if region_start else o.init_state(sc.init)
    g.enable_recovery(*AL, sc.REGION)
    o.enable(*AL, sc.REGION)
    return g, o, sc


def _same(g, o, what, did=False):
    assert np.array_equal(g.get_particles(), o.particles()), f"{what}: particles"
    ws, wf, p, inj = g.recovery_state()
    w, oinj = o.state()
    assert np.array_equal([ws, wf, p], w) and inj == oinj, f"{what}: {(ws, wf, p, inj)} vs {(*w, oinj)}"
    assert not did or np.array_equal(g.last_indices(), o.last_indices()), f"{what}: indices"
    return oinj


def _steps(g, o, sc, ts):
    out = []
    for t in ts:
        g.try_step(sc.controls[t], sc.obs[t])
        did = o.step(sc.controls[t], sc.obs[t])[1]
        out.append((did, _same(g, o, f"step {t}", did)))
    return out


@pytest.mark.parametrize("mode,n,path", [(1, 4096, "fused"), (1, 4096, "separate"), (1, 4096, "separate_graph"), (0, 4096, "fused"),
                                         (0, 4096, "separate"), (0, 4096, "separate_graph"), (1, (1 << 18) + 4096, "graph_beyond_2^18")])
def test_step_paths(mode, n, path, monkeypatch):
    monkeypatch.setenv("PFGPU_PF_FUSED", "1" if path == "fused" else "0")
    monkeypatch.setenv("PFGPU_PF_GRAPH", "0" if path == "separate" else "1")
    g, o, sc = _setup(mode, n, seed=3)
    gates, injected = zip(*_steps(g, o, sc, range(len(sc.controls))))
    assert sum(injected) > 0
    if mode == 0:                                  # the gate stays closed on some steps; no injection follows a closed gate
        assert not all(gates) and any(gates)
        assert all(a or b == 0 for a, b in zip(gates, injected[1:]))


def test_phase_api():
    """predict / update / resample one by one, two predicts in a row, an update without a resample"""
    g, o, sc = _setup(1, 4096, seed=4)
    total = 0
    for t, (u, z) in enumerate(zip(sc.controls, sc.obs)):
        g.try_predict_with_control(u); o.predict(u)
        total += _same(g, o, f"predict {t}")
        if t % 4 == 3:                             # a second predict: nothing to inject
            g.try_predict_with_control(u); o.predict(u)
            assert _same(g, o, f"second predict {t}") == 0
        g.try_update_with_observations(z); o.update(z)
        _same(g, o, f"update {t}")
        if t % 5 != 4:                             # else an update without a resample: the next predict injects nothing
            did = g.resample()
            assert did == o.resample()
            _same(g, o, f"resample {t}", did)
    assert total > 0


def test_kld_adaptive_from_region():
    g, o, sc = _setup(1, 64, seed=6, nmax=16384, region_start=True)
    _same(g, o, "init_region")
    counts = []
    for t in range(len(sc.controls)):
        counts.append((_steps(g, o, sc, [t])[0][1], o.count()))
    assert len({c for _, c in counts}) > 1 and sum(i for i, _ in counts) > 0


@pytest.mark.parametrize("reset", ["upload", "init_state", "init_region", "enable"])
def test_resets(reset):
    """after the kidnap has made p positive: each reset zeroes (w_slow, w_fast, p) and disarms the next predict"""
    g, o, sc = _setup(1, 4096, seed=9)
    t = 0
    while g.recovery_state()[2] == 0.0:
        assert t < len(sc.controls) - 1, "p never became positive"
        _steps(g, o, sc, [t]); t += 1
    if reset == "upload":
        a = o.particles(); g.set_particles(a); o.upload(a)
    elif reset == "init_state":
        rr.api._check(g.L, g.L.pfgpu_pf_init_state(g.h, rr.api._dp(np.asarray(sc.init, dtype=np.float64)))); o.init_state(sc.init)
    elif reset == "init_region":
        g.init_region(sc.REGION); o.init_region(sc.REGION)
    else:
        g.enable_recovery(*AL, sc.REGION); o.enable(*AL, sc.REGION)
    assert g.recovery_state() == (0.0, 0.0, 0.0, 0)
    g.try_predict_with_control(sc.controls[t]); o.predict(sc.controls[t])       # disarmed: no injection
    assert _same(g, o, f"after {reset}") == 0
    g.try_update_with_observations(sc.obs[t]); o.update(sc.obs[t])
    assert g.resample() == o.resample()
    _same(g, o, f"resample after {reset}", True)


def test_refusals():
    g = rr.MonteCarloLocalizer(rr.MonteCarloLocalizationConfig(256, 256))
    box, nan, inf = (-1.0, 1.0, -1.0, 1.0), float("nan"), float("inf")
    for a_s, a_f, reg in ((0.2, 0.1, box), (0.1, 0.1, box), (0.0, 0.1, box), (0.1, 1.5, box), (nan, 0.2, box), (0.1, 0.2, None),
                          (0.1, 0.2, (1.0, 1.0, 0.0, 1.0)), (0.1, 0.2, (0.0, 1.0, 2.0, 1.0)), (0.1, 0.2, (0.0, inf, 0.0, 1.0))):
        with pytest.raises(rr.InvalidParameter):
            g.enable_recovery(a_s, a_f, reg)
    for reg in ((0.0, 0.0, 0.0, 1.0), (0.0, 1.0, nan, 1.0)):
        with pytest.raises(rr.InvalidParameter):
            g.init_region(reg)
    L = rr.load_library()
    assert L.pfgpu_pf_recovery_enable(None, 0.1, 0.2, None) < 0 and L.pfgpu_pf_init_region(None, None) < 0
    assert L.pfgpu_pf_recovery_state(None, None, None) < 0
    g.enable_recovery(0.1, 1.0, box)
    g.disable_recovery()
    assert g.recovery_state() == (0.0, 0.0, 0.0, 0)


@pytest.mark.parametrize("fused", ["1", "0"])
def test_launch_counts(fused, monkeypatch):
    """disabled: the launches of a step are those of a filter that never had recovery; enabled: one more (the filter kernel)"""
    monkeypatch.setenv("PFGPU_PF_FUSED", fused)
    sc = scenarios.KidnapScenario(before=6, after=4, pitch_deg=12.0)
    per_step = []
    for state in ("never", "disabled", "on"):
        g = rr.MonteCarloLocalizer(rr.MonteCarloLocalizationConfig(*sc.config(4096)), seed=1)
        if state != "never":
            g.enable_recovery(*AL, sc.REGION)
        if state == "disabled":
            g.disable_recovery()
        launches = []
        for t in range(8):                         # (the first steps set up the graph)
            g.try_step(sc.controls[t], sc.obs[t])
            launches.append(g.stats().kernel_launches)
        per_step.append((launches[-1] - launches[2]) / 5)
    assert per_step[0] == per_step[1] and per_step[2] == per_step[0] + 1, per_step


@pytest.mark.parametrize("n", [1 << 16, 1 << 18])
def test_kidnap_and_global_localisation(n):
    """test_recovery_oracle.py's scenarios and assertions at more particles"""
    sc, gl = scenarios.KidnapScenario(), scenarios.KidnapScenario(before=0, after=30)
    for on in (False, True):
        g = rr.MonteCarloLocalizer.try_with_initial_state(sc.init, rr.MonteCarloLocalizationConfig(*sc.config(n)), seed=3)
        if on:
            g.enable_recovery(0.01, 0.2, sc.REGION)
        err = [sc.error(k, g.try_step(sc.controls[k], sc.obs[k])) for k in range(len(sc.controls))]
        assert max(err[:sc.before]) < 0.5
        assert (min(err[sc.before:]) < 1.0 and err[-1] < 1.0) if on else min(err[sc.before:]) > 5.0
    g = rr.MonteCarloLocalizer.try_with_region(gl.REGION, rr.MonteCarloLocalizationConfig(*gl.config(n)), seed=5)
    g.enable_recovery(0.01, 0.2, gl.REGION)
    assert min(gl.error(k, g.try_step(gl.controls[k], gl.obs[k])) for k in range(5)) < 1.0


def test_cpp_mirror_recovery(tmp_path):
    """host/recovery_check.cpp through the C++ mirror: the Python mirror's numbers, bit for bit"""
    pkg, exe = os.path.join(ROOT, "rust_robotics_b200"), str(tmp_path / "recovery_check")
    subprocess.run(["/usr/bin/g++", "-std=c++17", "-O1", os.path.join(pkg, "host", "recovery_check.cpp"), "-I", os.path.join(ROOT, "include"),
                    "-I", os.path.join(pkg, "host"), "-L", pkg, "-lpfgpu", f"-Wl,-rpath,{pkg}", "-o", exe], check=True)
    r = subprocess.run([exe], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr
    got = np.array([float.fromhex(x) if "0x" in x else float(x) for x in r.stdout.split()])
    f = rr.MonteCarloLocalizer.try_with_region((-10.0, 10.0, -10.0, 10.0), rr.MonteCarloLocalizationConfig(4096, 4096, 0.05, 2.326, 0.5, 0.1, 0.05, 0.1),
                                               seed=11)
    f.enable_recovery(0.1, 0.6, (-10.0, 10.0, -10.0, 10.0))
    want = []
    for t in range(10):
        z = [(1.0e4 if t >= 5 else float(np.sqrt((2.0 + 0.1 * t - lx) ** 2 + (-1.0 - ly) ** 2)), lx, ly)
             for lx, ly in ((10.0, 0.0), (0.0, 10.0), (-10.0, 0.0), (0.0, -10.0))]
        e = f.try_step([1.0, 0.0], z)
        want += [*f.recovery_state(), e[0], e[1]]
    assert got.shape == (len(want),) and np.array_equal(got, np.array(want, dtype=np.float64)) and any(want[3::6])


def test_recovery_multi_process():
    """one process per GPU (tests/mgpu_recovery_worker.py): each shard equals the oracle's slice"""
    c = C.c_int()
    rr.load_library().pfgpu_device_count(C.byref(c))
    if c.value < 2:
        pytest.skip("needs 2 GPUs")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr", "127.0.0.1",
           "--master-port", "29553", os.path.join(ROOT, "tests", "mgpu_recovery_worker.py"), str(4096 * 2), "20"]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0 and "MGPU_OK" in r.stdout, r.stdout[-2000:] + r.stderr[-4000:]
