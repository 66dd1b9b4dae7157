"""PF / MCL estimate and covariance (refresh_cache, pf.rs:382-413) on the device against two references, on clouds far from
the origin and far from the previous estimate.

  * Exact reference: tests/_pf_moments_cases.exact of the downloaded cloud (global slot order), est = sum w p (not divided by
    sum w), cov = sum w (p - est)(p - est)^T, every sum exactly rounded (math.fsum).
  * Oracle: OraclePF.estimate() where the oracle reaches the same state (the reference's own sequential arithmetic).

Bars (tests/_pf_moments_cases.violations):
  * estimate within 1e-12 (|exact| + 1) of the exact value (1e-6 relative would be 5 m at y = 5e6); against the oracle, plus
    the oracle's own rounding n 2^-53 sum |w p|;
  * |cov_ij - ref_ij| <= 1e-6 sqrt(ref_ii ref_jj) + (n 2^-53 max|p|)^2 against both references; diagonal entries >= 0;
  * a pose with inf or NaN gives non-finite entries exactly where the oracle's are, and the next finite cloud is finite and
    correct;
  * one cloud uploaded into handles with different histories gives bit-identical estimate and covariance, and the device's
    bits are those of tests/host/pf_moments_test.c replaying its reduction order.
"""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

import rust_robotics_b200 as rr
from rust_robotics_b200 import scenarios
import _pf_moments_cases as pm
from _oracle import OraclePF

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SW = np.deg2rad(40.0)
FAR = (-pm.UTM[0], -pm.UTM[1])                      # "the other end of the world"
dp = C.POINTER(C.c_double)


def sm_count(device=0):
    """multiprocessors of the device the handles run on, from the CUDA driver (the launch geometry of the moments kernels)"""
    cu = C.CDLL("libcuda.so.1")
    dev, sms = C.c_int(), C.c_int()
    assert cu.cuInit(0) == 0 and cu.cuDeviceGet(C.byref(dev), device) == 0
    assert cu.cuDeviceGetAttribute(C.byref(sms), 16, dev) == 0          # CU_DEVICE_ATTRIBUTE_MULTIPROCESSOR_COUNT
    return sms.value


@pytest.fixture(scope="module")
def replay(tmp_path_factory):
    """(cloud, form) -> the host replay of the device's reduction order at this GPU's geometry"""
    sms = sm_count()
    so = str(tmp_path_factory.mktemp("pf_moments") / "libpf_moments_test.so")
    subprocess.run(["gcc", "-O2", "-ffp-contract=off", "-fPIC", "-shared", "-o", so, os.path.join(ROOT, "tests", "host", "pf_moments_test.c"),
                    "-lm"], check=True)
    L = C.CDLL(so)
    L.pf_moments_replay.argtypes = [dp, C.c_size_t, C.c_int, C.c_uint, C.c_uint, C.c_uint, dp, dp]

    def run(a, form):
        a = np.ascontiguousarray(a, dtype=np.float64)
        b0, tiles, k = pm.geometry(a.shape[0], sms)
        est, cov = np.empty(4), np.empty(16)
        assert L.pf_moments_replay(a.ctypes.data_as(dp), a.shape[0], form, b0 if form == 0 else tiles, k, 1, est.ctypes.data_as(dp),
                                   cov.ctypes.data_as(dp)) == 0
        return est, cov.reshape(4, 4)
    return run


def pf(n, mode=0, seed=42, thr=0.5, sigma=0.2, sv=2.0, sw=SW, nmax=None):
    if mode == 0:
        return rr.ParticleFilterLocalizer(rr.ParticleFilterConfig(n, thr, sigma, sv, sw, 0.1), seed=seed)
    return rr.MonteCarloLocalizer(rr.MonteCarloLocalizationConfig(n, nmax or n, 0.05, 2.326, sigma, sv, sw, 0.1), seed=seed)


def oracle_pf(L, n, mode=0, seed=42, thr=0.5, sigma=0.2, sv=2.0, sw=SW, nmax=None):
    o = OraclePF(L, n, threshold=thr, range_noise=sigma, velocity_noise=sv, yaw_rate_noise=sw, seed=seed, mode=mode, max_particles=nmax or n)
    o.L.orc_pf_set_fast_search(o.h, 1)
    o.L.orc_pf_set_threads(o.h, os.cpu_count() or 1)
    return o


def device(g):
    return g.estimate(), g.calc_covariance()


def check(g, what, o=None, a=None):
    """g's estimate and covariance against the exact reference of its cloud (and the oracle's values); returns the cloud"""
    a = g.get_particles() if a is None else a
    est, cov = device(g)
    bad = pm.violations(est, cov, a)
    assert not bad, f"{what}: {bad}"
    if o is not None:
        oe, oc = o.estimate()
        oc = oc.reshape(4, 4).T
        with np.errstate(all="ignore"):
            slack = a.shape[0] * 2.0 ** -53 * np.nansum(np.abs(a[:, 4:5] * a[:, :4]), axis=0)
        bad = pm.violations(est, cov, a, (oe, oc), est_slack=slack)
        assert not bad, f"{what} (oracle): {bad}"
    return a


# ---------------------------------------------------------------------------------------------------------------------------
def _upload_params():
    out = []
    for n in pm.SIZES:
        for off in pm.OFFSETS:
            for sp in pm.SPREADS:
                for wk in pm.WEIGHTS:
                    big = n >= 1 << 16
                    if big and (off in ("1e2",) or sp in ("1m", "1cm") or wk in ("random", "zero")):
                        continue
                    if n in (1, 17) and wk == "dominant":
                        continue
                    out.append(pytest.param(n, off, sp, wk, id=f"{n}-{off}-{sp}-{wk}"))
    return out


@pytest.mark.parametrize("n,off,sp,wk", _upload_params())
def test_set_particles(oracle, replay, n, off, sp, wk):
    """set_particles into a fresh handle (previous estimate: the origin) and into one whose previous estimate is at the other
    end of the world: both within the bar of both references, bit-identical to each other and to the host replay"""
    a = pm.cloud(n, pm.OFFSETS[off], pm.SPREADS[sp], wk, seed=n + 1)
    fresh, travelled = pf(n), pf(n)
    travelled.set_particles(pm.cloud(n, FAR, 1.0, "uniform", seed=2))
    o = oracle_pf(oracle, n)
    o.set_particles(a)
    for g in (fresh, travelled):
        g.set_particles(a)
        check(g, "upload", o, a)
    e0, c0 = device(fresh)
    e1, c1 = device(travelled)
    re, rc = replay(a, 0)
    assert np.array_equal(e0, e1) and np.array_equal(c0, c1), "history changes the bits"
    assert np.array_equal(e0, re) and np.array_equal(c0, rc), "device bits differ from the replay of its reduction order"


@pytest.mark.parametrize("n", [1000, 4096, 1 << 16, 1 << 18])
@pytest.mark.parametrize("where", ["slot0", "thread_firsts", "injected_1km", "injected_10km"])
def test_outliers(oracle, replay, n, where):
    sms = sm_count()
    if where.startswith("injected"):
        a = pm.injected(n, 1e3 if where == "injected_1km" else 1e4, seed=n)
    else:
        a = pm.cloud(n, pm.UTM, 1e-2, "random", seed=3)
        a = pm.with_zero_weight_outliers(a, np.array([0]) if where == "slot0" else np.flatnonzero(pm.thread_first_slots(n, sms)))
        a[:, 4] /= a[:, 4].sum()
    g = pf(n)
    g.set_particles(a)
    o = oracle_pf(oracle, n)
    o.set_particles(a)
    check(g, where, o, a)
    re, rc = replay(a, 0)
    assert np.array_equal(device(g)[0], re) and np.array_equal(device(g)[1], rc)


@pytest.mark.parametrize("mode", [0, 1])
@pytest.mark.parametrize("n", [17, 1000, 4096, 1 << 16, 1 << 18])
def test_creation_at_utm(oracle, mode, n):
    """try_with_initial_state at UTM coordinates: the +-1 m / +-0.25 rad / +-0.5 cloud's first covariance"""
    s = (pm.UTM[0], pm.UTM[1], 40.0, -7.5)
    cfg = rr.ParticleFilterConfig(n, 0.5, 0.2, 2.0, SW, 0.1) if mode == 0 else rr.MonteCarloLocalizationConfig(n, n, 0.05, 2.326, 0.2, 2.0, SW, 0.1)
    g = (rr.ParticleFilterLocalizer if mode == 0 else rr.MonteCarloLocalizer).try_with_initial_state(s, cfg, seed=9)
    o = oracle_pf(oracle, n, mode=mode, seed=9)
    o.init_state(s)
    assert np.array_equal(g.get_particles(), o.particles())
    check(g, "try_with_initial_state", o)
    g.L.pfgpu_pf_init_state(g.h, np.ascontiguousarray([-pm.UTM[0], -pm.UTM[1], -40.0, 7.5]).ctypes.data_as(dp))
    o.init_state([-pm.UTM[0], -pm.UTM[1], -40.0, 7.5])
    check(g, "init_state after a run at the other end", o)


def test_init_region_at_utm():
    n = 4096
    g = pf(n)
    g.set_particles(pm.cloud(n, FAR, 1.0, "uniform"))
    g.init_region((pm.UTM[0] - 20.0, pm.UTM[0] + 20.0, pm.UTM[1] - 5.0, pm.UTM[1] + 5.0))
    check(g, "init_region")
    g.init_region((pm.UTM[0] - 1e-2, pm.UTM[0] + 1e-2, pm.UTM[1] - 1e-2, pm.UTM[1] + 1e-2))
    check(g, "init_region 2 cm")


def _utm_scenario(kind, steps):
    sc = scenarios.PfScenario(kind, steps=steps)
    sc.init = [sc.init[0] + pm.UTM[0], sc.init[1] + pm.UTM[1], sc.init[2], sc.init[3]]
    sc.obs = [np.column_stack([z[:, 0], z[:, 1] + pm.UTM[0], z[:, 2] + pm.UTM[1]]) for z in sc.obs]
    return sc


@pytest.mark.parametrize("fused,graph", [("1", "1"), ("0", "1"), ("0", "0"), ("1", "0")])
@pytest.mark.parametrize("kind", ["pf", "mcl"])
def test_step_paths_at_utm(oracle, replay, monkeypatch, kind, fused, graph):
    """try_step in every host form on the landmark scenario translated to UTM coordinates: particles and indices bit for bit
    the oracle's, estimate and covariance within the bar of both references and bit-identical to the replay of the form that
    ran (pf3_post_kernel when fused, the separate kernels otherwise)"""
    monkeypatch.setenv("PFGPU_PF_FUSED", fused)
    monkeypatch.setenv("PFGPU_PF_GRAPH", graph)
    steps = 30
    if kind == "pf":
        sc = _utm_scenario("c1", steps)
        n, mode, kw = 3000, 0, dict(thr=0.6, sigma=0.25)
    else:
        sc = _utm_scenario("c2", steps)
        n, mode, kw = 2048, 1, dict(sigma=0.25, sv=0.05, sw=0.02, seed=5)
    cls = rr.ParticleFilterLocalizer if mode == 0 else rr.MonteCarloLocalizer
    cfg = rr.ParticleFilterConfig(n, kw["thr"], kw["sigma"], 2.0, SW, 0.1) if mode == 0 else \
        rr.MonteCarloLocalizationConfig(n, n, 0.05, 2.326, kw["sigma"], kw["sv"], kw["sw"], 0.1)
    g = cls.try_with_initial_state(sc.init, cfg, seed=kw.get("seed", 42))
    o = oracle_pf(oracle, n, mode=mode, **kw)
    o.init_state(sc.init)
    resamples = 0
    for t in range(steps):
        obs = sc.obs[t][:: max(1, sc.obs[t].shape[0] // 24)] if kind == "mcl" else sc.obs[t]
        ge = g.try_step(sc.controls[t], obs)
        oe, did = o.step(sc.controls[t], obs)
        if did:
            resamples += 1
            assert np.array_equal(g.last_indices(), o.last_indices()), f"step {t}: indices"
        a = g.get_particles()
        assert np.array_equal(a, o.particles()), f"step {t}: particles"
        assert np.array_equal(ge, g.estimate())
        check(g, f"step {t}", o, a)
        if t % 5 == 0:
            re, rc = replay(a, 1 if fused == "1" else 0)
            assert np.array_equal(ge, re) and np.array_equal(g.calc_covariance(), rc), f"step {t}: bits differ from the replay"
    assert resamples > 0
    assert (g.stats().kernel_launches < 4 * steps) == (fused == "1")


def test_phase_api_at_utm(oracle):
    """predict, update and resample each refresh the estimate"""
    sc = _utm_scenario("c1", 8)
    n = 2048
    g = rr.ParticleFilterLocalizer.try_with_initial_state(sc.init, rr.ParticleFilterConfig(n, 0.9, 0.2, 2.0, SW, 0.1), seed=42)
    o = oracle_pf(oracle, n, thr=0.9)
    o.init_state(sc.init)
    for t in range(8):
        g.try_predict_with_control(sc.controls[t]); o.predict(sc.controls[t])
        check(g, f"predict {t}", o)
        g.try_update_with_observations(sc.obs[t]); o.update(sc.obs[t])
        check(g, f"update {t}", o)
        assert g.resample() == bool(o.resample())
        check(g, f"resample {t}", o)


def test_mcl_kld_adaptive_at_utm(oracle):
    sc = _utm_scenario("c2", 10)
    g = rr.MonteCarloLocalizer.try_with_initial_state(sc.init, rr.MonteCarloLocalizationConfig(64, 20000, 0.05, 2.326, 0.25, 0.05, 0.02, 0.1), seed=5)
    o = oracle_pf(oracle, 64, mode=1, sigma=0.25, sv=0.05, sw=0.02, seed=5, nmax=20000)
    o.init_state(sc.init)
    counts = set()
    for t in range(10):
        obs = sc.obs[t][::15]
        g.try_step(sc.controls[t], obs); o.step(sc.controls[t], obs)
        a = g.get_particles()
        assert np.array_equal(a, o.particles()), f"step {t}"
        counts.add(a.shape[0])
        check(g, f"step {t} ({a.shape[0]} particles)", o, a)
    assert len(counts) > 1


def test_recovery_injection_step():
    """a step that injects particles over a 2 km box around UTM coordinates (augmented MCL)"""
    sc = _utm_scenario("c2", 12)
    n = 4096
    g = rr.MonteCarloLocalizer.try_with_initial_state(sc.init, rr.MonteCarloLocalizationConfig(n, n, 0.05, 2.326, 0.25, 0.05, 0.02, 0.1), seed=5)
    g.enable_recovery(0.1, 0.9, (pm.UTM[0] - 1e3, pm.UTM[0] + 1e3, pm.UTM[1] - 1e3, pm.UTM[1] + 1e3))
    injected = 0
    for t in range(12):
        obs = sc.obs[t][::15] if t < 6 else np.column_stack([sc.obs[t][::15, 0] + 3.0, sc.obs[t][::15, 1:]])   # a kidnap-like jump
        g.try_step(sc.controls[t], obs)
        injected += g.recovery_state()[3]
        check(g, f"step {t}")
    assert injected > 0


def test_non_finite_poses(oracle):
    """inf / NaN in a pose: non-finite exactly where the oracle's values are; the next finite cloud is finite and correct"""
    n = 1000
    g = pf(n)
    o = oracle_pf(oracle, n)
    for col, val, w0 in [(0, np.inf, False), (1, -np.inf, False), (2, np.nan, False), (3, np.inf, True), (0, np.nan, True)]:
        a = pm.cloud(n, pm.UTM, 1e-2, "random", seed=col)
        a[n // 2, col] = val
        if w0:
            a[n // 2, 4] = 0.0
        g.set_particles(a); o.set_particles(a)
        est, cov = device(g)
        oe, oc = o.estimate()
        oc = oc.reshape(4, 4).T
        assert np.array_equal(np.isfinite(est), np.isfinite(oe)) and np.array_equal(np.isfinite(cov), np.isfinite(oc)), (col, val, w0)
        check(g, f"col {col} = {val}", o, a)
        b = pm.cloud(n, (1.0e4, -1.0e4), 1e-2, "uniform", seed=col)
        g.set_particles(b); o.set_particles(b)
        assert np.all(np.isfinite(device(g)[1]))
        check(g, "finite cloud after a non-finite one", o, b)


def test_sharded_multi_process():
    """two processes, one GPU each (tests/mgpu_pf_moments_worker.py)"""
    c = C.c_int()
    rr.load_library().pfgpu_device_count(C.byref(c))
    if c.value < 2:
        pytest.skip("needs 2 GPUs")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr", "127.0.0.1",
           "--master-port", "29551", os.path.join(ROOT, "tests", "mgpu_pf_moments_worker.py")]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0 and "MGPU_OK" in r.stdout, r.stdout[-2000:] + r.stderr[-4000:]
