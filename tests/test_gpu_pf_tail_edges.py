"""The PF / MCL step tail on adversarial raw weights against the CPU oracle, bit for bit: the fused tail (pf3_post_kernel, the
default for one GPU and up to 2^18 particles) and the separate kernels (PFGPU_PF_FUSED=0).

(a) Through the test hook pfgpu_test_pf_tail, which writes w_raw into the handle and issues exactly what a step issues after
    its predict + likelihood kernel.  Cases: every one of _weight_cases.CASES (the border ones where n = 2^k makes
    threshold = nth / n exact) and _pf_tail_cases.TAIL_CASES (+inf among zeros with the first inf in tile 0, on a tile edge,
    in the last tile and in the last slot; all inf; inf with NaN; finite weights whose sum overflows; a subnormal S), at one
    tile, K = 1 over many tiles, K > 1 with a partial last tile, and 2^18, in PF and MCL modes.  Compared: the gate, S, N_eff
    (PF), the ancestors, the particles and weights bit for bit (NaN-aware), and the estimate and covariance within the bars of
    _pf_moments_cases.violations.
(b) Through the public step, no hook: the motion noise is zero and the control (0, 0), so poses stay exact, and landmark
    ranges measured exactly from a pose that some particles sit on.  With sigma = 0.05 and 360 ranges each such particle's
    likelihood overflows to +inf (7.98^360 ~ 1e325) while the others are 0; with sigma = 1e-11 32 ranges do the same and the
    step fits in a CUDA graph.  A few wrong ranges at the end turn the overflowed products into inf * 0 = NaN (S = NaN, the
    uniform fallback).  A finite cloud checks N_eff on n * threshold and one ulp either side.  Each case runs fused, separate
    from the graph and separate without it; the {inf, 0} case also once with augmented MCL's recovery on (its filter skips a
    non-finite S) and once KLD-adaptive."""
import ctypes as C
import math

import numpy as np
import pytest

import rust_robotics_b200 as rr
import _pf_moments_cases as pm
import _pf_tail_cases as tc
import _weight_cases as wc
from _oracle import OraclePF

pytestmark = pytest.mark.gpu

SEED = 29
SW = np.deg2rad(40.0)
c_dp = C.POINTER(C.c_double)
PATHS = {"fused": {}, "separate": {"PFGPU_PF_FUSED": "0"}}


def sm_count(device=0):
    """multiprocessors of the device, from the CUDA driver (the tail's shape depends on it)"""
    cu = C.CDLL("libcuda.so.1")
    dev, sms = C.c_int(), C.c_int()
    assert cu.cuInit(0) == 0 and cu.cuDeviceGet(C.byref(dev), device) == 0
    assert cu.cuDeviceGetAttribute(C.byref(sms), 16, dev) == 0          # CU_DEVICE_ATTRIBUTE_MULTIPROCESSOR_COUNT
    return sms.value


def same(a, b):
    """bitwise equality that also holds NaN positions and the sign of zero"""
    a, b = np.asarray(a), np.asarray(b)
    na, nb = np.isnan(a), np.isnan(b)
    return (a.shape == b.shape and np.array_equal(na, nb) and np.array_equal(a[~na], b[~nb])
            and np.array_equal(np.signbit(a[~na]), np.signbit(b[~nb])))


def make(n, mode, thr=1.0, sigma=0.2, sv=2.0, sw=SW, nmax=None):
    if mode == 0:
        return rr.ParticleFilterLocalizer(rr.ParticleFilterConfig(n, thr, sigma, sv, sw, 0.1), seed=SEED)
    return rr.MonteCarloLocalizer(rr.MonteCarloLocalizationConfig(n, nmax or n, 0.05, 2.326, sigma, sv, sw, 0.1), seed=SEED)


# ---------------------------------------------------------------------------------------------------------------------------
# (a) through the hook
# ---------------------------------------------------------------------------------------------------------------------------
def _case_params():
    out = []
    for size, n in tc.SIZES.items():
        names = [("wc", c.name) for c in wc.CASES
                 if not (c.name.startswith("border") and n & (n - 1)) and not (c.small and n > 16384) and n >= c.min_n]
        names += [("tail", c.name) for c in tc.TAIL_CASES]
        for src, name in names:
            for mode in (0, 1):
                for path in PATHS:
                    out.append(pytest.param(size, src, name, mode, path, id=f"{size}-{'mcl' if mode else 'pf'}-{path}-{name}"))
    return out


_REF = {}


def _reference(oracle, size, src, name, mode):
    """(w_raw, threshold, oracle tail) of a case, shared by the fused and the separate run"""
    key = (size, src, name, mode)
    if key not in _REF:
        n = tc.SIZES[size]
        if src == "wc":
            c = wc.BY_NAME[name]
            w = c.build(n, SEED, 0, L=oracle, family="pf")
            nth = c.nth(n, w)
            thr = min(1.0, nth / n)
        else:
            _tiles, k = tc.pf3_shape(n, sm_count())
            w = tc.TAIL_BY_NAME[name].build(n, tc.NT * k)
            thr = 1.0
        _REF.clear()
        _REF[key] = (w, thr, tc.oracle_tail(w, mode, thr, SEED))
    return _REF[key]


def run_tail(g, w):
    """the hook: (S, Q, last cumulative weight, N_eff), gate"""
    w = np.ascontiguousarray(w, dtype=np.float64)
    s4, gate = np.empty(4), C.c_int()
    rc = g.L.pfgpu_test_pf_tail(g.h, w.ctypes.data_as(c_dp), w.size, s4.ctypes.data_as(c_dp), C.byref(gate))
    assert rc == 0, g.L.pfgpu_last_error().decode()
    return s4, bool(gate.value)


def test_hook_refuses_a_wrong_count():
    g = make(256, 0)
    w = np.ones(255)
    assert g.L.pfgpu_test_pf_tail(g.h, w.ctypes.data_as(c_dp), w.size, None, None) != 0


@pytest.mark.parametrize("size,src,name,mode,path", _case_params())
def test_pf_tail_on_weight_cases(oracle, monkeypatch, size, src, name, mode, path):
    n = tc.SIZES[size]
    w, thr, (did, neff, oidx, op, _oest, _ocov) = _reference(oracle, size, src, name, mode)
    for k, v in PATHS[path].items():
        monkeypatch.setenv(k, v)
    g = make(n, mode, thr)
    g.set_particles(tc.cloud(np.ones(n)))
    l0 = g.stats().kernel_launches
    s4, gate = run_tail(g, w)
    launches = g.stats().kernel_launches - l0
    assert (launches == 1) == (path == "fused"), f"{launches} launches: not the {path} tail"
    assert gate == did, f"gate {gate} vs oracle {did} (N_eff {s4[3]!r} vs {neff!r}, threshold {thr!r})"
    S = wc.seq_sum(w)
    assert same(s4[0], S), f"S {s4[0]!r} vs {S!r}"
    if mode == 0:
        if src == "wc" and wc.BY_NAME[name].path == "border":
            assert same(s4[3], neff), f"N_eff {s4[3]!r} vs oracle {neff!r}"
        else:
            assert s4[3] == pytest.approx(neff, rel=1e-9) or same(s4[3], neff), f"N_eff {s4[3]!r} vs oracle {neff!r}"
    gi = g.last_indices()
    if did:
        bad = np.flatnonzero(gi != oidx)
        assert bad.size == 0, f"{bad.size} ancestors differ, first at {bad[:4]}: {gi[bad[:4]]} vs {oidx[bad[:4]]}"
    else:
        assert gi.size == 0
    gp = g.get_particles()
    assert same(gp, op), f"particle rows differ: {np.flatnonzero(~((gp == op) | (np.isnan(gp) & np.isnan(op))).all(axis=1))[:5]}"
    bad = pm.violations(g.estimate(), g.calc_covariance(), op)
    assert not bad, bad


# ---------------------------------------------------------------------------------------------------------------------------
# (b) through the public step
# ---------------------------------------------------------------------------------------------------------------------------
POSE = (10.0, 5.0)
STEP_PATHS = {"fused": {}, "separate_graph": {"PFGPU_PF_FUSED": "0"}, "separate_plain": {"PFGPU_PF_FUSED": "0", "PFGPU_PF_GRAPH": "0"}}
N_B = 4096


def landmarks(k, wrong=0):
    """k landmark observations (range, x, y) measured exactly from POSE; the last `wrong` ranges are 5 m too long"""
    j = np.arange(k)
    lx = POSE[0] + (3.0 + 0.01 * j) * np.cos(2.0 * np.pi * j / k)
    ly = POSE[1] + (3.0 + 0.01 * j) * np.sin(2.0 * np.pi * j / k)
    dx, dy = POSE[0] - lx, POSE[1] - ly
    r = np.sqrt(dx * dx + dy * dy)
    r[k - wrong:] += 5.0
    return np.stack([r, lx, ly], axis=1)


def on_pose_cloud(n, seed):
    """every fifth particle from slot 2 (and the last) on POSE, the others 50 m and more away (likelihood 0).  Slot 0 is off
    POSE: a first inf there would coincide with PF's fallback index"""
    rng = np.random.default_rng(seed)
    a = np.empty((n, 5))
    a[:, 0] = POSE[0] + 50.0 + rng.uniform(0.0, 10.0, n)
    a[:, 1] = POSE[1] + rng.uniform(-10.0, 10.0, n)
    on = (np.arange(n) % 5 == 2) | (np.arange(n) == n - 1)
    a[on, 0], a[on, 1] = POSE
    a[:, 2] = rng.uniform(-3.0, 3.0, n)
    a[:, 3] = 0.0
    a[:, 4] = 1.0 / n
    return a


def near_pose_cloud(n, seed):
    """a finite cloud around POSE: every likelihood finite and positive"""
    rng = np.random.default_rng(seed)
    a = on_pose_cloud(n, seed)
    a[:, 0] = POSE[0] + rng.normal(0.0, 0.05, n)
    a[:, 1] = POSE[1] + rng.normal(0.0, 0.05, n)
    return a


def _run_steps(oracle, g, o, cloud, obs_seq, before_step=None):
    g.set_particles(cloud)
    o.set_particles(cloud)
    if before_step:
        before_step(g)
    out = []
    for t, obs in enumerate(obs_seq):
        ge = g.try_step([0.0, 0.0], obs)
        oe, did = o.step([0.0, 0.0], obs)
        gi, oi = g.last_indices(), (o.last_indices() if did else np.zeros(0, dtype=np.uint32))
        assert gi.size == oi.size, f"step {t}: gate {gi.size > 0} vs oracle {bool(did)}"
        bad = np.flatnonzero(gi != oi)
        assert bad.size == 0, f"step {t}: {bad.size} ancestors differ, first at {bad[:4]}: {gi[bad[:4]]} vs {oi[bad[:4]]}"
        gp, op = g.get_particles(), o.particles()
        assert same(gp, op), f"step {t}: particle rows differ"
        bad = pm.violations(ge, g.calc_covariance(), op)
        assert not bad, f"step {t}: {bad}"
        out.append(did)
    return out


def _oracle(oracle, n, mode, thr, sigma, nmax=None):
    o = OraclePF(oracle, n, threshold=thr, range_noise=sigma, velocity_noise=0.0, yaw_rate_noise=0.0, seed=SEED, mode=mode,
                 max_particles=nmax or n)
    o.L.orc_pf_set_fast_search(o.h, 0)
    return o


# name -> (sigma, observation count, wrong ranges at the end, class of S on the second step)
STEP_CASES = {
    "inf_zero_360": (0.05, 360, 0, "S_inf"),
    "inf_zero_32": (1e-11, 32, 0, "S_inf"),
    "nan_360": (0.05, 360, 10, "S_nan"),
    "nan_32": (1e-11, 32, 2, "S_nan"),
}


def _normalised(oracle, cloud, sigma, obs):
    """the oracle's normalised weights of `cloud` under `obs` (predict with (0, 0) and update, no resample)"""
    o = _oracle(oracle, cloud.shape[0], 0, 0.0, sigma)
    o.set_particles(cloud)
    o.predict([0.0, 0.0])
    o.update(obs)
    return o.particles()[:, 4]


@pytest.mark.parametrize("mode", [0, 1], ids=["pf", "mcl"])
@pytest.mark.parametrize("path", list(STEP_PATHS))
@pytest.mark.parametrize("case", list(STEP_CASES))
def test_step_with_overflowing_likelihoods(oracle, monkeypatch, case, path, mode):
    sigma, k, wrong, cls = STEP_CASES[case]
    obs = landmarks(k, wrong)
    cloud = on_pose_cloud(N_B, 3)
    # the second step's normalised weights show the class: NaN on the matching particles (S = inf), or uniform (S = NaN)
    wn = _normalised(oracle, cloud, sigma, obs)
    on = cloud[:, 0] == POSE[0]
    if cls == "S_inf":
        assert np.all(np.isnan(wn[on])) and np.all(wn[~on] == 0.0)
    else:
        assert np.all(wn == 1.0 / N_B)
    for kk, v in STEP_PATHS[path].items():
        monkeypatch.setenv(kk, v)
    g = make(N_B, mode, 1.0, sigma, 0.0, 0.0)
    o = _oracle(oracle, N_B, mode, 1.0, sigma)
    # a first step without observations (uniform weights, N_eff = n: PF keeps its cloud) so that the second one replays a graph
    did = _run_steps(oracle, g, o, cloud, [np.zeros((0, 3)), obs])
    assert did[1] == (cls == "S_inf" or mode == 1)       # S = inf: N_eff = 0; S = NaN: uniform, N_eff = n
    if mode == 0 and cls == "S_inf":
        assert np.all(g.last_indices() == 0)             # every slot takes PF's fallback


def test_step_recovery_skips_non_finite_S(oracle):
    """augmented MCL's filter: S = inf leaves w_slow and w_fast as the step before set them"""
    sigma, k, wrong, _ = STEP_CASES["inf_zero_360"]
    g = make(N_B, 0, 1.0, sigma, 0.0, 0.0)
    o = _oracle(oracle, N_B, 0, 1.0, sigma)
    g.set_particles(on_pose_cloud(N_B, 3))
    o.set_particles(on_pose_cloud(N_B, 3))
    g.enable_recovery(0.001, 0.1, region=(0.0, 20.0, -5.0, 15.0))
    states = []
    for obs in (np.zeros((0, 3)), landmarks(k, wrong)):
        g.try_step([0.0, 0.0], obs)
        _oe, did = o.step([0.0, 0.0], obs)
        states.append(g.recovery_state())
        gi = g.last_indices()
        assert np.array_equal(gi, o.last_indices() if did else np.zeros(0, dtype=np.uint32))
    ws, wf, p, inj = states[0]
    assert ws == 0.001 and wf == 0.1 and p == 0.0 and inj == 0        # w_avg = S / n = 1 on the first step
    assert states[1][:2] == (ws, wf) and states[1][2] == 0.0
    assert same(g.get_particles(), o.particles())


def test_step_kld_adaptive_on_inf_zero_cloud(oracle):
    """the KLD-adaptive resample (its own draw kernel) on the same S = inf step"""
    sigma, k, wrong, _ = STEP_CASES["inf_zero_360"]
    g = make(N_B, 1, 1.0, sigma, 0.0, 0.0, nmax=2 * N_B)
    o = _oracle(oracle, N_B, 1, 1.0, sigma, nmax=2 * N_B)
    cloud = on_pose_cloud(N_B, 3)
    g.set_particles(cloud)
    o.set_particles(cloud)
    for t, obs in enumerate((np.zeros((0, 3)), landmarks(k, wrong))):
        g.try_step([0.0, 0.0], obs)
        o.step([0.0, 0.0], obs)
        gi, oi = g.last_indices(), o.last_indices()
        assert np.array_equal(gi, oi), f"step {t}: ancestors"
        assert same(g.get_particles(), o.particles()), f"step {t}: particles"
    assert np.unique(oi).size == 1                       # every draw takes MCL's fallback, the last particle


@pytest.mark.parametrize("path", list(STEP_PATHS))
@pytest.mark.parametrize("direction", [0, 1, -1], ids=["eq", "up", "down"])
def test_step_neff_on_the_threshold(oracle, monkeypatch, path, direction):
    """N_eff exactly on n * threshold and one ulp either side (n = 2^12, threshold = N_eff / n exact)"""
    sigma = 0.2
    obs = landmarks(8)
    cloud = near_pose_cloud(N_B, 4)
    o = _oracle(oracle, N_B, 0, 0.0, sigma)
    o.set_particles(cloud)
    o.step([0.0, 0.0], np.zeros((0, 3)))
    o.predict([0.0, 0.0])
    o.update(obs)
    neff = o.neff()
    nth = neff if direction == 0 else math.nextafter(neff, math.inf if direction > 0 else -math.inf)
    thr = nth / N_B
    assert thr * N_B == nth and 0.0 < thr < 1.0
    for kk, v in STEP_PATHS[path].items():
        monkeypatch.setenv(kk, v)
    g = make(N_B, 0, thr, sigma, 0.0, 0.0)
    o = _oracle(oracle, N_B, 0, thr, sigma)
    did = _run_steps(oracle, g, o, cloud, [np.zeros((0, 3)), obs])
    assert did == [False, direction > 0]
