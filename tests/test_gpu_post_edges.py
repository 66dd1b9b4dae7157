"""The resample path on adversarial weight vectors (_weight_cases.py) against the CPU oracle, bit for bit.

FastSLAM 1.0: the catalogue's raw weights are uploaded with set_state and one step with no observations, u = (0, 0) and
q00 = q11 = 0 hands them to the post kernel untouched (the poses stay exact); a second step follows.  Every post-kernel shape
(shared tiles with one or several values per thread, global tiles, one tile per SM, the in-process sharded engine).
PF / MCL: the phase API's resample() (the separate-kernel resampler) on the same catalogue, and the default step above 2^18
particles, which runs the separate kernels too."""
import ctypes as C
import math
import os

import numpy as np
import pytest

import rust_robotics_b200 as rr
from rust_robotics_b200 import scenarios
import _weight_cases as wc
from _oracle import OracleFS, OraclePF

pytestmark = pytest.mark.gpu

SEED = 17
M = 4
RTOL = 1e-6

# name -> (n, environment of the post kernel's shape)
SHAPES = {
    "1000": (1000, {}),
    "1024": (1024, {}),
    "4096x8": (4096, {"PFGPU_POST_TILES": "2"}),
    "5000global": (5000, {"PFGPU_POST_SMEM_CAP": "0", "PFGPU_POST_TILES": "3"}),
    "65536": (65536, {}),
    "65537": (65537, {}),
    "131072": (131072, {}),
}
FULL = ("1000", "1024", "4096x8")


def _params():
    out = []
    for s, (n, _) in SHAPES.items():
        for c in wc.CASES:
            if (s in FULL or c.finite) and n >= c.min_n and not (c.small and n > 8192):
                out.append(pytest.param(s, c, id=f"{s}-{c.name}"))
    return out


def _state(n, w):
    p = np.empty((n, 4))
    p[:, 0] = w                                        # rows are (w, x, y, yaw)
    p[:, 1] = np.arange(n) * 0.5 + 1.0
    p[:, 2] = -np.arange(n) * 0.25 - 1.0
    p[:, 3] = np.linspace(-3.0, 3.0, n)
    lm = np.zeros((n, M, 6))
    lm[:, :, 0] = np.arange(n)[:, None] + 1.0
    lm[:, :, 1] = np.arange(M)[None, :] + 2.0
    lm[:, :, 2] = lm[:, :, 5] = 1000.0
    return p, lm


def same(a, b):
    """bitwise equality that also holds NaN positions and the sign of zero"""
    a, b = np.asarray(a), np.asarray(b)
    na, nb = np.isnan(a), np.isnan(b)
    return (a.shape == b.shape and np.array_equal(na, nb) and np.array_equal(a[~na], b[~nb])
            and np.array_equal(np.signbit(a[~na]), np.signbit(b[~nb])))


def _exact_cdf_resamples(g):
    out = (C.c_ulonglong * 32)()
    assert g.L.pfgpu_fs_post_trace(g.h, out) == 0
    return int(out[11])


def _check_neff(gn, o, case):
    on = o.last_neff()
    if case.path == "border":
        assert same(gn, on), f"N_eff {gn!r} vs oracle {on!r}"
    else:
        assert gn == pytest.approx(on, rel=1e-9) or same(gn, on), f"N_eff {gn!r} vs oracle {on!r}"


def _run_fs(oracle, n, case, make, set_state, step, best, indices, state, neff=lambda g: g.last_neff()):
    w = case.build(n, SEED, 0, L=oracle, family="fs")
    nth = case.nth(n, w)
    g = make(nth)
    o = OracleFS(oracle, n, M, seed=SEED, q00=0.0, q11=0.0, nth=nth)
    p, lm = _state(n, w)
    set_state(g, p, lm)
    o.set_state(p, lm)
    resamples = 0
    for t in range(2):
        did = step(g)
        assert did == bool(o.step([0.0, 0.0], [])), f"step {t}: gate"
        if did:
            resamples += 1
            gi, oi = indices(g), o.last_indices()
            assert np.array_equal(gi, oi), f"step {t}: {int((gi != oi).sum())} indices differ, first at {np.flatnonzero(gi != oi)[:4]}"
        gp, gl = state(g)
        op, ol = o.state()
        assert same(gp, op), f"step {t}: pose / weight rows {np.flatnonzero(~((gp == op) | (np.isnan(gp) & np.isnan(op))).all(axis=1))[:5]}"
        assert np.array_equal(gl, ol), f"step {t}: landmarks"
        if case.name not in wc.NO_BEST:
            assert best(g) == o.best(), f"step {t}: best particle"
        if t == 0:
            _check_neff(neff(g), o, case)
    return g, w, resamples


@pytest.mark.parametrize("shape,case", _params())
def test_fs_post_kernel_on_weight_cases(oracle, monkeypatch, shape, case):
    n, env = SHAPES[shape]
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    g, w, resamples = _run_fs(
        oracle, n, case,
        make=lambda nth: rr.FastSlam1(n, M, rr.FsConfig(q00=0.0, q11=0.0, nth=nth), seed=SEED),
        set_state=lambda g, p, lm: g.set_state(p, lm),
        step=lambda g: g.fastslam_update([0.0, 0.0], []),
        best=lambda g: g.get_best_particle()[0],
        indices=lambda g: g.last_indices(),
        state=lambda g: g.state())
    if env.get("PFGPU_POST_SMEM_CAP") == "0":
        assert g.post_shape()[3] == "global"
    if case.path == "serial":
        assert g.stats().serial_fallbacks > 0, "the sums never took the serial walk"
    pow2_cert = n & (n - 1) == 0 and n <= 1 << 16
    first_exact = _exact_cdf_resamples(g)
    if resamples and case.path == "refused" and pow2_cert:
        assert first_exact >= 1, "the certificate never refused"
    if resamples and case.path == "cert" and pow2_cert:
        assert first_exact < resamples, "the certified CDF was never used"


SHARDED = {"2x2048": (2, 2048), "4x960": (4, 3840)}


@pytest.mark.parametrize("layout", list(SHARDED))
@pytest.mark.parametrize("case", [c for c in wc.CASES if c.finite or c.name.startswith("all_")], ids=lambda c: c.name)
def test_fs_sharded_post_on_weight_cases(oracle, layout, case):
    world, n = SHARDED[layout]
    nl = n // world

    def make(nth):
        return rr.FastSlam1.create_sharded_local(n, M, [0] * world, rr.FsConfig(q00=0.0, q11=0.0, nth=nth), seed=SEED)

    def set_state(ranks, p, lm):
        for r, g in enumerate(ranks):
            g.set_state(p[r * nl:(r + 1) * nl], lm[r * nl:(r + 1) * nl])

    def best(ranks):
        bs = {g.get_best_particle()[0] for g in ranks}
        assert len(bs) == 1, f"ranks disagree on the best particle: {bs}"
        return bs.pop()

    def neff(ranks):
        ns = [g.last_neff() for g in ranks]
        assert all(same(x, ns[0]) for x in ns), f"ranks disagree on N_eff: {ns}"
        return ns[0]

    def state(ranks):
        ss = [g.state() for g in ranks]
        return np.concatenate([s[0] for s in ss]), np.concatenate([s[1] for s in ss])

    _run_fs(oracle, n, case, make, set_state,
            step=lambda ranks: rr.FastSlam1.step_all(ranks, [0.0, 0.0], []),
            best=best, indices=lambda ranks: np.concatenate([g.last_indices() for g in ranks]), state=state, neff=neff)


# ------------------------------------------------------------------------------------------------
# PF / MCL
# ------------------------------------------------------------------------------------------------
PF_CASES = [c for c in wc.CASES if not c.name.startswith("border")]
MONOTONE = lambda c: c.finite and c.name != "neg_zero"        # noqa: E731  (-0.0 keeps the CDF non-decreasing, but the
                                                               # linear scan is the reference either way)


def _pf_params():
    out = []
    for n in (1000, 4099, 300000):
        for mode in (0, 1):
            for c in PF_CASES:
                if n > 8192 and (not MONOTONE(c) or c.small):
                    continue                                     # the reference's linear scan over 300 000 values per slot
                out.append(pytest.param(n, mode, c, id=f"{n}-{'mcl' if mode else 'pf'}-{c.name}"))
    return out


@pytest.mark.parametrize("n,mode,case", _pf_params())
def test_pf_phase_resample_on_weight_cases(oracle, n, mode, case):
    w = case.build(n, SEED, 0, L=oracle, family="pf")
    a = np.empty((n, 5))
    a[:, 0] = np.arange(n) * 0.5
    a[:, 1] = -np.arange(n) * 0.25
    a[:, 2] = np.linspace(-3.0, 3.0, n)
    a[:, 3] = 1.0
    a[:, 4] = w
    if mode == 0:
        g = rr.ParticleFilterLocalizer(rr.ParticleFilterConfig(n, 1.0, 0.2, 2.0, np.deg2rad(40.0), 0.1), seed=SEED)
    else:
        g = rr.MonteCarloLocalizer(rr.MonteCarloLocalizationConfig(n, n, 0.05, 2.326, 0.2, 2.0, np.deg2rad(40.0), 0.1), seed=SEED)
    o = OraclePF(oracle, n, threshold=1.0, seed=SEED, mode=mode, max_particles=n)
    o.L.orc_pf_set_fast_search(o.h, 1 if n > 8192 else 0)
    o.L.orc_pf_set_threads(o.h, os.cpu_count() or 1)
    g.set_particles(a)
    o.set_particles(a)
    assert same(g.get_particles(), o.particles())
    did = g.resample()
    assert did == bool(o.resample())
    if did:
        gi, oi = g.last_indices(), o.last_indices()
        assert np.array_equal(gi, oi), f"{int((gi != oi).sum())} indices differ, first at {np.flatnonzero(gi != oi)[:4]}: {gi[gi != oi][:4]} vs {oi[gi != oi][:4]}"
    assert same(g.get_particles(), o.particles())


def _assert_cov_close(got, want):
    got, want = np.asarray(got).reshape(4, 4), np.asarray(want).reshape(4, 4)
    d = np.maximum(np.abs(np.diag(want)), 1e-9 * np.max(np.abs(np.diag(want))) + 1e-300)
    err = np.max(np.abs(got - want) / np.sqrt(np.outer(d, d)))
    assert err < RTOL, f"covariance: {err}"


def _pf_default_step_run(oracle, kind, n, steps, k=None):
    if kind == "pf":
        sc = scenarios.PfScenario("c1", steps=steps)
        g = rr.ParticleFilterLocalizer.try_with_initial_state(sc.init, rr.ParticleFilterConfig(n, 1.0, 0.25, 2.0, np.deg2rad(40.0), 0.1), seed=5)
        o = OraclePF(oracle, n, threshold=1.0, range_noise=0.25, seed=5)
    else:
        sc = scenarios.PfScenario("c2", steps=steps)
        g = rr.MonteCarloLocalizer.try_with_initial_state(sc.init, rr.MonteCarloLocalizationConfig(n, n, 0.05, 2.326, 0.25, 0.05, 0.02, 0.1), seed=5)
        o = OraclePF(oracle, n, range_noise=0.25, velocity_noise=0.05, yaw_rate_noise=0.02, seed=5, mode=1, max_particles=n)
    o.L.orc_pf_set_fast_search(o.h, 1)
    o.L.orc_pf_set_threads(o.h, os.cpu_count() or 1)
    o.init_state(sc.init)
    resamples = 0
    for t in range(steps):
        obs = sc.obs[t] if k is None else sc.obs[t][:k]
        ge = g.try_step(sc.controls[t], obs)
        oe, did = o.step(sc.controls[t], obs)
        np.testing.assert_allclose(ge, oe, rtol=RTOL, atol=1e-9, err_msg=f"step {t}: estimate")
        if did:
            resamples += 1
            gi, oi = g.last_indices(), o.last_indices()
            assert np.array_equal(gi, oi), f"step {t}: {int((gi != oi).sum())} indices differ"
    assert np.array_equal(g.get_particles(), o.particles()), "particles differ from the oracle"
    _oe, oc = o.estimate()
    _assert_cov_close(g.calc_covariance().T.ravel(), oc)
    assert resamples > 0 and g.stats().serial_fallbacks == 0
    return g


def test_pf_default_step_above_2_18_bit_exact(oracle):
    """C1 at 300 000 particles: the step replays the separate kernels from a CUDA graph (the fused tail stops at 2^18)"""
    g = _pf_default_step_run(oracle, "pf", 300000, 10)
    assert g.stats().kernel_launches > 4 * 10


def test_mcl_config2_step_bit_exact(oracle):
    """bench config 2: MCL, 2^20 particles x 360 beams (observations staged in device memory), 3 steps"""
    sc = scenarios.PfScenario("c2", steps=1)
    assert sc.obs[0].shape[0] == 360
    _pf_default_step_run(oracle, "mcl", 1 << 20, 3)
