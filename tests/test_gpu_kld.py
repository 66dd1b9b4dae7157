"""KLD-adaptive MCL (resample_adaptive, mcl.rs:322-365; pf_kld.cuh) on the device against the oracle, on the adversarial clouds
of tests/_kld_cases.py: stops on both sides of the stop kernel's 1024-draw chunks, generations that run to n_max, bin keys at
the quantiser's edges, hash-set probe chains that collide and wrap, 2^16-bin clouds, and weights that stress the draw.

Each case is uploaded into a fresh filter and into the oracle and resampled once (the phase API).  Bit for bit: the particle
count, the ancestor of every draw and every particle with its weight 1/n.  Then a few ordinary steps with landmark observations
run at the new count (so the count grows or shrinks again and every launch is re-sized), on every step form: the default step,
separate kernels with and without the graph (PFGPU_PF_FUSED / PFGPU_PF_GRAPH; an adaptive filter takes the separate kernels
whatever they say, and the results must not depend on them), and predict / update / resample one by one.  After every step the
same comparison, and the estimate and covariance within the bars of tests/test_gpu_pf_moments.py."""
import numpy as np
import pytest

import rust_robotics_b200 as rr
import _kld_cases as K
import _pf_moments_cases as pm
from _oracle import OraclePF

pytestmark = pytest.mark.gpu

RN, SV, SW, DT = 0.5, 0.3, 0.2, 0.1
FORMS = {"fused": ("1", "1"), "graph": ("0", "1"), "separate": ("0", "0"), "phase": None}
STEPS = 3


def bits(a):
    return np.ascontiguousarray(a, dtype=np.float64).view(np.uint64)


def same(a, b):
    """bit for bit, except that a NaN made by arithmetic matches any NaN (the device's and the host's NaN payloads differ)"""
    a, b = np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64)
    if a.shape != b.shape:
        return False
    na, nb = np.isnan(a), np.isnan(b)
    return np.array_equal(na, nb) and np.array_equal(bits(np.where(na, 0.0, a)), bits(np.where(nb, 0.0, b)))


def pair(oracle, c, cloud):
    g = rr.MonteCarloLocalizer(rr.MonteCarloLocalizationConfig(c.n_min, c.n_max, c.eps, c.z, RN, SV, SW, DT), seed=c.seed)
    o = OraclePF(oracle, c.n_min, range_noise=RN, velocity_noise=SV, yaw_rate_noise=SW, dt=DT, seed=c.seed, mode=1, max_particles=c.n_max,
                 kld_epsilon=c.eps, kld_z=c.z)
    o.L.orc_pf_set_fast_search(o.h, int(c.monotone))     # the lower bound is the linear scan there (tests/test_kld_oracle.py)
    o.L.orc_pf_set_threads(o.h, 8)
    g.set_particles(cloud)
    o.set_particles(cloud)
    return g, o


def compare(g, o, what, resampled=True, moments=True):
    n = o.count()
    assert g.particle_count() == n, f"{what}: count {g.particle_count()} vs oracle {n}"
    if resampled:
        gi, oi = g.last_indices(), o.last_indices()
        assert np.array_equal(gi, oi), f"{what}: ancestors differ at draws {np.flatnonzero(gi != oi)[:5] if gi.size == oi.size else (gi.size, oi.size)}"
    gp, op = g.get_particles(), o.particles()
    assert same(gp, op), f"{what}: particles differ at rows {np.flatnonzero(~((gp == op) | (np.isnan(gp) & np.isnan(op))).all(axis=1))[:5]}"
    if resampled:
        assert np.all(gp[:, 4] == 1.0 / n), what
    if moments:
        est, cov = g.estimate(), g.calc_covariance()
        oe, oc = o.estimate()
        with np.errstate(all="ignore"):                 # (a cloud at 1e300 m has no finite rounding bar: it is inf there)
            bad = pm.violations(est, cov, gp)
            assert not bad, f"{what}: {bad}"
            slack = n * 2.0 ** -53 * np.nansum(np.abs(gp[:, 4:5] * gp[:, :4]), axis=0)
            bad = pm.violations(est, cov, gp, (oe, oc.reshape(4, 4).T), est_slack=slack)
            assert not bad, f"{what} (oracle): {bad}"


def observations(cloud, t):
    """four landmarks 10 m around the middle of the cloud's finite positions, ranges from that point"""
    p = cloud[:, :2][np.all(np.isfinite(cloud[:, :2]) & (np.abs(cloud[:, :2]) < 1e6), axis=1)]
    cx, cy = (np.median(p, axis=0) if p.size else (0.0, 0.0))
    cx, cy = cx + 0.1 * t, cy
    lms = [(cx + 10.0, cy), (cx, cy + 10.0), (cx - 10.0, cy), (cx, cy - 10.0)]
    return np.array([[10.0 + 0.3 * ((j + t) % 3 - 1), lx, ly] for j, (lx, ly) in enumerate(lms)])


def run(oracle, monkeypatch, c, form):
    if FORMS[form] is not None:
        monkeypatch.setenv("PFGPU_PF_FUSED", FORMS[form][0])
        monkeypatch.setenv("PFGPU_PF_GRAPH", FORMS[form][1])
    cloud = c.cloud(oracle)
    g, o = pair(oracle, c, cloud)
    assert g.resample() and o.resample() == 1
    if c.expect is not None:
        assert o.count() == c.expect, f"{c.name}: the oracle stops at {o.count()}, the case was built for {c.expect}"
    compare(g, o, f"{c.name} resample", moments=c.n_max <= (1 << 18))
    counts = [o.count()]
    u = np.array([1.0, 0.1])
    for t in range(STEPS):
        obs = observations(cloud, t)
        if form == "phase":
            g.try_predict_with_control(u); o.predict(u)
            compare(g, o, f"{c.name} predict {t}", resampled=False, moments=False)
            g.try_update_with_observations(obs); o.update(obs)
            compare(g, o, f"{c.name} update {t}", resampled=False, moments=False)
            assert g.resample() and o.resample() == 1
        else:
            g.try_step(u, obs)
            o.step(u, obs)
        compare(g, o, f"{c.name} {form} step {t}", moments=t == STEPS - 1 or o.count() <= (1 << 18))
        counts.append(o.count())
    return g, o, counts


def _params():
    out = []
    for c in K.CASES:
        for form in (["phase"] if c.big else FORMS):
            out.append(pytest.param(c.name, form, id=f"{c.name}-{form}"))
    return out


@pytest.mark.parametrize("name,form", _params())
def test_kld_case_matches_oracle(oracle, monkeypatch, name, form):
    run(oracle, monkeypatch, K.BY_NAME[name], form)


@pytest.mark.parametrize("name", ["hash_collisions", "zcarry_2049", "quantiser_edges", "w_nan"])
def test_kld_repeatable(oracle, monkeypatch, name):
    """one case twice on fresh filters: the same bits, the count included, after the resample and after every step"""
    c = K.BY_NAME[name]
    outs = []
    for _ in range(2):
        cloud = c.cloud(oracle)
        g = rr.MonteCarloLocalizer(rr.MonteCarloLocalizationConfig(c.n_min, c.n_max, c.eps, c.z, RN, SV, SW, DT), seed=c.seed)
        g.set_particles(cloud)
        g.resample()
        rec = [(g.particle_count(), g.last_indices().copy(), bits(g.get_particles()))]
        for t in range(STEPS):
            g.try_step([1.0, 0.1], observations(cloud, t))
            rec.append((g.particle_count(), g.last_indices().copy(), bits(g.get_particles())))
        outs.append(rec)
    for (n0, i0, p0), (n1, i1, p1) in zip(*outs):
        assert n0 == n1 and np.array_equal(i0, i1) and np.array_equal(p0, p1)


@pytest.mark.parametrize("name,second", [("stop_1025", "never_3079"), ("never_1024_min1023", "stop_2049"), ("w_nan", "zcarry_1025"),
                                         ("hash_collisions", "w_cdf_ties")])
def test_kld_upload_at_new_count(oracle, name, second):
    """after the first resample, a second cloud uploaded at the new count and resampled with the next draws (call 1): the first
    case fixes the count, the second one's cloud is cut or tiled to it"""
    c, d = K.BY_NAME[name], K.BY_NAME[second]
    g, o = pair(oracle, c, c.cloud(oracle))
    g.resample(); o.resample()
    n = o.count()
    assert g.particle_count() == n
    b = d.cloud(oracle)
    b = np.concatenate([b] * (n // b.shape[0] + 1))[:n]
    b[:, 4] /= np.nansum(np.abs(b[:, 4]))
    g.set_particles(b); o.set_particles(b)
    o.L.orc_pf_set_fast_search(o.h, int(d.monotone))
    assert g.resample() and o.resample() == 1
    compare(g, o, f"{name} then {second}")
