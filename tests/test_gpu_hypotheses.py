"""Pose hypotheses on the GPU (include/pfgpu.h pfgpu_pf_hypotheses, DESIGN §3.10) against the numpy restatement
(tests/_cluster_oracle.py) on the same particle set: membership, count, bins, label and every particle's cluster exactly, the order
wherever the masses differ by more than 1e-12 relative, mass / mean / covariance to 1e-9 relative (1e-12 absolute).  Clouds are
uploaded (adversarial cases, a corridor, one cluster per particle) or taken from real runs on every step path.  Plus determinism,
agreement with estimate(), the two-mode behaviour on the symmetric floor plan, an untouched step, refusals, the C++ mirror and the
sharded engine."""
import ctypes as C
import math
import os
import subprocess
import sys

import numpy as np
import pytest

import _cluster_oracle as O
import rust_robotics_b200 as rr
from rust_robotics_b200 import scenarios
from test_cluster_oracle import SYM_START, symmetric_blobs, two_mode_outcome

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SV, SW = 0.2, 0.1


def mcl(n, seed=1, nmax=None):
    return rr.MonteCarloLocalizer(rr.MonteCarloLocalizationConfig(n, nmax or n, 0.05, 2.326, 0.25, SV, SW, 0.1), seed=seed)


def check(g, xy=0.5, K=24, p=None):
    """g's hypotheses of its current set against the oracle's; returns them"""
    p = g.get_particles() if p is None else p
    hs, total, rk = g.hypotheses(len(p), xy, K, labels=True)
    oh, ork = O.hypotheses(p, xy, K)
    assert total == len(oh) == len(hs)
    glab, olab = np.array([h.label for h in hs] + [-1]), np.array([h.label for h in oh] + [-1])
    assert np.array_equal(glab[rk], olab[ork]), "cluster of each particle"
    at = {h.label: i for i, h in enumerate(oh)}
    for i, h in enumerate(hs):
        o = oh[at[h.label]]
        assert at[h.label] == i or abs(o.mass - oh[i].mass) <= 1e-12 * oh[i].mass, f"rank {i}: order"
        assert (h.count, h.bins, h.label) == (o.count, o.bins, o.label), f"rank {i}: counts"
        assert np.isclose(h.weight, o.mass, rtol=1e-9, atol=1e-12), f"rank {i}: mass"
        dm = h.mean - o.mean
        dm[2] = O.wrap(dm[2])
        assert np.all(np.abs(dm) <= 1e-9 * np.abs(o.mean) + 1e-12), f"rank {i}: mean {h.mean} {o.mean}"
        assert np.allclose(h.cov, o.cov, rtol=1e-9, atol=1e-12), f"rank {i}: cov"
    return hs, total, rk


def adversarial(n, seed):
    rng = np.random.default_rng(seed)
    p = np.zeros((n, 5))
    p[:, 0], p[:, 1] = rng.normal(3.0, 2.0, n), rng.normal(-1.0, 2.0, n)
    p[:, 2], p[:, 3] = rng.uniform(-50.0, 50.0, n), rng.normal(1.0, 0.2, n)
    p[:, 4] = rng.random(n) / n
    special = [[0.5, 0.0, 0.0, 0.0], [-0.0, -0.0, -0.0, 0.0], [-1e-300, 0.49999999999999994, math.pi, 1.0], [0.0, 0.0, -math.pi, 1.0],
               [1.0, 1.0, 2 * O.TWO_PI, 0.0], [1.0, 1.0, -O.TWO_PI, 0.0], [2.0, 2.0, 1e3, 0.0], [2.0, 2.0, -1e3, 0.0],
               [1e12, 0.0, 0.0, 0.0], [-1e12, 1e12, 0.0, 0.0], [np.nan, 0.0, 0.0, 0.0], [0.0, np.inf, 0.0, 0.0],
               [0.0, 0.0, -np.inf, 0.0], [0.0, 0.0, 0.0, np.nan], [9.0, 9.0, math.pi - 0.01, 0.0], [9.0, 9.0, -math.pi + 0.01, 0.0]]
    wsp = [0.5, 0.25, 0.125, 1.0, 0.5, 0.5, 0.25, 0.25, 1.0, 1.0, 1.0, 1.0, 1.0, 1.0, 0.5, 0.5]
    for j, (s, w) in enumerate(zip(special, wsp)):
        if j < n:
            p[j, :4], p[j, 4] = s, w
    bad_w = [0.0, -1.0, np.nan, np.inf]
    for j, w in enumerate(bad_w):
        if len(special) + j < n:
            p[len(special) + j, 4] = w
    return p


@pytest.mark.parametrize("n", [1, 2, 1000, 1 << 16, 1 << 20])
def test_uploaded_adversarial_clouds(n):
    g = mcl(n)
    g.set_particles(adversarial(n, n))
    for xy, K in ((0.5, 24), (0.25, 36), (1.0, 1), (0.5, 2)):
        check(g, xy, K)


def test_corridor_spanning_more_than_1000_bins():
    n = 1 << 16
    rng = np.random.default_rng(2)
    p = np.zeros((n, 5))
    p[:, 0] = rng.uniform(-300.0, 300.0, n)                  # 1200 x-bins, every one occupied
    p[:, 1] = rng.normal(0.0, 0.1, n)
    p[:, 2] = rng.normal(0.0, 0.05, n) + 1e3
    p[:, 3] = 1.0
    p[:, 4] = rng.random(n)
    p[:4, 0] = [1e3, -1e3, 2e3, 400.0]                        # and a few strays
    g = mcl(n)
    g.set_particles(p)
    hs, total, _ = check(g)
    assert hs[0].bins > 1000 and hs[0].count > n - 10


def test_every_particle_its_own_cluster_cap_below_total():
    n = 1 << 16
    rng = np.random.default_rng(3)
    p = np.zeros((n, 5))
    p[:, 0], p[:, 1] = 2.0 * (np.arange(n) % 256), 2.0 * (np.arange(n) // 256)
    p[:, 2] = rng.uniform(-3.0, 3.0, n)
    p[:, 4] = rng.integers(1, 50, n) / 64.0                   # many exact ties: order by label
    g = mcl(n)
    g.set_particles(p)
    full, total, rk = check(g)
    assert total == n
    for cap in (0, 1, 7, 1000):
        hs, t2 = g.hypotheses(cap)
        assert t2 == n and len(hs) == cap
        for a, b in zip(hs, full):
            assert a.weight == b.weight and a.label == b.label and np.array_equal(a.mean, b.mean) and np.array_equal(a.cov, b.cov)


def test_deterministic_and_agrees_with_estimate():
    sc = scenarios.ScanScenario(steps=6)
    g = rr.MonteCarloLocalizer.try_with_initial_state([*sc.truth[0], 1.0], rr.MonteCarloLocalizationConfig(1 << 18, 1 << 18, 0.05, 2.326, 0.25, SV, SW, 0.1), seed=4)
    g.set_likelihood_field(sc.obstacles, sc.RES)
    for t in range(6):
        g.try_step_scan(sc.controls[t], *sc.scan_args(t))
    L = rr.load_library()
    bufs = []
    for _ in range(2):
        out, tot, rk = (rr.api._Hyp * 64)(), C.c_size_t(), np.empty(1 << 18, dtype=np.uint32)
        assert L.pfgpu_pf_hypotheses(g.h, 2.0, 8, out, 64, C.byref(tot), rk.ctypes.data_as(rr.api.c_u32p)) == 0
        bufs.append((bytes(out), tot.value, rk.tobytes()))
    assert bufs[0] == bufs[1]
    hs, total = g.hypotheses(4, 2.0, 8)                        # 2 m x 45 degree bins: one cluster holds the whole cloud
    assert total == 1 and hs[0].count == 1 << 18
    est, cov = g.estimate(), g.calc_covariance()
    for a in (0, 1, 3):
        assert abs(hs[0].mean[a] - est[a]) <= 1e-9 * max(1.0, abs(est[a]))
    for a, b in ((0, 0), (0, 1), (1, 1), (0, 3), (1, 3), (3, 3)):
        assert abs(hs[0].cov[a, b] - cov[a, b]) <= 1e-9 * max(1e-3, abs(cov[a, b]))


def _run_paths(kind, monkeypatch):
    """a handle after a few steps of one step path; returns it"""
    if kind in ("fused", "separate"):
        monkeypatch.setenv("PFGPU_PF_FUSED", "1" if kind == "fused" else "0")
    sc = scenarios.ScanScenario(steps=5)
    init = [*sc.truth[0], 1.0]
    if kind == "pf_phase":
        ks = scenarios.KidnapScenario(before=4, after=0)
        g = rr.ParticleFilterLocalizer.try_with_initial_state(ks.init, rr.ParticleFilterConfig(4096, 0.5, 0.25, 0.5, 0.1, 0.1), seed=3)
        for t in range(4):
            g.try_predict_with_control(ks.controls[t])
            g.try_update_with_observations(ks.obs[t])
            if t < 3:
                g.resample()
        return g                                             # non-uniform weights
    if kind == "landmark":
        ks = scenarios.KidnapScenario(before=6, after=0)
        g = rr.MonteCarloLocalizer.try_with_initial_state(ks.init, rr.MonteCarloLocalizationConfig(1 << 16, 1 << 16, 0.05, 2.326, 0.25, 0.5, 0.1, 0.1), seed=3)
        for t in range(6):
            g.try_step(ks.controls[t], ks.obs[t])
        return g
    n = {"fused": 4096, "separate": 4096, "beyond_2^18": (1 << 18) + 4096, "kld": 256, "recovery": 1 << 16}[kind]
    cfg = rr.MonteCarloLocalizationConfig(n, 16384 if kind == "kld" else n, 0.05, 2.326, 0.25, SV, SW, 0.1)
    if kind in ("kld", "recovery"):
        g = rr.MonteCarloLocalizer.try_with_region(sc.REGION, cfg, seed=6)
    else:
        g = rr.MonteCarloLocalizer.try_with_initial_state(init, cfg, seed=6)
    g.set_likelihood_field(sc.obstacles, sc.RES, **(dict(sigma_hit=2.0, max_beams=3) if kind == "kld" else {}))
    if kind == "recovery":
        g.enable_recovery(0.1, 0.6, sc.REGION)
    for t in range(5):
        g.try_step_scan(sc.controls[t], *sc.scan_args(t))
    return g


@pytest.mark.parametrize("kind", ["fused", "separate", "beyond_2^18", "pf_phase", "kld", "recovery", "landmark"])
def test_clouds_from_runs(kind, monkeypatch):
    g = _run_paths(kind, monkeypatch)
    for xy, K in ((0.5, 24), (0.1, 72)):
        check(g, xy, K)


def test_query_leaves_the_step_untouched():
    sc = scenarios.ScanScenario(steps=10)
    runs = []
    for query in (False, True):
        g = rr.MonteCarloLocalizer.try_with_region(sc.REGION, rr.MonteCarloLocalizationConfig(4096, 4096, 0.05, 2.326, 0.25, SV, SW, 0.1), seed=2)
        g.set_likelihood_field(sc.obstacles, sc.RES)
        g.enable_recovery(0.1, 0.6, sc.REGION)
        out, per_step = [], []
        for t in range(10):
            before = g.stats().kernel_launches
            e = g.try_step_scan(sc.controls[t], *sc.scan_args(t))
            per_step.append(g.stats().kernel_launches - before)
            out.append((e.tobytes(), g.get_particles().tobytes(), g.last_indices().tobytes()))
            if query:
                g.hypotheses(8, 0.5, 24, labels=True)
        runs.append((out, per_step))
    assert runs[0][0] == runs[1][0]
    assert runs[0][1] == runs[1][1]


@pytest.mark.parametrize("n", [1 << 16, 1 << 18])
def test_symmetric_plan_two_blobs(n):
    sc = scenarios.ScanScenario(steps=30, start=SYM_START, symmetric=True)
    g = mcl(n, seed=3)
    g.set_likelihood_field(sc.obstacles, sc.RES)
    g.set_particles(symmetric_blobs(sc, n, 3))
    for t in range(30):
        est = g.try_step_scan(sc.controls[t], *sc.scan_args(t))
    hs, _ = g.hypotheses(8)
    errs, masses, distinct, est_d = two_mode_outcome(sc, 29, [O.Hyp(h.weight, h.count, h.bins, h.label, h.mean, h.cov) for h in hs], est)
    print(f"n={n}: masses {masses}, errors {errs}, estimate distances {est_d}")
    assert distinct and all(e[0] < 0.5 and e[1] < 0.1 for e in errs), errs
    assert all(0.4 <= m <= 0.6 for m in masses), masses
    assert min(est_d) > 3.0, est_d


@pytest.mark.parametrize("seed", [1, 2, 3])
def test_symmetric_plan_global_localisation(seed):
    """From a region start both answers survive 60 steps only under a flat enough model: with AMCL's sigma_hit 0.2 and 60 beams
    the first resamples keep one mode (H100, all three seeds: one cluster of mass 1).  sigma_hit 1.0 and 20 beams keep both
    (H100: heaviest two masses 0.862 / 0.138, 0.961 / 0.039, 0.838 / 0.162 for seeds 1, 2, 3)."""
    sc = scenarios.ScanScenario(steps=60, start=SYM_START, symmetric=True)
    n = 1 << 18
    g = rr.MonteCarloLocalizer.try_with_region(sc.REGION, rr.MonteCarloLocalizationConfig(n, n, 0.05, 2.326, 0.25, SV, SW, 0.1), seed=seed)
    g.set_likelihood_field(sc.obstacles, sc.RES, sigma_hit=1.0, max_beams=20)
    g.enable_recovery(0.001, 0.1, sc.REGION)
    for t in range(60):
        g.try_step_scan(sc.controls[t], *sc.scan_args(t))
    hs, total = g.hypotheses(3)
    x, y, a = sc.truth[59]

    def near(q):
        return [i for i, h in enumerate(hs) if math.hypot(h.mean[0] - q[0], h.mean[1] - q[1]) < 0.5 and abs(scenarios.normalize_angle(h.mean[2] - q[2])) < 0.1]
    print(f"seed {seed}: {total} clusters, masses {[h.weight for h in hs]}, truth {near((x, y, a))}, mirror {near((-x, -y, a + math.pi))}")
    t_i, m_i = near((x, y, a)), near((-x, -y, a + math.pi))
    assert t_i and m_i and set(t_i) != set(m_i)


def test_refusals():
    g = mcl(256)
    for xy, K in ((0.0, 24), (-1.0, 24), (np.nan, 24), (np.inf, 24), (0.5, 0), (0.5, 65537)):
        with pytest.raises(rr.InvalidParameter):
            g.hypotheses(4, xy, K)
    L = rr.load_library()
    assert L.pfgpu_pf_hypotheses(g.h, 0.5, 24, None, 1, None, None) < 0
    assert L.pfgpu_pf_hypotheses(None, 0.5, 24, None, 0, None, None) < 0
    tot = C.c_size_t()
    assert L.pfgpu_pf_hypotheses(g.h, 0.5, 65536, None, 0, C.byref(tot), None) == 0 and tot.value >= 1
    p = g.get_particles()
    p[:, 4] = 0.0
    g.set_particles(p)
    hs, total, rk = g.hypotheses(4, labels=True)
    assert hs == [] and total == 0 and np.all(rk == -1)


def test_cpp_mirror_hypotheses(tmp_path):
    """host/cluster_check.cpp through the C++ mirror: the Python mirror's numbers, bit for bit"""
    pkg, exe = os.path.join(ROOT, "rust_robotics_b200"), str(tmp_path / "cluster_check")
    subprocess.run(["/usr/bin/g++", "-std=c++17", "-O1", os.path.join(pkg, "host", "cluster_check.cpp"), "-I", os.path.join(ROOT, "include"),
                    "-I", os.path.join(pkg, "host"), "-L", pkg, "-lpfgpu", f"-Wl,-rpath,{pkg}", "-o", exe], check=True)
    r = subprocess.run([exe], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr
    got = np.array([float.fromhex(x) for x in r.stdout.split()])
    f = rr.MonteCarloLocalizer(rr.MonteCarloLocalizationConfig(4096, 4096, 0.05, 2.326, 0.2, 0.2, 0.1, 0.1), seed=13)
    f.init_region((-9.0, 9.0, -9.0, 9.0))
    lms = [[5.0, 1.0, 1.0], [4.0, -2.0, 0.5], [6.0, 3.0, -3.0]]
    for _ in range(4):
        f.try_step([1.0, 0.1], lms)
    hs, total, rk = f.hypotheses(5, 0.5, 24, labels=True)
    want = [float(total)] + [v for h in hs for v in [h.weight, *h.mean, *h.cov.T.ravel(), h.count, h.bins, h.label]] + [float(v) for v in rk[:64]]
    assert got.shape == (len(want),) and np.array_equal(got, np.array(want))


def test_hypotheses_multi_process():
    """one process per GPU (tests/mgpu_hypotheses_worker.py): every rank returns the same bits, and a single-GPU handle holding the
    gathered set returns them too"""
    c = C.c_int()
    rr.load_library().pfgpu_device_count(C.byref(c))
    if c.value < 2:
        pytest.skip("needs 2 GPUs")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr", "127.0.0.1",
           "--master-port", "29561", os.path.join(ROOT, "tests", "mgpu_hypotheses_worker.py"), str(4096 * 2), "6"]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0 and "MGPU_OK" in r.stdout, r.stdout[-2000:] + r.stderr[-4000:]
