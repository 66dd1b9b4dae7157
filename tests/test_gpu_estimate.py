"""FastSLAM estimate (FastSlam1.estimate / estimate_all; pfgpu_fs_moments + pfgpu_fs_estimate_merge) against a float64 numpy
restatement of its definition (DESIGN §3.4), computed here from the downloaded state and from the CPU oracle's state.

The definition: W = sum of the stored weights.  Pose: weighted mean and covariance of (x, y, yaw), yaw deviations wrapped about the
centre c = the current pose of the last particle, mean yaw wrapped.  Landmark l: over the copies with cov00 < cov00_max,
mass = sum w / W, mean = weighted mean of (x, y), cov = sum w (P + d d^T) / sum w.  mass 0 -> NaN mean / cov; W <= 0 or not
finite -> everything NaN, mass 0.
"""
import ctypes as C
import math
import os
import subprocess
import sys

import numpy as np
import pytest

import rust_robotics_b200 as rr
from rust_robotics_b200 import scenarios
from _oracle import OracleFS

pytestmark = pytest.mark.gpu


def _wrap(a):
    a = np.asarray(a, dtype=np.float64)
    return np.where(np.abs(a) <= math.pi, a, a - 2.0 * math.pi * np.rint(a / (2.0 * math.pi)))


def ref_estimate(pw, lm, centre, cov00_max=100.0):
    """§3.4 in float64 numpy, two-pass; pw: (n, 4) (w, x, y, yaw), lm: (n, m, 6) or None"""
    w = pw[:, 0]
    W = w.sum()
    m = 0 if lm is None else lm.shape[1]
    nan = np.nan
    if not (np.isfinite(W) and W > 0):
        return np.full(3, nan), np.full((3, 3), nan), np.zeros(m), np.full((m, 2), nan), np.full((m, 2, 2), nan)
    c = np.asarray(centre, dtype=np.float64)
    d = np.stack([pw[:, 1] - c[0], pw[:, 2] - c[1], _wrap(pw[:, 3] - c[2])], axis=1)
    a = (w[:, None] * d).sum(axis=0) / W
    mean = c + a
    mean[2] = _wrap(mean[2])
    e = d - a
    cov = np.einsum("i,ij,ik->jk", w, e, e) / W
    mass, lmean, lcov = np.zeros(m), np.full((m, 2), nan), np.full((m, 2, 2), nan)
    lb = max(1, min(64, (1 << 22) // max(len(w), 1)))        # landmarks per block: bounded temporaries at 2^22 particles
    for l0 in range(0, m, lb):
        blk = lm[:, l0:l0 + lb, :]
        sel = blk[:, :, 2] < cov00_max
        ws = np.where(sel, w[:, None], 0.0)
        sw = ws.sum(axis=0)
        x, y = np.where(sel, blk[:, :, 0], 0.0), np.where(sel, blk[:, :, 1], 0.0)
        with np.errstate(invalid="ignore", divide="ignore"):
            mx, my = (ws * x).sum(axis=0) / sw, (ws * y).sum(axis=0) / sw
            dx, dy = np.where(sel, x - mx, 0.0), np.where(sel, y - my, 0.0)
            P = [np.where(sel, blk[:, :, 2 + k], 0.0) for k in range(4)]
            cc = np.stack([(ws * (P[0] + dx * dx)).sum(axis=0), (ws * (P[1] + dx * dy)).sum(axis=0),
                           (ws * (P[2] + dx * dy)).sum(axis=0), (ws * (P[3] + dy * dy)).sum(axis=0)], axis=1) / sw[:, None]
        some = sw != 0
        mass[l0:l0 + lb] = np.where(some, sw / W, 0.0)
        lmean[l0:l0 + lb] = np.where(some[:, None], np.stack([mx, my], axis=1), nan)
        lcov[l0:l0 + lb] = np.where(some[:, None, None], cc.reshape(-1, 2, 2), nan)
    return mean, cov, mass, lmean, lcov


def _close(got, ref, what, scale=None):
    got, ref = np.asarray(got), np.asarray(ref)
    assert np.array_equal(np.isnan(got), np.isnan(ref)), f"{what}: NaN pattern"
    ok = ~np.isnan(ref)
    tol = 1e-9 * ((1.0 + np.abs(ref)) if scale is None else scale)
    bad = ok & ~(np.abs(got - ref) <= tol)
    assert not bad.any(), f"{what}: {np.argwhere(bad)[:4].tolist()} got {got[bad][:4]} want {ref[bad][:4]}"


def check(est, ref, what):
    mean, cov, mass, lmean, lcov = ref
    _close(est.pose, mean, f"{what}: pose mean")
    _close(est.pose_cov, cov, f"{what}: pose cov", scale=np.nanmax(np.abs(cov)) if np.isfinite(cov).any() else 1.0)
    if est.mass is None:
        return
    assert est.mass.shape == mass.shape
    assert np.array_equal(est.mass == 0.0, mass == 0.0), f"{what}: zero masses differ"
    assert np.all(np.abs(est.mass - mass) <= 1e-12 * np.abs(mass)), f"{what}: mass"
    _close(est.mean, lmean, f"{what}: landmark mean")
    scale = np.nanmax(np.abs(lcov), axis=(1, 2), initial=0.0)[:, None, None] if lcov.size else 1.0
    _close(est.cov, lcov, f"{what}: landmark cov", scale=scale)


def _centre(pw):
    """the estimate's centre: the current pose of the last particle"""
    return pw[-1, 1:4]


def _check_engine(g, what, cov00_max=100.0, oracle=None):
    pw, lm = g.state()
    est = g.estimate(cov00_max)
    check(est, ref_estimate(pw, lm, _centre(pw), cov00_max), what)
    if oracle is not None:
        op, ol = oracle.state()
        check(est, ref_estimate(op, ol, _centre(op), cov00_max), what + " (oracle state)")
    return est


def _mid_circle(side, steps):
    mid = 10.0 * (side - 1) / 2.0
    return scenarios.FastSlamScenario(side, (mid, mid - 40.0, 0.0), (1.0, 0.025), steps)


def _corridor(m, steps, speed=1.2, max_range=2.5, seed=3):
    """m landmarks 1 m apart on the x axis, passed 1 m to the side: landmarks leave the view and keep old ancestry rows"""
    lm = np.stack([np.arange(m, dtype=np.float64), np.zeros(m)], axis=1)
    u = [speed / 0.1, 0.0]
    rng = np.random.default_rng(seed)
    x = [0.0, 1.0, 0.0]
    obs = []
    for _ in range(steps):
        x = scenarios.motion_model(x, u)
        obs.append(scenarios.get_observations(x, lm, rng, max_range=max_range))
    return lm, u, [0.0, 1.0, 0.0], obs


# ---------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("variant", [1, 2])
@pytest.mark.parametrize("n", [64, 1000, 4096])
def test_estimate_trajectory(oracle, variant, n):
    """C3's map and circle: after steps that resampled and steps that did not, against numpy on the GPU and the oracle state"""
    steps = 24
    sc = scenarios.c3_scenario(steps=steps)
    cls = rr.FastSlam1 if variant == 1 else rr.FastSlam2
    g = cls(n, sc.m, rr.FsConfig(nth=n / 1.5), seed=11)
    o = OracleFS(oracle, n, sc.m, seed=11, variant=variant, nth=n / 1.5)
    g.seed_map(sc.start, sc.landmarks); o.seed_map(sc.start, sc.landmarks)
    _check_engine(g, "seeded", oracle=o)
    kinds = set()
    for t in range(steps):
        did = g.fastslam_update(sc.control, sc.obs[t])
        assert did == bool(o.step(sc.control, sc.obs[t]))
        if t % 3 == 0 or did not in kinds:          # both kinds of step as soon as they occur
            kinds.add(did)
            _check_engine(g, f"step {t} (resampled={did})", oracle=o)
            _check_engine(g, f"step {t} inf", cov00_max=math.inf)
    assert True in kinds and (variant == 2 or False in kinds)       # (FastSLAM 2.0 resamples every step here)


def test_estimate_corridor_live_rows(oracle):
    """landmarks leave and re-enter view: several live ancestry rows, read through by the map pass"""
    n, m, steps = 128, 256, 220
    lm, u, start, obs = _corridor(m, steps)
    g = rr.FastSlam1(n, m, rr.FsConfig(nth=float(n), max_range=2.5), seed=5)
    o = OracleFS(oracle, n, m, seed=5, nth=float(n), max_range=2.5)
    g.seed_map(start, lm); o.seed_map(start, lm)
    for t in range(steps):
        assert g.fastslam_update(u, obs[t]) == bool(o.step(u, obs[t]))
        if t % 40 == 39:
            _check_engine(g, f"step {t}", oracle=o)
            _check_engine(g, f"step {t} inf", cov00_max=math.inf)


@pytest.mark.parametrize("variant", [1, 2])
def test_estimate_config3(variant):
    """the full config-3 shape (65 536 particles x 256 landmarks); two calls return the same bits; pose only = the same pose"""
    n, steps = 1 << 16, 12
    sc = scenarios.c3_scenario(steps=steps)
    cls = rr.FastSlam1 if variant == 1 else rr.FastSlam2
    g = cls(n, sc.m, rr.FsConfig(nth=n / 1.5), seed=42)
    g.seed_map(sc.start, sc.landmarks)
    for t in range(steps):
        g.fastslam_update(sc.control, sc.obs[t], want_flag=False)
    est = _check_engine(g, "config 3")
    again = g.estimate()
    for a, b in zip(est, again):
        assert np.array_equal(a.view(np.uint64), b.view(np.uint64))
    pose_only = g.estimate(landmarks=False)
    assert pose_only.mass is None and np.array_equal(pose_only.pose, est.pose) and np.array_equal(pose_only.pose_cov, est.pose_cov)
    assert (est.mass > 0).sum() > 50


def test_estimate_global_tiles():
    """2^22 particles (the post kernel's global-tile regime) on a 9-landmark map (3 x 3 grid inside a 20 m circle)"""
    n = 1 << 22
    sc = scenarios.FastSlamScenario(3, (10.0, 0.0, 0.0), (1.0, 0.05), 3)
    g = rr.FastSlam1(n, sc.m, rr.FsConfig(nth=n / 1.5), seed=3)
    assert g.post_shape()[3] == "global"
    g.seed_map(sc.start, sc.landmarks)
    for t in range(3):
        g.fastslam_update(sc.control, sc.obs[t], want_flag=False)
    _check_engine(g, "2^22")


def test_estimate_16384_landmarks():
    """16 384 landmarks x 3 000 particles (n not a multiple of 64)"""
    n = 3000
    sc = _mid_circle(128, 6)
    g = rr.FastSlam1(n, sc.m, rr.FsConfig(nth=n / 1.5), seed=8)
    g.seed_map(sc.start, sc.landmarks)
    for t in range(6):
        g.fastslam_update(sc.control, sc.obs[t], want_flag=False)
    _check_engine(g, "16384 landmarks")
    _check_engine(g, "16384 landmarks inf", cov00_max=math.inf)


# ---------------------------------------------------------------------------------------------------------------------------
def test_estimate_edge_cases():
    nan = np.nan
    # m = 0
    g = rr.FastSlam1(100, 0, seed=1)
    e = g.estimate()
    assert e.mass.shape == (0,) and e.mean.shape == (0, 2) and e.cov.shape == (0, 2, 2)
    check(e, ref_estimate(g.state()[0], np.zeros((100, 0, 6)), g.state()[0][99, 1:4]), "m = 0")
    # fresh create_particles: W = n / 100; FS1's unseeded quirk keeps cov 1000, so the default filter takes nothing
    n, m = 200, 5
    g = rr.FastSlam1(n, m, seed=1)
    g.fastslam_update([1.0, 0.1], [(5.0, 0.1, 0), (7.0, -0.4, 2)])
    pw, lm = g.state()
    assert np.all(lm[:, :, 2] == 1000.0)
    e = g.estimate()
    assert np.all(e.mass == 0.0) and np.isnan(e.mean).all() and np.isnan(e.cov).all()
    check(e, ref_estimate(pw, lm, _centre(pw)), "unseeded")
    f = rr.FastSlam1(n, m, seed=1)
    pw0, lm0 = f.state()
    assert np.all(pw0[:, 0] == 0.01)
    e = f.estimate(math.inf)
    assert np.allclose(e.mass, 1.0, rtol=1e-12, atol=0.0) and np.allclose(e.pose, 0.0) and np.allclose(e.pose_cov, 0.0)
    check(e, ref_estimate(pw0, lm0, pw0[-1, 1:4], math.inf), "fresh, W = n/100")
    # a threshold that filters every copy; cov00_max = inf; NaN is refused
    g = rr.FastSlam1(256, 8, seed=2)
    g.seed_map([1.0, 2.0, 0.3], np.arange(16.0).reshape(8, 2))
    e = g.estimate(0.0)
    assert np.all(e.mass == 0.0) and np.isnan(e.mean).all() and np.isnan(e.cov).all()
    pw, lm = g.state()
    check(g.estimate(math.inf), ref_estimate(pw, lm, pw[-1, 1:4], math.inf), "inf")
    with pytest.raises(rr.InvalidParameter):
        g.estimate(nan)
    # all-zero and NaN weights via set_state: everything NaN, masses 0
    rng = np.random.default_rng(0)
    for wv in (0.0, nan):
        p = np.concatenate([np.full((256, 1), wv), rng.normal(size=(256, 3))], axis=1)
        g.set_state(p, lm)
        e = g.estimate(math.inf)
        assert np.isnan(e.pose).all() and np.isnan(e.pose_cov).all() and np.all(e.mass == 0.0)
        assert np.isnan(e.mean).all() and np.isnan(e.cov).all()
    # a yaw cloud across +-pi: mean near +-pi, small variance
    yaw = _wrap(math.pi + rng.normal(scale=0.05, size=256))
    assert (yaw > 0).any() and (yaw < 0).any()
    p = np.stack([rng.uniform(0.5, 1.5, 256), rng.normal(size=256), rng.normal(size=256), yaw], axis=1)
    g.set_state(p, lm)
    e = g.estimate(math.inf)
    assert abs(abs(e.pose[2]) - math.pi) < 0.02 and e.pose_cov[2, 2] < 0.01
    check(e, ref_estimate(p, lm, p[-1, 1:4], math.inf), "yaw across pi")
    # pose only
    e = g.estimate(landmarks=False)
    assert e.mass is None and e.mean is None and e.cov is None


@pytest.mark.parametrize("world", [1, 2])
def test_estimate_after_set_state(world):
    """set_state after steps (a restored checkpoint): the centre comes from the state now held, not from the last step.  A tight
    cloud across +-pi far from the stepped cloud: mean yaw near +-pi, small variance, and numpy's answer; then the checkpoint
    restored gives the estimate it had"""
    n, steps = 1024, 6
    sc = scenarios.c3_scenario(steps=steps)
    ranks = rr.FastSlam1.create_sharded_local(n, sc.m, [0] * world, rr.FsConfig(nth=n / 1.5), seed=6) if world > 1 else \
        [rr.FastSlam1(n, sc.m, rr.FsConfig(nth=n / 1.5), seed=6)]
    for g in ranks:
        g.seed_map(sc.start, sc.landmarks)
    for t in range(steps):
        rr.FastSlam1.step_all(ranks, sc.control, sc.obs[t])
    states = [g.state() for g in ranks]
    before = rr.FastSlam1.estimate_all(ranks, math.inf)
    assert abs(before.pose[2]) < 1.0                     # the stepped cloud heads near yaw 0
    rng = np.random.default_rng(1)
    for x0, sx in ((0.0, 1.0), (1.0e5, 1.0e-2)):
        yaw = _wrap(math.pi + rng.normal(scale=0.05, size=n))
        assert (yaw > 0).any() and (yaw < 0).any()
        p = np.stack([rng.uniform(0.5, 1.5, n), x0 + rng.normal(scale=sx, size=n), -x0 + rng.normal(scale=sx, size=n), yaw], axis=1)
        lm = np.concatenate([s[1] for s in states])
        for r, g in enumerate(ranks):
            g.set_state(p[r * g.n_local:(r + 1) * g.n_local], lm[r * g.n_local:(r + 1) * g.n_local])
        e = rr.FastSlam1.estimate_all(ranks, math.inf)
        assert abs(abs(e.pose[2]) - math.pi) < 0.02 and e.pose_cov[2, 2] < 0.01, (e.pose, e.pose_cov)
        assert abs(e.pose[0] - x0) < 10 * sx and e.pose_cov[0, 0] < 2 * sx * sx
        check(e, ref_estimate(p, lm, _centre(p), math.inf), f"set_state after steps, cloud at {x0}")
    for g, (pw, lm) in zip(ranks, states):
        g.set_state(pw, lm)
    again = rr.FastSlam1.estimate_all(ranks, math.inf)
    for a, b in zip(before, again):
        assert np.array_equal(a, b, equal_nan=True)


# ---------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("variant", [1, 2])
@pytest.mark.parametrize("world,n", [(2, 1024), (4, 4096)])
def test_estimate_sharded_in_process(variant, world, n):
    """estimate_all over in-process ranks = the one-GPU engine on the same seed = numpy over the concatenated shard states"""
    steps = 16
    sc = scenarios.c3_scenario(steps=steps)
    cls = rr.FastSlam1 if variant == 1 else rr.FastSlam2
    ranks = cls.create_sharded_local(n, sc.m, [0] * world, rr.FsConfig(nth=n / 1.5), seed=9)
    one = cls(n, sc.m, rr.FsConfig(nth=n / 1.5), seed=9)
    for g in ranks + [one]:
        g.seed_map(sc.start, sc.landmarks)
    resamples, remote = 0, 0
    for t in range(steps):
        did = cls.step_all(ranks, sc.control, sc.obs[t])
        assert did == one.fastslam_update(sc.control, sc.obs[t])
        resamples += did
        if did:          # slots whose ancestor lives on another rank: their maps are read through the peer mapping
            remote += sum(int(((g.last_indices() // g.n_local) != r).sum()) for r, g in enumerate(ranks))
        if t % 4 == 3:
            for cm in (100.0, math.inf):
                e = cls.estimate_all(ranks, cm)
                states = [g.state() for g in ranks]
                pw = np.concatenate([s[0] for s in states]); lm = np.concatenate([s[1] for s in states])
                ref = ref_estimate(pw, lm, _centre(pw), cm)
                check(e, ref, f"step {t} sharded")
                check(one.estimate(cm), ref, f"step {t} one GPU")
                p_only = cls.estimate_all(ranks, cm, landmarks=False)
                assert np.array_equal(p_only.pose, e.pose)
    assert resamples > 1 and remote > 0


@pytest.mark.parametrize("world", [1, 2, 4])
def test_estimate_multi_process(world):
    """one process per GPU (tests/mgpu_estimate_worker.py): every rank's moments, gathered and merged on every rank, = numpy over
    the oracle's full state; world = 1 runs the same script on one GPU"""
    c = C.c_int()
    rr.load_library().pfgpu_device_count(C.byref(c))
    if c.value < world:
        pytest.skip(f"needs {world} GPUs")
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={world}", "--master-addr", "127.0.0.1",
           "--master-port", "29547", os.path.join(root, "tests", "mgpu_estimate_worker.py"), str(2048 * world), "16"]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0 and "MGPU_OK" in r.stdout, r.stdout[-2000:] + r.stderr[-4000:]


# ---------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("variant", [1, 2])
@pytest.mark.parametrize("world", [1, 2])
@pytest.mark.parametrize("env", [{"PFGPU_PDL": "1"}, {"PFGPU_PDL": "0"}, {"PFGPU_EARLY_LAUNCH": "1"}])
def test_estimate_leaves_step_unchanged(oracle, monkeypatch, variant, world, env):
    """an estimate after every step: gate, indices, best particle and final state bit for bit the oracle's and a run without"""
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    n, steps = 1024, 20
    sc = scenarios.c3_scenario(steps=steps)
    cls = rr.FastSlam1 if variant == 1 else rr.FastSlam2

    def make():
        gs = cls.create_sharded_local(n, sc.m, [0] * world, rr.FsConfig(nth=n / 1.5), seed=4) if world > 1 else \
            [cls(n, sc.m, rr.FsConfig(nth=n / 1.5), seed=4)]
        for g in gs:
            g.seed_map(sc.start, sc.landmarks)
        return gs

    gs, plain = make(), make()
    o = OracleFS(oracle, n, sc.m, seed=4, variant=variant, nth=n / 1.5)
    o.seed_map(sc.start, sc.landmarks)
    for t in range(steps):
        for g in gs:
            g.fastslam_update(sc.control, sc.obs[t], want_flag=False)
        e = cls.estimate_all(gs)                      # between this step's post kernel and the next step's EKF launch
        assert np.isfinite(e.pose).all()
        did = cls.step_all(plain, sc.control, sc.obs[t])
        assert gs[0].did_resample() == did == bool(o.step(sc.control, sc.obs[t])), f"step {t}: gate"
        if did:
            idx = np.concatenate([g.last_indices() for g in gs])
            assert np.array_equal(idx, o.last_indices()) and np.array_equal(idx, np.concatenate([g.last_indices() for g in plain]))
        assert gs[0].get_best_particle()[0] == o.best() == plain[0].get_best_particle()[0]
    op, ol = o.state()
    for r, (g, q) in enumerate(zip(gs, plain)):
        gp, gl = g.state()
        qp, ql = q.state()
        lo, hi = r * g.n_local, (r + 1) * g.n_local
        assert np.array_equal(gp, op[lo:hi]) and np.array_equal(gl, ol[lo:hi]), f"rank {r}: state differs from the oracle"
        assert np.array_equal(gp, qp) and np.array_equal(gl, ql)


# ---------------------------------------------------------------------------------------------------------------------------
def test_cpp_mirror_estimate(tmp_path):
    """host/estimate_check.cpp through the C++ mirror's FastSlam::estimate(): the Python mirror's numbers, bit for bit"""
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    pkg = os.path.join(root, "rust_robotics_b200")
    exe = str(tmp_path / "estimate_check")
    subprocess.run(["/usr/bin/g++", "-std=c++17", "-O1", os.path.join(pkg, "host", "estimate_check.cpp"), "-I", os.path.join(root, "include"),
                    "-I", os.path.join(pkg, "host"), "-L", pkg, "-lpfgpu", f"-Wl,-rpath,{pkg}", "-o", exe], check=True)
    r = subprocess.run([exe], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr
    got = np.array([float(x) for x in r.stdout.split()])
    fs = rr.FastSlam1(1000, 4, seed=42)
    for _ in range(3):
        fs.fastslam_update([1.0, 0.1], [(5.0, 0.1, 0), (7.0, -0.4, 2)])
    want = []
    for e in (fs.estimate(math.inf), fs.estimate(), fs.estimate(100.0, landmarks=False)):
        want += list(e.pose) + list(e.pose_cov.T.ravel())
        if e.mass is not None:
            for l in range(4):
                want += [e.mass[l], e.mean[l, 0], e.mean[l, 1]] + list(e.cov[l].ravel())
    want = np.array(want)
    assert got.shape == want.shape and np.array_equal(got, want, equal_nan=True)
