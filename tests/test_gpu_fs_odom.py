"""FastSLAM with the odometry motion model (pfgpu_fs_step_odom / pfgpu_fs_step_unknown_odom, DESIGN §3.15) against the CPU oracle
(tests/host/fs_odom_oracle.c) bit for bit: poses, weights, every landmark field, resample indices, gate, best particle, association
counts and existence counters — FastSLAM 1.0 and 2.0, known and unknown association, k = 0, long lists with repeated ids, the
global-tile post kernel, velocity and odometry steps on one handle, 2 and 4 in-process ranks, and every refusal."""
import ctypes as C
import math
import os
import subprocess
import sys

import numpy as np
import pytest

import rust_robotics_b200 as rr
from rust_robotics_b200 import scenarios
from _fs_odom_oracle import OracleFsOdom

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
THREADS = max(1, min(32, os.cpu_count() or 1))


def _drive(sc, steps):
    """odometry pairs along sc.truth with a stop, a turn in place and a reverse, and the observations of each step"""
    odo = [list(sc.start)] + [list(p) for p in sc.truth[:steps]]
    pairs = []
    for t in range(steps):
        a, b = odo[t], odo[t + 1]
        if t % 7 == 3:
            b = list(a)                                          # stop
        elif t % 7 == 5:
            b = [a[0], a[1], a[2] + 0.4]                         # turn in place
        elif t % 7 == 6:
            b = [a[0] - 0.3 * math.cos(a[2]), a[1] - 0.3 * math.sin(a[2]), a[2]]   # reverse
        pairs.append((a, b))
    return pairs


def _same(gs, o, what):
    op, ol = o.state()
    lo = 0
    for r, g in enumerate(gs):
        gp, gl = g.state()
        assert np.array_equal(gp, op[lo:lo + g.n_local], equal_nan=True), f"{what} rank {r}: poses / weights differ"
        assert np.array_equal(gl, ol[lo:lo + g.n_local], equal_nan=True), f"{what} rank {r}: landmarks differ"
        lo += g.n_local


def _check(gs, o, t, did, odid):
    assert did == odid, f"step {t}: gate"
    if did:
        assert np.array_equal(np.concatenate([g.last_indices() for g in gs]), o.last_indices()), f"step {t}: indices"
    assert math.isclose(gs[0].last_neff(), o.last_neff(), rel_tol=1e-9), f"step {t}: N_eff"
    for g in gs:
        assert g.get_best_particle()[0] == o.best(), f"step {t}: best particle"


def _setup(variant, n, m, sc, world=1, seed=5, seeded=True):
    cls = rr.FastSlam2 if variant == 2 else rr.FastSlam1
    cfg = rr.FsConfig(nth=n / 1.5)
    gs = cls.create_sharded_local(n, m, [0] * world, cfg, seed=seed) if world > 1 else [cls(n, m, cfg, seed=seed)]
    o = OracleFsOdom(n, m, seed=seed, variant=variant, nth=n / 1.5)
    o.L.orc_fs_set_threads(o.h, THREADS)
    if seeded:
        for g in gs:
            g.seed_map(sc.start, sc.landmarks)
        o.seed_map(sc.start, sc.landmarks)
    else:
        pw = np.tile([1.0 / n, *sc.start], (n, 1))
        lm = np.tile([0.0, 0.0, 1000.0, 0.0, 0.0, 1000.0], (n, m, 1))
        lo = 0
        for g in gs:
            g.set_state(pw[lo:lo + g.n_local], lm[lo:lo + g.n_local])
            lo += g.n_local
        o.set_state(pw, lm)
    return gs, o


def _known(variant, n, steps, world=1, velocity_every=0, long_lists=False, alpha=None):
    sc = scenarios.FastSlamScenario(4, (15.0, 15.0, 0.0), (1.0, 0.05), steps, seed=3, max_range=40.0)
    gs, o = _setup(variant, n, sc.m, sc, world)
    if alpha is not None:
        for g in gs:
            g.set_odometry_noise(*alpha)
        o.set_odom_noise(alpha)
    resamples = 0
    for t, (a, b) in enumerate(_drive(sc, steps)):
        z = sc.obs[t] if t % 5 != 2 else []                            # some steps without observations
        if long_lists and z:
            z = (z + z[::-1] + z)[:40]                                  # > 31 observations and repeated ids: split launches
        if velocity_every and t % velocity_every == velocity_every - 1:
            for g in gs:
                g.fastslam_update(sc.control, z, want_flag=False)
            odid = o.step(sc.control, z)
        else:
            for g in gs:
                g.fastslam_update_odometry(a, b, z, want_flag=False)
            odid = o.step_odom(a, b, z)
        for g in gs:
            g.sync()
        did = gs[0].did_resample()
        _check(gs, o, t, did, bool(odid))
        _same(gs, o, f"step {t}")
        resamples += int(did)
    return resamples


@pytest.mark.parametrize("variant", [1, 2])
def test_known_ids_match_oracle(variant):
    assert _known(variant, 1024, 14) > 0


@pytest.mark.parametrize("variant", [1, 2])
def test_long_lists_and_repeated_ids(variant):
    _known(variant, 512, 8, long_lists=True)


@pytest.mark.parametrize("variant", [1, 2])
def test_velocity_and_odometry_interleaved(variant):
    _known(variant, 512, 12, velocity_every=3)


@pytest.mark.parametrize("world", [2, 4])
@pytest.mark.parametrize("variant", [1, 2])
def test_in_process_ranks(variant, world):
    _known(variant, 1024, 10, world=world)


@pytest.mark.parametrize("n", [64, 1 << 16])
def test_particle_counts(n):
    _known(2, n, 6)


def test_alphas_zero_and_custom():
    _known(2, 512, 8, alpha=(0.0, 0.0, 0.0, 0.0))
    _known(1, 512, 8, alpha=(0.05, 0.01, 0.3, 0.02))


@pytest.mark.parametrize("ex", [False, True])
@pytest.mark.parametrize("world", [1, 2])
def test_unknown_association_match_oracle(ex, world):
    n = 1024
    sc = scenarios.FastSlamScenario(4, (15.0, 15.0, 0.0), (1.0, 0.05), 12, seed=3, max_range=40.0)
    m = sc.m + 4
    gs, o = _setup(2, n, m, sc, world, seeded=False)
    if ex:
        for g in gs:
            g.enable_existence(30.0)
        o.enable_existence(30.0)
    for t, (a, b) in enumerate(_drive(sc, 12)):
        z = [(d, ang) for d, ang, _ in sc.obs[t]] if t % 5 != 2 else []
        for g in gs:
            g.fastslam2_update_unknown_odometry(a, b, z, want_flag=False)
        odid = o.step_unknown_odom(a, b, z)
        for g in gs:
            g.sync()
        did = gs[0].did_resample()
        _check(gs, o, t, did, bool(odid))
        _same(gs, o, f"step {t}")
        assert tuple(int(v) for v in np.sum([g.assoc_counts() for g in gs], axis=0)) == tuple(int(v) for v in o.counts), f"step {t}: counts"
        if ex:
            assert np.array_equal(np.concatenate([g.existence_counts() for g in gs]), o.existence_counts()), f"step {t}: tau"
            assert sum(g.removed_count() for g in gs) == o.removed, f"step {t}: removed"


def test_standstill_keeps_poses():
    sc = scenarios.FastSlamScenario(4, (15.0, 15.0, 0.0), (1.0, 0.05), 4, seed=3, max_range=40.0)
    for cls in (rr.FastSlam1, rr.FastSlam2):
        g = cls(256, sc.m, rr.FsConfig(nth=0.0), seed=9)
        g.seed_map(sc.start, sc.landmarks)
        g.fastslam_update(sc.control, sc.obs[0])                   # spread the cloud first
        before = g.state()[0]
        still = [1.0, 2.0, 0.3]
        g.fastslam_update_odometry(still, still, sc.obs[1])
        after = g.state()[0]
        assert np.array_equal(before[:, 1:], after[:, 1:]), cls.__name__


def test_refusals():
    g1 = rr.FastSlam1(64, 4, seed=1)
    g2 = rr.FastSlam2(64, 4, seed=1)
    assert g1.odometry_noise() == (0.2, 0.2, 0.2, 0.2)
    for bad in ([-0.1, 0, 0, 0], [float("nan"), 0, 0, 0], [float("inf"), 0, 0, 0]):
        with pytest.raises(rr.InvalidParameter):
            g1.set_odometry_noise(*bad)
    g1.set_odometry_noise(0.1, 0.2, 0.3, 0.4)
    assert g1.odometry_noise() == (0.1, 0.2, 0.3, 0.4)
    for bad in ([float("nan"), 0, 0], [0, float("inf"), 0]):
        with pytest.raises(rr.InvalidParameter):
            g1.fastslam_update_odometry(bad, [0, 0, 0], [])
        with pytest.raises(rr.InvalidParameter):
            g2.fastslam2_update_unknown_odometry([0, 0, 0], bad, [])
    with pytest.raises(rr.InvalidParameter):
        g2.fastslam2_update_unknown_odometry([0, 0, 0], [1, 0, 0], [(1.0, 0.1)], gate_d2=0.0)
    with pytest.raises(rr.InvalidParameter):
        g1.fastslam_update_odometry([0, 0, 0], [1, 0, 0], [(1.0, 0.1, 7)])          # lm_id out of range
    with pytest.raises(rr.InvalidParameter, match="not supported"):
        rr.FastSlam2.fastslam2_update_unknown_odometry(g1, [0, 0, 0], [1, 0, 0], [(1.0, 0.1)])   # FastSLAM 1.0
    g2.enable_existence(10.0)
    with pytest.raises(rr.InvalidParameter, match="not supported"):
        g2.fastslam2_update_odometry([0, 0, 0], [1, 0, 0], [(1.0, 0.1, 0)])            # known ids with existence counters


@pytest.mark.parametrize("unknown", [False, True])
def test_step_all_in_process_ranks(unknown):
    """step_all_odometry / step_all_unknown_odometry on 2 in-process ranks: the oracle's state, bit for bit"""
    n, steps = 512, 8
    sc = scenarios.FastSlamScenario(4, (15.0, 15.0, 0.0), (1.0, 0.05), steps, seed=3, max_range=40.0)
    gs, o = _setup(2, n, sc.m + (4 if unknown else 0), sc, 2, seeded=not unknown)
    for t, (a, b) in enumerate(_drive(sc, steps)):
        if unknown:
            z = [(d, ang) for d, ang, _ in sc.obs[t]]
            did, odid = rr.FastSlam2.step_all_unknown_odometry(gs, a, b, z), o.step_unknown_odom(a, b, z)
        else:
            did, odid = rr.FastSlam2.step_all_odometry(gs, a, b, sc.obs[t]), o.step_odom(a, b, sc.obs[t])
        _check(gs, o, t, did, bool(odid))
        _same(gs, o, f"step {t}")


def test_cpp_mirror_fs_odom(tmp_path):
    """host/fs_odom_check.cpp through the C++ mirror: the Python mirror's numbers, bit for bit"""
    pkg, exe = os.path.join(ROOT, "rust_robotics_b200"), str(tmp_path / "fs_odom_check")
    subprocess.run(["/usr/bin/g++", "-std=c++17", "-O1", os.path.join(pkg, "host", "fs_odom_check.cpp"), "-I", os.path.join(ROOT, "include"),
                    "-I", os.path.join(pkg, "host"), "-L", pkg, "-lpfgpu", f"-Wl,-rpath,{pkg}", "-o", exe], check=True)
    r = subprocess.run([exe], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr
    got = np.array([float.fromhex(x) for x in r.stdout.split()])
    odom = [(0.0, 0.0, 0.0), (0.1, 0.0, 0.01), (0.1, 0.0, 0.01), (0.1, 0.0, 0.4), (0.05, -0.02, 0.41), (0.15, 0.02, 0.42)]
    z = [(5.0, 0.6, 0), (4.2, -0.5, 1), (6.5, 2.0, 2)]
    cfg = rr.FsConfig(nth=1024 / 1.5)
    f1, f2, fu = rr.FastSlam1(1024, 4, cfg, seed=7), rr.FastSlam2(1024, 4, cfg, seed=7), rr.FastSlam2(1024, 8, cfg, seed=7)
    f1.set_odometry_noise(0.1, 0.05, 0.1, 0.05)
    want = list(f1.odometry_noise())
    for t in range(len(odom) - 1):
        f1.fastslam_update_odometry(odom[t], odom[t + 1], z)
        f2.fastslam2_update_odometry(odom[t], odom[t + 1], z)
        fu.fastslam2_update_unknown_odometry(odom[t], odom[t + 1], [(d, a) for d, a, _ in z])
        for f in (f1, f2, fu):
            want += list(f.get_best_particle()[1])
    assert got.shape == (len(want),) and np.array_equal(got, np.array(want))


@pytest.mark.parametrize("world", [1, 2])
def test_fs_odom_multi_process(world):
    """one process per GPU (tests/mgpu_fs_odom_worker.py): the kernels' own waits and landmark reads through cudaIpc"""
    c = C.c_int()
    rr.load_library().pfgpu_device_count(C.byref(c))
    if c.value < world:
        pytest.skip(f"needs {world} GPUs")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={world}", "--master-addr", "127.0.0.1",
           "--master-port", "29571", os.path.join(ROOT, "tests", "mgpu_fs_odom_worker.py"), str(1024 * world), "12"]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0 and "MGPU_OK" in r.stdout, r.stdout[-2000:] + r.stderr[-4000:]


def _track(g, sc, odometry):
    """(mean position error over the drive, weighted position spread after every step) of FastSLAM 2.0 on FsOdomScenario"""
    err, spread = [], []
    for t in range(sc.steps):
        if odometry:
            g.fastslam2_update_odometry(*sc.odom_pair(t), sc.obs[t], want_flag=False)
        else:
            g.fastslam2_update(sc.controls[t], sc.obs[t], want_flag=False)
        p = g.state(landmarks=False)[0]
        w = p[:, 0] / p[:, 0].sum()
        mx, my = float((w * p[:, 1]).sum()), float((w * p[:, 2]).sum())
        err.append(math.hypot(mx - sc.truth[t][0], my - sc.truth[t][1]))
        spread.append(math.sqrt(float((w * ((p[:, 1] - mx) ** 2 + (p[:, 2] - my) ** 2)).sum())))
    return float(np.mean(err)), spread


def test_odometry_tracks_and_holds_still():
    """FsOdomScenario (a drive, a 15-step stop, a turn in place, a reverse, a drive; odometry with drift), 4096 particles, the
    velocity twin fed the controls that reproduce each odometry step.  Observed (the device equals the oracle bit for bit): mean
    position error 0.086 m with odometry against 0.260 m with velocity; across the stop the odometry cloud's spread goes from 0.190
    to 0.174 m, the velocity model's from 0.591 to 0.633 m."""
    sc = scenarios.FsOdomScenario()
    a, b = sc.phases["stop"]
    out = {}
    for odometry in (True, False):
        g = rr.FastSlam2(4096, sc.m, rr.FsConfig(nth=4096 / 1.5), seed=11)
        g.seed_map(sc.start, sc.landmarks)
        out[odometry] = _track(g, sc, odometry)
    (e_odo, s_odo), (e_vel, s_vel) = out[True], out[False]
    assert e_odo < 0.09 and e_vel > 0.25 and e_odo < e_vel, (e_odo, e_vel)
    assert s_odo[b - 1] <= s_odo[a - 1] < 0.2, (s_odo[a - 1], s_odo[b - 1])
    assert s_vel[b - 1] > s_vel[a - 1] > 0.55, (s_vel[a - 1], s_vel[b - 1])
