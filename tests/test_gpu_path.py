"""FastSLAM path history (FastSlam1.enable_history / path / path_estimate; pfgpu_fs_history_enable, pfgpu_fs_path,
pfgpu_fs_path_moments; DESIGN §3.6) against the definition restated from the CPU oracle (tests/_path_oracle.py): per-step poses
from state() and resample parents from last_indices(), backtracked.  Paths must match bit for bit; the smoothed moments match a
float64 numpy restatement at the estimate tests' tolerance."""
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
from _assoc_oracle import OracleFS2Assoc
from _path_oracle import Genealogy, ref_path_estimate

pytestmark = pytest.mark.gpu
THREADS = max(1, min(32, os.cpu_count() or 1))


def _small(steps, start=(15.0, 15.0, 0.0), control=(1.0, 0.025), seed=42):
    """16 landmarks (10 m grid): a map small enough for the oracle's state at 65 536 particles"""
    return scenarios.FastSlamScenario(4, start, control, steps, seed=seed)


class Run:
    """GPU engine(s) and the CPU oracle stepped side by side; gen follows the oracle while history is enabled"""

    def __init__(self, oracle_lib, variant, n, sc, seed=7, world=1, unknown=False, seeded=True):
        self.sc, self.n, self.unknown, self.t = sc, n, unknown, 0
        cls = rr.FastSlam1 if variant == 1 else rr.FastSlam2
        cfg = rr.FsConfig(nth=n / 1.5)
        self.gs = cls.create_sharded_local(n, sc.m, [0] * world, cfg, seed=seed) if world > 1 else [cls(n, sc.m, cfg, seed=seed)]
        self.o = OracleFS2Assoc(n, sc.m, seed=seed, nth=n / 1.5) if unknown else OracleFS(oracle_lib, n, sc.m, seed=seed, variant=variant, nth=n / 1.5)
        self.o.L.orc_fs_set_threads(self.o.h, THREADS)
        self.gen = None
        if seeded:
            self.seed_map()

    def seed_map(self):
        for g in self.gs:
            g.seed_map(self.sc.start, self.sc.landmarks)
        self.o.seed_map(self.sc.start, self.sc.landmarks)
        if self.gen is not None:
            self.gen.root(self.t, self.o.state()[0])

    def set_state(self, pw, lm):
        nl = self.gs[0].n_local
        for r, g in enumerate(self.gs):
            g.set_state(pw[r * nl:(r + 1) * nl], lm[r * nl:(r + 1) * nl])
        self.o.set_state(pw, lm)
        if self.gen is not None:
            self.gen.root(self.t, self.o.state()[0])

    def enable(self, cap):
        for g in self.gs:
            g.enable_history(cap)
        self.gen = Genealogy(cap)
        self.gen.root(self.t, self.o.state()[0])

    def step(self):
        z = self.sc.obs[self.t % len(self.sc.obs)]
        u = self.sc.control
        if self.unknown:
            zz = [(d, a) for d, a, _ in z]
            for g in self.gs:
                g.fastslam2_update_unknown(u, zz, want_flag=False)
            odid = self.o.step_unknown(u, zz)
        else:
            for g in self.gs:
                g.fastslam_update(u, z, want_flag=False)
            odid = self.o.step(u, z)
        for g in self.gs:
            g.sync()
        did = self.gs[0].did_resample()
        assert did == bool(odid), f"step {self.t}: gate"
        self.t += 1
        if self.gen is not None:
            self.gen.record(self.t, self.o.state()[0], self.o.last_indices())
        return did

    def check_paths(self, slots, what, max_steps=None):
        first, last = self.gen.window()
        for g in self.gs:
            assert g.history_window() == (first, last), f"{what}: window"
        for s in slots:
            want = self.gen.path(s, max_steps)
            for r, g in enumerate(self.gs):
                got = g.path(s, max_steps)
                assert np.array_equal(got.steps, want[0]), f"{what}: slot {s} rank {r} steps"
                assert np.array_equal(got.slots, want[1]), f"{what}: slot {s} rank {r} slots"
                assert np.array_equal(got.poses, want[2]), f"{what}: slot {s} rank {r} poses"

    def slots(self, k=8, seed=0):
        best = self.o.best()
        assert all(g.get_best_particle()[0] == best for g in self.gs)
        rng = np.random.default_rng(seed)
        return sorted({best, 0, self.n - 1, *rng.integers(0, self.n, k).tolist()})

    def check_moments(self, what, max_steps=None):
        pw, _ = self.o.state()
        steps, mean, cov = ref_path_estimate(self.gen, pw[:, 0], max_steps)
        est = rr.FastSlam1.path_estimate_all(self.gs, max_steps) if len(self.gs) > 1 else self.gs[0].path_estimate(max_steps)
        assert np.array_equal(est.steps, steps), f"{what}: steps"
        _close(est.pose, mean, f"{what}: mean")
        for j in range(len(steps)):
            _close(est.pose_cov[j], cov[j], f"{what}: cov at step {steps[j]}", scale=np.max(np.abs(cov[j])) + 1e-300)
        return est


def _close(got, ref, what, scale=None):
    got, ref = np.asarray(got), np.asarray(ref)
    assert np.array_equal(np.isnan(got), np.isnan(ref)), f"{what}: NaN pattern"
    ok = ~np.isnan(ref)
    tol = 1e-9 * ((1.0 + np.abs(ref)) if scale is None else scale)
    bad = ok & ~(np.abs(got - ref) <= tol)
    assert not bad.any(), f"{what}: {np.argwhere(bad)[:4].tolist()} got {got[bad][:4]} want {ref[bad][:4]}"


# ---------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("variant", [1, 2])
@pytest.mark.parametrize("n", [64, 1000, 65536])
def test_path_against_oracle(oracle, variant, n):
    """best, first, last and sampled slots after a run with resamples and steps without; then the smoothed moments"""
    steps = 12
    run = Run(oracle, variant, n, _small(steps))
    run.enable(1000)
    kinds = [run.step() for _ in range(steps)]
    assert any(kinds)
    run.check_paths(run.slots(), f"variant {variant} n {n}")
    run.check_paths(run.slots(seed=1)[:3], f"variant {variant} n {n} last 5", max_steps=5)
    run.check_moments(f"variant {variant} n {n}")


def test_path_unknown_association():
    n, steps = 1000, 8
    sc = scenarios.FastSlamScenario(6, (25.0, 5.0, 0.0), (1.0, 0.05), steps, seed=7, max_range=80.0)
    run = Run(None, 2, n, sc, seed=5, unknown=True, seeded=False)
    run.enable(100)
    pw = np.tile([1.0 / n, *sc.start], (n, 1))
    run.set_state(pw, np.tile([0.0, 0.0, 1000.0, 0.0, 0.0, 1000.0], (n, sc.m, 1)))      # (restarts the window at step 0)
    assert sum(run.step() for _ in range(steps)) > 1
    run.check_paths(run.slots(), "unknown association")
    run.check_moments("unknown association")


def test_path_ring_wraps(oracle):
    """C = 5 entries over 17 steps: the window is the last five steps; its oldest entry is a root"""
    run = Run(oracle, 1, 1000, _small(17))
    run.enable(5)
    for _ in range(17):
        run.step()
    assert run.gs[0].history_window() == (13, 17)
    run.check_paths(run.slots(), "wrapped")
    run.check_moments("wrapped")


def test_path_enable_late_and_restart(oracle):
    """history enabled part-way through a run; set_state and seed_map restart the window at the current step"""
    n = 1000
    run = Run(oracle, 2, n, _small(30))
    for _ in range(4):
        run.step()
    run.enable(50)
    assert run.gs[0].history_window() == (4, 4)
    for _ in range(6):
        run.step()
    run.check_paths(run.slots(), "enabled at step 4")
    pw, lm = run.o.state()
    run.set_state(pw, lm)
    assert run.gs[0].history_window() == (10, 10)
    run.check_paths(run.slots(), "right after set_state")
    for _ in range(5):
        run.step()
    run.check_paths(run.slots(), "after set_state")
    run.seed_map()
    assert run.gs[0].history_window() == (15, 15)
    for _ in range(4):
        run.step()
    run.check_paths(run.slots(), "after seed_map")
    run.check_moments("after seed_map")


def test_path_global_tile_post(oracle, monkeypatch):
    monkeypatch.setenv("PFGPU_POST_SMEM_CAP", "0")
    run = Run(oracle, 1, 4096, _small(10))
    assert run.gs[0].post_shape()[3] == "global"
    run.enable(20)
    assert any([run.step() for _ in range(10)])
    run.check_paths(run.slots(), "global tile")


def test_path_moments_yaw_across_pi(oracle):
    """a cloud whose yaws straddle +-pi: wrapped about the centre; two calls return the same bits"""
    n, steps = 1000, 8
    sc = _small(steps, start=(15.0, 15.0, math.pi), control=(1.0, 0.0))
    run = Run(oracle, 1, n, sc, seeded=False)
    run.enable(20)
    rng = np.random.default_rng(4)
    yaw = math.pi + rng.uniform(-0.05, 0.05, n)
    yaw = np.where(yaw > math.pi, yaw - 2.0 * math.pi, yaw)
    pw = np.stack([np.full(n, 1.0 / n), 15.0 + rng.normal(0, 0.1, n), 15.0 + rng.normal(0, 0.1, n), yaw], axis=1)
    lm = np.tile([0.0, 0.0, 1000.0, 0.0, 0.0, 1000.0], (n, sc.m, 1))
    run.set_state(pw, lm)
    for _ in range(steps):
        run.step()
    est = run.check_moments("yaw across pi")
    assert (np.abs(est.pose[:, 2]) > 3.0).all()
    a, b = run.gs[0].path_moments(), run.gs[0].path_moments()
    assert np.array_equal(a[0], b[0]) and all(bytes(x) == bytes(y) for x, y in zip(a[1], b[1]))


@pytest.mark.parametrize("world", [2, 4, 8])
def test_path_sharded_in_process(oracle, world):
    """every rank's path of every queried global slot = the one-GPU engine's, lineages crossing ranks included; per-step merged
    moments = the one-GPU moments up to summation order"""
    n, steps = 1024, 12
    sc = _small(steps)
    one = Run(oracle, 1, n, sc, seed=9)
    sh = Run(oracle, 1, n, sc, seed=9, world=world)
    one.enable(100); sh.enable(100)
    for _ in range(steps):
        one.step(); sh.step()
    slots = one.slots(k=24)
    crossed = 0
    for s in slots:
        want = one.gs[0].path(s)
        crossed += int(len(set((want.slots // (n // world)).tolist())) > 1)
        for r, g in enumerate(sh.gs):
            got = g.path(s)
            assert all(np.array_equal(x, y) for x, y in zip(got, want)), f"world {world} rank {r} slot {s}"
    assert crossed > 0
    sh.check_paths(slots, f"world {world} vs oracle")
    a, b = one.gs[0].path_estimate(), rr.FastSlam1.path_estimate_all(sh.gs)
    assert np.array_equal(a.steps, b.steps)
    _close(b.pose, a.pose, f"world {world}: mean")
    for j in range(len(a.steps)):
        _close(b.pose_cov[j], a.pose_cov[j], f"world {world}: cov {j}", scale=np.max(np.abs(a.pose_cov[j])) + 1e-300)


@pytest.mark.parametrize("world", [1, 2])
def test_path_multi_process(world):
    """one process per GPU (tests/mgpu_path_worker.py): peers' rings through cudaIpc; world = 1 runs the script on one GPU"""
    c = C.c_int()
    rr.load_library().pfgpu_device_count(C.byref(c))
    if c.value < world:
        pytest.skip(f"needs {world} GPUs")
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={world}", "--master-addr", "127.0.0.1",
           "--master-port", "29549", os.path.join(root, "tests", "mgpu_path_worker.py"), str(1024 * world), "12"]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0 and "MGPU_OK" in r.stdout, r.stdout[-2000:] + r.stderr[-4000:]


@pytest.mark.parametrize("world", [1, 2])
def test_history_leaves_step_unchanged(oracle, world):
    """with history enabled: gate, indices, best particle and state bit for bit the oracle's and an engine's without history;
    exactly one more kernel launch per step, and none once disabled"""
    n, steps = 1024, 10
    sc = _small(2 * steps)
    hist = Run(oracle, 2, n, sc, seed=4, world=world)
    plain = Run(oracle, 2, n, sc, seed=4, world=world)
    hist.enable(64)
    l0h, l0p = [g.stats().kernel_launches for g in hist.gs], [g.stats().kernel_launches for g in plain.gs]
    for t in range(steps):
        a, b = hist.step(), plain.step()
        assert a == b
        if a:
            assert np.array_equal(np.concatenate([g.last_indices() for g in hist.gs]), hist.o.last_indices())
            assert np.array_equal(np.concatenate([g.last_indices() for g in hist.gs]), np.concatenate([g.last_indices() for g in plain.gs]))
        assert hist.gs[0].get_best_particle()[0] == plain.gs[0].get_best_particle()[0] == hist.o.best()
    for r in range(world):
        dh = hist.gs[r].stats().kernel_launches - l0h[r]
        dp = plain.gs[r].stats().kernel_launches - l0p[r]
        assert dh == dp + steps, f"rank {r}: {dh} launches with history, {dp} without"
    op, ol = hist.o.state()
    nl = hist.gs[0].n_local
    for r, (g, q) in enumerate(zip(hist.gs, plain.gs)):
        gp, gl = g.state()
        qp, ql = q.state()
        assert np.array_equal(gp, qp) and np.array_equal(gl, ql)
        assert np.array_equal(gp, op[r * nl:(r + 1) * nl]) and np.array_equal(gl, ol[r * nl:(r + 1) * nl])
    for g in hist.gs:
        g.enable_history(0)
    hist.gen = None
    l1h, l1p = [g.stats().kernel_launches for g in hist.gs], [g.stats().kernel_launches for g in plain.gs]
    for _ in range(3):
        assert hist.step() == plain.step()
    for r in range(world):
        assert hist.gs[r].stats().kernel_launches - l1h[r] == plain.gs[r].stats().kernel_launches - l1p[r], f"rank {r}: disabled"


def test_history_validation(oracle):
    run = Run(oracle, 1, 64, _small(6))
    g = run.gs[0]
    with pytest.raises(rr.api.InvalidParameter):
        g.history_window()
    with pytest.raises(rr.api.InvalidParameter):
        g.path(0, max_steps=4)
    with pytest.raises(rr.api.InvalidParameter):
        g.path_moments(max_steps=4)
    run.enable(4)
    run.step(); run.step()
    with pytest.raises(rr.api.InvalidParameter):
        g.path(64)
    with pytest.raises(rr.api.InvalidParameter):
        g.path(0, max_steps=0)
    with pytest.raises(rr.api.InvalidParameter):
        g.path_moments(max_steps=0)
    with pytest.raises(rr.api.PfgpuError):
        g.enable_history(1 << 31)                 # 2^31 entries x 64 slots x 28 B: does not fit; history stays as it was
    assert g.history_window() == (0, 2)
    run.check_paths([0, 63], "after a refused enable")
    g.enable_history(0)
    run.gen = None
    with pytest.raises(rr.api.InvalidParameter):
        g.path(0, max_steps=4)
    run.step()
    run.enable(3)
    assert g.history_window() == (3, 3)
    run.step(); run.step(); run.step()
    assert g.history_window() == (4, 6)
    run.check_paths([0, 31, 63], "re-enabled")


def test_cpp_mirror_path(tmp_path):
    """host/path_check.cpp through the C++ mirror's FastSlam::path(): the Python mirror's path, bit for bit"""
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    pkg = os.path.join(root, "rust_robotics_b200")
    exe = str(tmp_path / "path_check")
    subprocess.run(["/usr/bin/g++", "-std=c++17", "-O1", os.path.join(pkg, "host", "path_check.cpp"), "-I", os.path.join(root, "include"),
                    "-I", os.path.join(pkg, "host"), "-L", pkg, "-lpfgpu", f"-Wl,-rpath,{pkg}", "-o", exe], check=True)
    r = subprocess.run([exe], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr
    got = np.array([float(x) for x in r.stdout.split()]).reshape(-1, 5)
    fs = rr.FastSlam1(1000, 4, seed=42)
    fs.enable_history(100)
    for _ in range(5):
        fs.fastslam_update([1.0, 0.1], [(5.0, 0.1, 0), (7.0, -0.4, 2)])
    p = fs.path()
    want = np.column_stack([p.steps.astype(np.float64), p.slots.astype(np.float64), p.poses])
    assert got.shape == want.shape and np.array_equal(got, want)
