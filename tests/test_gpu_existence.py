"""Landmark existence counters (FastSlam2.enable_existence, pfgpu_fs_existence_*; DESIGN §3.7) against the CPU oracle
(tests/host/fs2_exist_oracle.c) bit for bit at every step: poses, weights, every landmark field, every counter (read through the
rows), resample indices, gate, best particle and (matched, born, dropped, removed); plus the long-run behaviour, the refusals and
the C++ mirror."""
import ctypes as C
import math
import os
import subprocess
import sys

import numpy as np
import pytest

import _existence as E
import rust_robotics_b200 as rr
from rust_robotics_b200 import scenarios
from _exist_oracle import OracleFS2Exist

pytestmark = pytest.mark.gpu
THREADS = max(1, min(32, os.cpu_count() or 1))
FRESH = [0.0, 0.0, 1000.0, 0.0, 0.0, 1000.0]


def _oracle(n, m, seed, **cfg):
    o = OracleFS2Exist(n, m, seed=seed, **cfg)
    o.L.orc_fs_set_threads(o.h, THREADS)
    return o


def _noid(z):
    return [(d, a) for d, a, _ in z]


def _wide(steps):
    """36 landmarks (10 m grid) seen out to 80 m: all 36 observed every step"""
    return scenarios.FastSlamScenario(6, (25.0, 5.0, 0.0), (1.0, 0.05), steps, seed=7, max_range=80.0)


def _initial(n, m, sc, phantoms):
    """fresh maps; with phantoms, the first half of the slots hold landmarks nothing observes, 3 to 12 m from the start, so that
    copies are removed and their slots reused"""
    pw = np.tile([1.0 / n, *sc.start], (n, 1))
    lm = np.tile(FRESH, (n, m, 1))
    if phantoms:
        rng = np.random.default_rng(n * 7 + m)
        k = m // 2
        ang, rad = rng.uniform(-math.pi, math.pi, (n, k)), rng.uniform(3.0, 12.0, (n, k))
        lm[:, :k, 0] = sc.start[0] + 5.0 + rad * np.cos(ang)
        lm[:, :k, 1] = sc.start[1] + 5.0 + rad * np.sin(ang)
        lm[:, :k, 2] = lm[:, :k, 5] = 0.5
        lm[:, :k, 3] = lm[:, :k, 4] = 0.0
    return pw, lm


def _check(gs, o, t, did, odid, tracking):
    assert did == odid, f"step {t}: gate"
    if did:
        assert np.array_equal(np.concatenate([g.last_indices() for g in gs]), o.last_indices()), f"step {t}: indices"
    for g in gs:
        assert g.get_best_particle()[0] == o.best(), f"step {t}: best particle"
    assert tuple(int(v) for v in np.sum([g.assoc_counts() for g in gs], axis=0)) == tuple(int(v) for v in o.counts), f"step {t}: counts"
    gp = np.concatenate([g.state()[0] for g in gs])
    gl = np.concatenate([g.state()[1] for g in gs])
    op, ol = o.state()
    assert np.array_equal(gp, op, equal_nan=True), f"step {t}: poses / weights"
    assert np.array_equal(gl, ol, equal_nan=True), f"step {t}: landmarks"
    if tracking:
        assert sum(g.removed_count() for g in gs) == o.removed, f"step {t}: removed"
        assert np.array_equal(np.concatenate([g.existence_counts() for g in gs]), o.existence_counts()), f"step {t}: counters"
    else:
        assert all(g.removed_count() == 0 for g in gs)


def _run(n, m, sc, steps, r=8.0, seed=5, seeded=False, phantoms=True, world=1, enable_at=0, disable_at=None, k0_at=(), reset_at=None):
    cfg = rr.FsConfig(nth=n / 1.5)
    gs = rr.FastSlam2.create_sharded_local(n, m, [0] * world, cfg, seed=seed) if world > 1 else [rr.FastSlam2(n, m, cfg, seed=seed)]
    o = _oracle(n, m, seed, nth=n / 1.5)
    nl = n // world
    if seeded:
        for g in gs:
            g.seed_map(sc.start, sc.landmarks)
        o.seed_map(sc.start, sc.landmarks)
    else:
        pw, lm = _initial(n, m, sc, phantoms)
        for q, g in enumerate(gs):
            g.set_state(pw[q * nl:(q + 1) * nl], lm[q * nl:(q + 1) * nl])
        o.set_state(pw, lm)
    tracking, tot = False, np.zeros(4, dtype=np.int64)
    for t in range(steps):
        if t == enable_at:
            for g in gs:
                g.enable_existence(r)
            o.enable_existence(r)
            tracking = True
        if t == disable_at:
            for g in gs:
                g.enable_existence(0)
            o.enable_existence(0)
            tracking = False
        if t == reset_at:                                              # upload: every counter back to 1
            pw, lm = o.state()
            for q, g in enumerate(gs):
                g.set_state(pw[q * nl:(q + 1) * nl], lm[q * nl:(q + 1) * nl])
            o.set_state(pw, lm)
        z = [] if t in k0_at else _noid(sc.obs[t])
        if world > 1:
            did = rr.FastSlam2.step_all_unknown(gs, sc.control, z)
        else:
            did = gs[0].fastslam2_update_unknown(sc.control, z)
        odid = o.step_unknown(sc.control, z)
        _check(gs, o, t, did, odid, tracking)
        tot += np.array([*o.counts.astype(np.int64), o.removed if tracking else 0])
    return gs, o, tot


@pytest.mark.parametrize("n,m,seeded", [(64, 8, False), (1000, 8, False), (4096, 64, False), (65536, 8, False), (64, 1, False),
                                        (1000, 36, True), (4096, 36, True)])
def test_existence_bit_exact(n, m, seeded):
    sc = _wide(8)
    gs, o, tot = _run(n, m, sc, 8, seeded=seeded, k0_at=(5,))
    assert tot[3] > 0 or m == 1 or seeded                              # removals (the phantom landmarks)
    assert gs[0].stats().resamples > 1


def test_config3_shape_256_slots():
    """2^16 particles x 256 slots, fresh maps on the config-3 grid, counters on"""
    sc = scenarios.c3_scenario(steps=3)
    gs, o, tot = _run(65536, sc.m, sc, 3, phantoms=True, r=20.0)
    assert tot[1] > 0 and tot[3] > 0


def test_enabled_mid_run_and_resets():
    """enabled after steps that left rows live; set_state (upload) and seed_map restart every counter at 1; k = 0 steps; r = inf"""
    sc = _wide(10)
    _run(2048, 40, sc, 10, enable_at=3, reset_at=6, k0_at=(4, 8), r=math.inf)
    gs, o, tot = _run(1000, 36, sc, 6, seeded=True, enable_at=2, k0_at=(0, 3))
    for g in gs:
        g.seed_map(sc.start, sc.landmarks)
    o.seed_map(sc.start, sc.landmarks)
    assert np.array_equal(gs[0].existence_counts(), o.existence_counts()) and (o.existence_counts() == 1).all()


def test_k0_only_and_disable():
    """steps without observations (the motion step, then the negative evidence); and after disabling, the untracked step's bits"""
    sc = _wide(8)
    gs, o, tot = _run(4096, 16, sc, 5, k0_at=range(5), r=12.0)
    assert tot[3] > 0 and tot[:3].sum() == 0
    gs, o, tot = _run(2048, 40, sc, 8, enable_at=1, disable_at=4)
    assert tot[3] > 0


def test_global_tile_post_kernel(monkeypatch):
    monkeypatch.setenv("PFGPU_POST_SMEM_CAP", "0")
    monkeypatch.setenv("PFGPU_POST_TILES", "2")
    sc = _wide(6)
    gs, o, tot = _run(3000, 40, sc, 6)
    assert gs[0].post_shape()[3] == "global" and tot[3] > 0


@pytest.mark.parametrize("world,n", [(2, 2048), (4, 4096)])
def test_sharded_in_process(world, n):
    sc = _wide(8)
    gs, o, tot = _run(n, 40, sc, 8, world=world, k0_at=(6,))
    idx = o.last_indices()
    assert tot[3] > 0 and gs[0].stats().resamples > 1
    if idx.size:
        nl = n // world
        assert (idx // nl != np.arange(n) // nl).any()                 # ancestors on other ranks


@pytest.mark.parametrize("world", [1, 2])
def test_existence_multi_process(world):
    """one process per GPU (tests/mgpu_existence_worker.py): peers' counters through cudaIpc"""
    c = C.c_int()
    rr.load_library().pfgpu_device_count(C.byref(c))
    if c.value < world:
        pytest.skip(f"needs {world} GPUs")
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={world}", "--master-addr", "127.0.0.1",
           "--master-port", "29551", os.path.join(root, "tests", "mgpu_existence_worker.py"), str(1024 * world), "10"]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0 and "MGPU_OK" in r.stdout, r.stdout[-2000:] + r.stderr[-4000:]


def test_refusals():
    L = rr.load_library()
    g = rr.FastSlam2(64, 4)
    for r in (math.nan, -1.0, -math.inf):
        with pytest.raises(rr.InvalidParameter):
            g.enable_existence(r)
    with pytest.raises(rr.InvalidParameter):                          # counters disabled: nothing to read
        g.existence_counts()
    g.enable_existence()                                               # config.max_range
    with pytest.raises(rr.InvalidParameter):
        g.fastslam2_update([1.0, 0.0], [(5.0, 0.1, 0)])
    assert "existence" in L.pfgpu_last_error().decode()
    g.fastslam2_update_unknown([1.0, 0.0], [(5.0, 0.1)])
    g.enable_existence(0)
    g.fastslam2_update([1.0, 0.0], [(5.0, 0.1, 0)])                    # disabled again: known ids are fine
    assert g.removed_count() == 0


def test_long_run_maps_stop_filling():
    """test_fs2_existence_oracle.py's 1 000-step run on the GPU, with the same assertions (and, bit-exact, the same numbers)"""
    sc = E.scenario()
    out = []
    for r in (E.RANGE, 0.0):
        g = rr.FastSlam2(E.N, E.M, rr.FsConfig(nth=E.N / 1.5), seed=E.SEED)
        g.set_state(np.tile([1.0 / E.N, *sc.start], (E.N, 1)), np.tile(FRESH, (E.N, E.M, 1)))
        if r:
            g.enable_existence(r)

        def step(u, z):
            g.fastslam2_update_unknown(u, z, want_flag=False)
            return g.assoc_counts()[2], g.removed_count()
        out.append(E.run(step, lambda: g.particle_landmarks(g.get_best_particle()[0]), sc))
    on, off = out
    E.check(on, off)
    assert on[-1, 0] == 49 and on[-1, 1] == 55 and on[:, 3].sum() == 16014
    assert off[-1, 2] == 1820


def test_cpp_mirror_existence(tmp_path):
    """host/existence_check.cpp through the C++ mirror: the Python mirror's numbers, bit for bit"""
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    pkg = os.path.join(root, "rust_robotics_b200")
    exe = str(tmp_path / "existence_check")
    subprocess.run(["/usr/bin/g++", "-std=c++17", "-O1", os.path.join(pkg, "host", "existence_check.cpp"), "-I", os.path.join(root, "include"),
                    "-I", os.path.join(pkg, "host"), "-L", pkg, "-lpfgpu", f"-Wl,-rpath,{pkg}", "-o", exe], check=True)
    r = subprocess.run([exe], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr
    got = np.array([float(x) for x in r.stdout.split()])
    fs = rr.FastSlam2(1000, 6, seed=42)
    fs.enable_existence(6.0)
    want = []
    for t in range(6):
        z = [(5.0, 0.1), (7.0, -0.4)] if t % 3 != 2 else [(3.0, 1.2)]
        did = fs.fastslam2_update_unknown([1.0, 0.1], z)
        want += [float(did), float(fs.removed_count())]
    idx, _ = fs.get_best_particle()
    want += [float(v) for v in fs.existence_counts(idx, 1)[0]]
    assert got.shape == (len(want),) and np.array_equal(got, np.array(want))
