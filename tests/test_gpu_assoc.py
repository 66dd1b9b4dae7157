"""FastSLAM 2.0 with unknown data association (FastSlam2.fastslam2_update_unknown, pfgpu_fs_step_unknown; DESIGN §3.5) against the
CPU oracle (tests/host/fs2_assoc_oracle.c) bit for bit: poses, weights, every landmark field, resample indices, gate, N_eff, best
particle and the (matched, born, dropped) counts, over multi-step runs that resample (so ancestry rows are live when the kernel
reads through them) — and one behavioural check that the associations are the right ones."""
import math
import os

import numpy as np
import pytest

import rust_robotics_b200 as rr
from rust_robotics_b200 import scenarios
from _assoc_oracle import OracleFS2Assoc

pytestmark = pytest.mark.gpu
THREADS = max(1, min(32, os.cpu_count() or 1))


def _oracle(n, m, seed, **cfg):
    o = OracleFS2Assoc(n, m, seed=seed, **cfg)
    o.L.orc_fs_set_threads(o.h, THREADS)
    return o


def _noid(z):
    return [(d, a) for d, a, _ in z]


def _wide(steps):
    """36 landmarks (10 m grid) seen out to 80 m: all 36 observed every step, more than one warp's worth"""
    return scenarios.FastSlamScenario(6, (25.0, 5.0, 0.0), (1.0, 0.05), steps, seed=7, max_range=80.0)


def _same_state(g, o, what, lo=0):
    gp, gl = g.state()
    op, ol = o.state()
    op, ol = op[lo:lo + g.n_local], ol[lo:lo + g.n_local]
    assert np.array_equal(gp, op, equal_nan=True), f"{what}: poses / weights differ"
    assert np.array_equal(gl, ol, equal_nan=True), f"{what}: landmarks differ"


def _step_check(gs, o, t, did, odid, counts_too=True):
    assert did == odid, f"step {t}: gate"
    if did:
        assert np.array_equal(np.concatenate([g.last_indices() for g in gs]), o.last_indices()), f"step {t}: indices"
    # N_eff itself comes from tree-order sums on the device (only the gate decision is exact, DESIGN §3.2)
    assert math.isclose(gs[0].last_neff(), o.last_neff(), rel_tol=1e-9), f"step {t}: N_eff"
    for g in gs:
        assert g.get_best_particle()[0] == o.best(), f"step {t}: best particle"
    if counts_too:
        assert tuple(int(v) for v in np.sum([g.assoc_counts() for g in gs], axis=0)) == tuple(int(v) for v in o.counts), f"step {t}: counts"


def _run(n, m, sc, steps, seed=5, seeded=False, gate=16.0, world=1, every=True):
    cfg = rr.FsConfig(nth=n / 1.5)
    gs = rr.FastSlam2.create_sharded_local(n, m, [0] * world, cfg, seed=seed) if world > 1 else [rr.FastSlam2(n, m, cfg, seed=seed)]
    o = _oracle(n, m, seed, nth=n / 1.5)
    if seeded:
        for g in gs:
            g.seed_map(sc.start, sc.landmarks)
        o.seed_map(sc.start, sc.landmarks)
    else:
        pw = np.tile([1.0 / n, *sc.start], (n, 1))
        lm = np.tile([0.0, 0.0, 1000.0, 0.0, 0.0, 1000.0], (n, m, 1))
        for r, g in enumerate(gs):
            g.set_state(pw[r * g.n_local:(r + 1) * g.n_local], lm[r * g.n_local:(r + 1) * g.n_local])
        o.set_state(pw, lm)
    resamples, tot = 0, np.zeros(3, dtype=np.int64)
    for t in range(steps):
        z = _noid(sc.obs[t])
        did = rr.FastSlam2.step_all_unknown(gs, sc.control, z, gate) if world > 1 else gs[0].fastslam2_update_unknown(sc.control, z, gate)
        _step_check(gs, o, t, did, o.step_unknown(sc.control, z, gate))
        resamples += int(did)
        tot += o.counts.astype(np.int64)
        if every or t == steps - 1:
            for r, g in enumerate(gs):
                _same_state(g, o, f"step {t} rank {r}", r * g.n_local)
    return gs, o, resamples, tot


@pytest.mark.parametrize("n,m,seeded", [(64, 8, False), (1000, 8, False), (4096, 64, False), (65536, 8, False), (64, 0, False),
                                        (64, 1, False), (4096, 36, True), (1000, 36, True)])
def test_unknown_association_bit_exact(n, m, seeded):
    sc = _wide(8)
    assert max(len(z) for z in sc.obs) > 31
    gs, o, resamples, tot = _run(n, m, sc, 8, seeded=seeded)
    assert resamples > 1 or m == 0                                      # no slot: no weight ever changes
    if m == 0:
        assert tot[0] == 0 and tot[1] == 0 and tot[2] > 0
    if m <= 8:
        assert tot[2] > 0                                              # the map fills up: drops
    if not seeded and m >= 36:
        assert tot[1] > 0
    assert gs[0].stats().serial_fallbacks == 0


def test_config3_shape_seeded_bit_exact():
    """256 slots, the config-3 grid seeded (every slot initialised: every scan evaluates the metric for all 256)"""
    sc = scenarios.c3_scenario(steps=5)
    _run(4096, sc.m, sc, 5, seeded=True, every=False)


def test_config3_shape_fresh_65536():
    sc = scenarios.c3_scenario(steps=3)
    gs, o, resamples, tot = _run(65536, sc.m, sc, 3, every=False)
    assert tot[1] > 0 and tot[0] > 0


@pytest.mark.parametrize("gate", [math.inf, 1.0])
def test_gates(gate):
    sc = _wide(6)
    _run(1000, 40, sc, 6, seeded=False, gate=gate)


@pytest.mark.parametrize("world,n", [(2, 2048), (4, 4096), (2, 1920)])
def test_sharded_in_process_bit_exact(world, n):
    sc = _wide(8)
    gs, o, resamples, tot = _run(n, 40, sc, 8, world=world)
    assert resamples > 1
    idx = o.last_indices()
    # ancestors on other ranks: some slot's ancestor lives on another rank (checked at the last resample if it resampled last)
    if idx.size:
        nl = n // world
        assert (idx // nl != np.arange(n) // nl).any()


def test_global_tile_post_kernel(monkeypatch):
    monkeypatch.setenv("PFGPU_POST_SMEM_CAP", "0")
    monkeypatch.setenv("PFGPU_POST_TILES", "2")
    sc = _wide(6)
    gs, o, resamples, tot = _run(3000, 40, sc, 6)
    assert gs[0].post_shape()[3] == "global" and resamples > 0


def test_interleaved_with_known_id_steps():
    sc = _wide(10)
    n, m = 2048, sc.m
    g = rr.FastSlam2(n, m, rr.FsConfig(nth=n / 1.5), seed=8)
    o = _oracle(n, m, 8, nth=n / 1.5)
    g.seed_map(sc.start, sc.landmarks)
    o.seed_map(sc.start, sc.landmarks)
    resamples = 0
    for t in range(10):
        if t % 3 == 1:
            did, odid = g.fastslam2_update(sc.control, sc.obs[t]), bool(o.step(sc.control, sc.obs[t]))
            _step_check([g], o, t, did, odid, counts_too=False)
        else:
            did = g.fastslam2_update_unknown(sc.control, _noid(sc.obs[t]))
            _step_check([g], o, t, did, o.step_unknown(sc.control, _noid(sc.obs[t])))
        resamples += int(did)
        _same_state(g, o, f"step {t}")
    assert resamples > 1


def test_k0_is_the_known_id_step():
    sc = _wide(4)
    n, m = 1000, 40
    a, b = rr.FastSlam2(n, m, rr.FsConfig(nth=n / 1.5), seed=3), rr.FastSlam2(n, m, rr.FsConfig(nth=n / 1.5), seed=3)
    o = _oracle(n, m, 3, nth=n / 1.5)
    for t in range(4):
        z = [] if t % 2 == 0 else _noid(sc.obs[t])
        da = a.fastslam2_update_unknown(sc.control, z)
        db = b.fastslam2_update(sc.control, []) if not z else b.fastslam2_update_unknown(sc.control, z)
        _step_check([a], o, t, da, o.step_unknown(sc.control, z))
        assert da == db
        if not z:
            assert a.assoc_counts() == (0, 0, 0)
        pa, la = a.state()
        pb, lb = b.state()
        assert np.array_equal(pa, pb) and np.array_equal(la, lb)
        _same_state(a, o, f"step {t}")


def test_identical_slots_lower_index_wins():
    n, m = 64, 4
    g = rr.FastSlam2(n, m, rr.FsConfig(nth=0.0), seed=2)
    o = _oracle(n, m, 2, nth=0.0)
    pw = np.tile([1.0 / n, 0.0, 0.0, 0.0], (n, 1))
    lm = np.tile([0.0, 0.0, 1000.0, 0.0, 0.0, 1000.0], (n, m, 1))
    lm[:, 1] = lm[:, 2] = [10.0, 0.0, 1.0, 0.0, 0.0, 1.0]           # slots 1 and 2 identical, slot 0 and 3 empty
    g.set_state(pw, lm)
    o.set_state(pw, lm)
    z = [(10.0, 0.0)]
    _step_check([g], o, 0, g.fastslam2_update_unknown([1.0, 0.0], z), o.step_unknown([1.0, 0.0], z))
    _same_state(g, o, "step 0")
    _, l = g.state()
    assert g.assoc_counts() == (n, 0, 0)
    assert (l[:, 1] != lm[:, 1]).any(axis=1).all() and np.array_equal(l[:, 2], lm[:, 2])


def test_particle_on_a_landmark_and_odd_weights():
    """a particle whose predicted pose sits exactly on a landmark (d = 0: S is NaN and never wins), zero and NaN weights"""
    n, m = 128, 6
    g = rr.FastSlam2(n, m, rr.FsConfig(nth=n / 1.5), seed=4)
    o = _oracle(n, m, 4, nth=n / 1.5)
    rng = np.random.default_rng(4)
    pw = np.column_stack([np.full(n, 1.0 / n), rng.uniform(-1, 1, n), rng.uniform(-1, 1, n), rng.uniform(-3, 3, n)])
    lm = np.tile([0.0, 0.0, 1000.0, 0.0, 0.0, 1000.0], (n, m, 1))
    lm[:, 0, :] = np.column_stack([pw[:, 1], pw[:, 2], np.full(n, 2.0), np.zeros(n), np.zeros(n), np.full(n, 2.0)])
    lm[:, 1, :] = [5.0, 5.0, 2.0, 0.0, 0.0, 2.0]
    pw[3, 0] = 0.0
    pw[5, 0] = math.nan
    g.set_state(pw, lm)
    o.set_state(pw, lm)
    for t, z in enumerate([[(7.0, 0.8), (0.5, 0.0)], [(7.0, 0.8)], [(3.0, -1.0), (7.0, 0.8)]]):
        u = [0.0, 0.0] if t == 0 else [1.0, 0.1]                       # u = 0: x_pred is the pose itself, on landmark 0
        _step_check([g], o, t, g.fastslam2_update_unknown(u, z), o.step_unknown(u, z))
        _same_state(g, o, f"step {t}")
    pw[:, 0] = 0.0
    g.set_state(pw, lm)
    o.set_state(pw, lm)
    _step_check([g], o, 3, g.fastslam2_update_unknown([1.0, 0.1], [(7.0, 0.8)]), o.step_unknown([1.0, 0.1], [(7.0, 0.8)]))
    _same_state(g, o, "all-zero weights")


def test_refusals():
    g1 = rr.FastSlam1(64, 4)
    L = rr.load_library()
    with pytest.raises(rr.InvalidParameter):                          # FastSLAM 1.0: unsupported
        rr.FastSlam2.fastslam2_update_unknown(g1, [1.0, 0.0], [(1.0, 0.0)])
    assert "FastSLAM 2.0" in L.pfgpu_last_error().decode()
    g = rr.FastSlam2(64, 4)
    for gate in (0.0, -1.0, math.nan, -math.inf):
        with pytest.raises(rr.InvalidParameter):
            g.fastslam2_update_unknown([1.0, 0.0], [(1.0, 0.0)], gate)
    for z in ([(math.nan, 0.0)], [(1.0, math.inf)]):
        with pytest.raises(rr.InvalidParameter):
            g.fastslam2_update_unknown([1.0, 0.0], z)
    with pytest.raises(rr.InvalidParameter):
        g.fastslam2_update_unknown([math.nan, 0.0], [(1.0, 0.0)])
    g.fastslam2_update_unknown([1.0, 0.0], [(1.0, 0.0)], math.inf)    # +inf is a valid gate


def test_best_particle_map_has_one_slot_per_landmark():
    """Four landmarks 20 m apart around the start, the reference's noise (R = diag(0.5, 0.0305): at the ~14 m ranges here one
    observation is off by about 0.7 m in range and 2.4 m across the beam), ten steps: an observation of one landmark lies within the
    gate of that landmark's estimate and far outside any other's, so the best particle must end with exactly one initialised slot
    per landmark it has seen.  Each slot must lie within 3 m of its landmark: the average of about ten such observations (about
    0.8 m) plus the particle's own pose error (FastSLAM 2.0's MOTION_COV adds about 0.3 m per step and axis) — and well below half
    the spacing.  (Over much longer runs the reference's MOTION_COV lets the pose drift until a particle re-observes a landmark
    outside the gate and adds it twice: see DESIGN §3.5.)"""
    land = scenarios.grid_landmarks(4, pitch=20.0) + 5.0
    rng = np.random.default_rng(11)
    start, control = [35.0, 35.0, 0.0], [1.0, 0.1]
    x, obs, seen = list(start), [], set()
    for _ in range(10):
        x = scenarios.motion_model(x, control)
        z = scenarios.get_observations(x, land, rng)
        seen |= {l for _, _, l in z}
        obs.append(_noid(z))
    n, m = 4096, 32
    g = rr.FastSlam2(n, m, rr.FsConfig(nth=n / 1.5), seed=12)
    g.set_state(np.tile([1.0 / n, *start], (n, 1)), np.tile([0.0, 0.0, 1000.0, 0.0, 0.0, 1000.0], (n, m, 1)))
    for z in obs:
        g.fastslam2_update_unknown(control, z, want_flag=False)
    best, _ = g.get_best_particle()
    lm = g.particle_landmarks(best)
    est = lm[lm[:, 2] < 100.0, :2]
    assert len(seen) == 4 and len(est) == len(seen), (len(est), len(seen))
    d = np.hypot(est[:, None, 0] - land[None, :, 0], est[:, None, 1] - land[None, :, 1])
    assert sorted(d.argmin(axis=1).tolist()) == sorted(seen)          # one slot per landmark, no landmark twice
    assert d.min(axis=1).max() < 3.0, d.min(axis=1)


def test_cpp_mirror_update_unknown(tmp_path):
    """host/assoc_check.cpp through the C++ mirror's FastSlam::update_unknown: the Python mirror's numbers, bit for bit"""
    import subprocess
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    pkg = os.path.join(root, "rust_robotics_b200")
    exe = str(tmp_path / "assoc_check")
    subprocess.run(["/usr/bin/g++", "-std=c++17", "-O1", os.path.join(pkg, "host", "assoc_check.cpp"), "-I", os.path.join(root, "include"),
                    "-I", os.path.join(pkg, "host"), "-L", pkg, "-lpfgpu", f"-Wl,-rpath,{pkg}", "-o", exe], check=True)
    r = subprocess.run([exe], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr
    got = np.array([float(x) for x in r.stdout.split()])
    fs = rr.FastSlam2(1000, 6, seed=42)
    want = []
    for _ in range(4):
        did = fs.fastslam2_update_unknown([1.0, 0.1], [(5.0, 0.1), (7.0, -0.4), (5.1, 0.12)])
        want += [float(did)] + [float(c) for c in fs.assoc_counts()]
    idx, pw = fs.get_best_particle()
    want += list(pw)
    for l in fs.particle_landmarks(idx):
        want += [l[0], l[1], l[2]]
    assert got.shape == (len(want),) and np.array_equal(got, np.array(want))
