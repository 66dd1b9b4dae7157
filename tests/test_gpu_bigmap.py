"""FastSLAM maps of more than 1 024 landmarks per particle (up to 65 536): the CUDA path against the CPU oracle, bit for bit.

Past 1 024 landmarks the post kernel's lazy-clone bookkeeping (live-row bitmap, row list, retarget of the identity landmarks)
spans several bitmap words per CTA slice and row ids above 1 023; these runs cover FastSLAM 1.0 and 2.0, one GPU and the sharded
engine (all ranks in this process, on one device).
"""
import math

import numpy as np
import pytest

import rust_robotics_b200 as rr
from rust_robotics_b200 import scenarios
from _oracle import OracleFS

pytestmark = pytest.mark.gpu

FULL_STATE_EVERY_BYTES = 1 << 28     # compare every landmark at intervals while the map state stays below this many bytes


def _mid_circle(side, steps):
    """side x side grid at 10 m pitch; C3's 40 m circle (u = (1.0, 0.025)) centred on the middle of the grid"""
    mid = 10.0 * (side - 1) / 2.0
    return scenarios.FastSlamScenario(side, (mid, mid - 40.0, 0.0), (1.0, 0.025), steps)


def _compare(g, o, what, landmarks=True):
    gp, gl = g.state(landmarks)
    op, ol = o.state()
    assert np.array_equal(gp, op), f"{what}: pose/weight rows {np.flatnonzero((gp != op).any(axis=1))[:5]}"
    if landmarks:
        assert np.array_equal(gl, ol), f"{what}: landmarks differ for particles {np.flatnonzero((gl != ol).any(axis=(1, 2)))[:5]}"


def _shard_compare(ranks, o, what):
    op, ol = o.state()
    for r, g in enumerate(ranks):
        lo, hi = r * g.n_local, (r + 1) * g.n_local
        gp, gl = g.state()
        assert np.array_equal(gp, op[lo:hi]), f"{what}: rank {r} pose/weight rows differ"
        assert np.array_equal(gl, ol[lo:hi]), f"{what}: rank {r} landmarks differ for particles {np.flatnonzero((gl != ol[lo:hi]).any(axis=(1, 2)))[:5]}"


@pytest.mark.parametrize("variant", [1, 2])
@pytest.mark.parametrize("side", [33, 64, 128])
@pytest.mark.parametrize("n,steps", [(64, 24), (1000, 16), (4096, 12)])
def test_bigmap_trajectory_bit_exact(oracle, variant, side, n, steps):
    """1 089, 4 096 and 16 384 landmarks: gate, ancestry and best particle every step, the whole state at intervals and at the end"""
    sc = _mid_circle(side, steps)
    cls = rr.FastSlam1 if variant == 1 else rr.FastSlam2
    g = cls(n, sc.m, rr.FsConfig(nth=n / 1.5), seed=7)
    o = OracleFS(oracle, n, sc.m, seed=7, variant=variant, nth=n / 1.5)
    g.seed_map(sc.start, sc.landmarks); o.seed_map(sc.start, sc.landmarks)
    assert 8 <= sc.mean_k() <= 16
    full = n * sc.m * 48 <= FULL_STATE_EVERY_BYTES
    resamples = 0
    for t in range(steps):
        did = g.fastslam_update(sc.control, sc.obs[t]) if variant == 1 else g.fastslam2_update(sc.control, sc.obs[t])
        assert did == bool(o.step(sc.control, sc.obs[t])), f"step {t}: gate"
        if did:
            resamples += 1
            assert np.array_equal(g.last_indices(), o.last_indices()), f"step {t}: indices"
        assert g.get_best_particle()[0] == o.best(), f"step {t}: best particle"
        if t % 5 == 2:
            _compare(g, o, f"step {t}", landmarks=full)
    _compare(g, o, "end")
    assert resamples > 1
    assert g.stats().serial_fallbacks == 0


def _corridor(m, steps, speed=1.2, max_range=2.5, seed=3):
    """m landmarks 1 m apart on the x axis; the robot drives along it 1 m to the side at `speed` m per step"""
    lm = np.stack([np.arange(m, dtype=np.float64), np.zeros(m)], axis=1)
    u = [speed / 0.1, 0.0]
    rng = np.random.default_rng(seed)
    x = [0.0, 1.0, 0.0]
    obs = []
    for _ in range(steps):
        x = scenarios.motion_model(x, u)
        obs.append(scenarios.get_observations(x, lm, rng, max_range=max_range))
    return lm, u, [0.0, 1.0, 0.0], obs


def _max_live_rows(m, obs, gates):
    """the lazy clone's live ancestry rows, from the observation lists and the gate sequence alone: a landmark updated in a
    step reads its own columns (identity); a resample gives every identity landmark one row shared by all of them; a row is
    live while some landmark still reads through it"""
    row = np.full(m, -1, dtype=np.int64)           # -1: identity; otherwise the resample that gave the landmark its row
    best = 0
    for t, (z, gate) in enumerate(zip(obs, gates)):
        for _, _, l in z:
            row[l] = -1
        if gate:
            row[row < 0] = t
        best = max(best, len(np.unique(row[row >= 0])))
    return best


def test_bigmap_many_live_rows_bit_exact(oracle):
    """a corridor of 2 048 landmarks passed at 1.2 m per step with nth = n: at least one landmark leaves the view every step and
    keeps the row of the resample before, so more than 1 024 ancestry rows are live at once (row ids above 1 023, row lists
    compacted from many bitmap words)"""
    n, m, steps = 128, 2048, 1240
    lm, u, start, obs = _corridor(m, steps)
    assert all(len(z) > 0 for z in obs)
    g = rr.FastSlam1(n, m, rr.FsConfig(nth=float(n), max_range=2.5), seed=5)
    o = OracleFS(oracle, n, m, seed=5, nth=float(n), max_range=2.5)
    g.seed_map(start, lm); o.seed_map(start, lm)
    gates = []
    for t in range(steps):
        did = g.fastslam_update(u, obs[t])
        assert did == bool(o.step(u, obs[t])), f"step {t}: gate"
        gates.append(did)
        if did:
            assert np.array_equal(g.last_indices(), o.last_indices()), f"step {t}: indices"
        assert g.get_best_particle()[0] == o.best(), f"step {t}: best particle"
        if t % 100 == 99:
            _compare(g, o, f"step {t}")
    _compare(g, o, "end")
    live = _max_live_rows(m, obs, gates)
    assert live > 1024, f"only {live} ancestry rows were live at once"
    assert g.stats().serial_fallbacks == 0


def test_bigmap_65536_landmarks(oracle):
    """the largest map: seed_map, steps with a resample and download, bit for bit"""
    n = 64
    sc = _mid_circle(256, 8)
    assert sc.m == 65536
    g = rr.FastSlam1(n, sc.m, rr.FsConfig(nth=n / 1.5), seed=13)
    o = OracleFS(oracle, n, sc.m, seed=13, nth=n / 1.5)
    g.seed_map(sc.start, sc.landmarks); o.seed_map(sc.start, sc.landmarks)
    _compare(g, o, "seed")
    resamples = 0
    for t in range(8):
        did = g.fastslam_update(sc.control, sc.obs[t])
        assert did == bool(o.step(sc.control, sc.obs[t])), f"step {t}: gate"
        if did:
            resamples += 1
            assert np.array_equal(g.last_indices(), o.last_indices()), f"step {t}: indices"
        assert g.get_best_particle()[0] == o.best()
    _compare(g, o, "end")
    assert resamples > 0
    assert g.stats().serial_fallbacks == 0


def test_bigmap_limit():
    """65 536 landmarks is the limit; one more is refused (PFGPU_ERR_UNSUPPORTED) by every create call"""
    L = rr.load_library()
    for make in (lambda: rr.FastSlam1(64, 65537), lambda: rr.FastSlam2(64, 65537),
                 lambda: rr.FastSlam1.create_sharded_local(128, 65537, [0, 0])):
        with pytest.raises(rr.InvalidParameter):
            make()
        assert "65536 landmarks" in L.pfgpu_last_error().decode()
    g = rr.FastSlam1(64, 65536)
    assert g.m == 65536


@pytest.mark.parametrize("variant", [1, 2])
@pytest.mark.parametrize("world,n", [(2, 1024), (4, 4096)])
def test_bigmap_sharded_in_process_bit_exact(oracle, variant, world, n):
    """4 096 landmarks sharded over in-process ranks on one GPU: every rank's shard equals the oracle's slice"""
    steps = 16
    sc = _mid_circle(64, steps)
    cls = rr.FastSlam1 if variant == 1 else rr.FastSlam2
    ranks = cls.create_sharded_local(n, sc.m, [0] * world, rr.FsConfig(nth=n / 1.5), seed=9)
    o = OracleFS(oracle, n, sc.m, seed=9, variant=variant, nth=n / 1.5)
    for g in ranks:
        g.seed_map(sc.start, sc.landmarks)
    o.seed_map(sc.start, sc.landmarks)
    resamples = 0
    for t in range(steps):
        did = cls.step_all(ranks, sc.control, sc.obs[t])
        assert did == bool(o.step(sc.control, sc.obs[t])), f"step {t}: gate"
        if did:
            resamples += 1
            assert np.array_equal(np.concatenate([g.last_indices() for g in ranks]), o.last_indices()), f"step {t}: indices"
        for g in ranks:
            assert g.get_best_particle()[0] == o.best(), f"step {t}: best particle"
        if t % 6 == 0:
            _shard_compare(ranks, o, f"step {t}")
    _shard_compare(ranks, o, "end")
    assert resamples > 1
    assert all(g.stats().serial_fallbacks == 0 for g in ranks)


def test_bigmap_get_observations_on_device(oracle):
    """get_observations at 16 384 landmarks: the ids of scenarios.get_observations in the same order, and the oracle's tuples"""
    lms = scenarios.grid_landmarks(128)
    g = rr.FastSlam1(64, lms.shape[0], seed=42)
    o = OracleFS(oracle, 64, lms.shape[0], seed=42)
    rng = np.random.default_rng(4)
    poses = [[635.0, 595.0, 0.0], [0.0, 0.0, 1.0], [1270.0, 1270.0, -2.0], [403.7, 911.2, 0.3]] + \
            [[rng.uniform(-10, 1280), rng.uniform(-10, 1280), rng.uniform(-math.pi, math.pi)] for _ in range(6)]
    seen = 0
    for call, xt in enumerate(poses):
        z = g.get_observations(xt, lms, call)
        want = scenarios.get_observations(xt, lms, np.random.default_rng(0))
        assert [t[2] for t in z] == [t[2] for t in want], f"pose {xt}"
        assert z == o.observations(xt, lms, 42, call)
        seen += len(z)
    assert seen > 40
