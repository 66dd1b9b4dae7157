"""The post kernel's instantiation for one value and at most one local slot per thread (fs3_post_kernel<512, false, 1>, config
3's shape) against the generic one (PFGPU_POST_K1=0), bit for bit: two engines on the same seed and inputs, stepped side by
side, agree on poses, weights, ancestors, maps (read through the lazy-clone rows), best particle, N_eff and gate after every
step.  Each case also checks which kernel each engine ran."""
import numpy as np
import pytest

import rust_robotics_b200 as rr
from rust_robotics_b200 import scenarios
import _weight_cases as wc

pytestmark = pytest.mark.gpu

SEED = 23


def _pair(monkeypatch, make, env=None):
    for k, v in (env or {}).items():
        monkeypatch.setenv(k, v)
    out = []
    for k1 in ("1", "0"):
        monkeypatch.setenv("PFGPU_POST_K1", k1)             # read when an engine is created
        out.append(make())
    a, b = out
    assert a.post_k1(), "the one-value kernel did not run"
    assert not b.post_k1()
    assert a.post_shape() == b.post_shape()
    return a, b


def same(x, y):
    """bitwise equality that also holds NaN positions and the sign of zero"""
    x, y = np.asarray(x), np.asarray(y)
    nx, ny = np.isnan(x), np.isnan(y)
    return (x.shape == y.shape and np.array_equal(nx, ny) and np.array_equal(x[~nx], y[~ny])
            and np.array_equal(np.signbit(x[~nx]), np.signbit(y[~ny])))


def _compare(a, b, t, did_a, did_b, best=True):
    assert did_a == did_b, f"step {t}: gate"
    assert a.last_gate() == b.last_gate(), f"step {t}: gate"
    assert same(a.last_neff(), b.last_neff()), f"step {t}: N_eff"
    if did_a:
        assert np.array_equal(a.last_indices(), b.last_indices()), f"step {t}: ancestors"
    pa, la = a.state()
    pb, lb = b.state()
    assert same(pa, pb), f"step {t}: poses / weights"
    assert same(la, lb), f"step {t}: maps"
    if best:
        ba, bb = a.get_best_particle(), b.get_best_particle()
        assert ba[0] == bb[0] and same(ba[1:], bb[1:]), f"step {t}: best particle"


def _trajectory(monkeypatch, n, steps, nth, variant=1, env=None, sc=None):
    sc = sc or scenarios.FastSlamScenario(16, (75.0, 35.0, 0.0), (1.0, 0.025), steps)      # C3's map and circle
    cls = rr.FastSlam1 if variant == 1 else rr.FastSlam2
    a, b = _pair(monkeypatch, lambda: cls(n, sc.m, rr.FsConfig(nth=nth), seed=SEED), env)
    for g in (a, b):
        g.seed_map(sc.start, sc.landmarks)
    resamples = 0
    for t in range(steps):
        step = (lambda g: g.fastslam_update(sc.control, sc.obs[t])) if variant == 1 else (lambda g: g.fastslam2_update(sc.control, sc.obs[t]))
        da, db = step(a), step(b)
        _compare(a, b, t, da, db)
        resamples += int(da)
    return a, b, resamples


@pytest.mark.parametrize("nth", ["default", "every", "literal"])
def test_k1_config3_trajectory(monkeypatch, nth):
    n = 1 << 16
    a, b, resamples = _trajectory(monkeypatch, n, 12, {"default": n / 1.5, "every": n + 1.0, "literal": 100.0 / 1.5}[nth])
    assert a.post_shape() == (128, 512, 1, "shared")
    assert (resamples == 0) == (nth == "literal")


def test_k1_exact_cdf(monkeypatch):
    n = 1 << 16
    _, _, resamples = _trajectory(monkeypatch, n, 8, n + 1.0, env={"PFGPU_FS_EXACT_CDF": "1"})
    assert resamples == 8


def test_k1_fastslam2(monkeypatch):
    n = 1 << 16
    _, _, resamples = _trajectory(monkeypatch, n, 10, n / 1.5, variant=2)
    assert resamples > 0


def test_k1_odd_count_512_threads(monkeypatch):
    """below 2^16 the default shape is 256 threads: PFGPU_POST_NT=512 gives 47 tiles x 512, the last one partly filled"""
    n = 24001
    a, _, resamples = _trajectory(monkeypatch, n, 12, n / 1.5, env={"PFGPU_POST_NT": "512"})
    assert a.post_shape() == (47, 512, 1, "shared")
    assert resamples > 0


def test_k1_many_live_rows(monkeypatch):
    """a straight drive at 2 m per step across C3's map, resampling every step: the landmarks left behind keep their rows
    step after step, so the later resamples compose many more live rows than one batch of the clone phase holds (8192
    particles on 16 tiles x 512 threads)"""
    n, steps = 8192, 48
    sc = scenarios.FastSlamScenario(16, (5.0, 75.0, 0.0), (20.0, 0.0), steps)
    a, _, resamples = _trajectory(monkeypatch, n, steps, n + 1.0, env={"PFGPU_POST_NT": "512"}, sc=sc)
    assert a.post_shape() == (16, 512, 1, "shared")
    assert resamples == steps


@pytest.mark.parametrize("case", [c for c in wc.CASES if c.name != "serial_walk"], ids=lambda c: c.name)
def test_k1_weight_cases(oracle, monkeypatch, case):
    """the adversarial raw weights of _weight_cases.py at 2^16 (but the one-thread serial walk), handed to the post kernel
    untouched (no observations, u = 0, no motion noise), two steps"""
    n, m = 1 << 16, 4
    w = case.build(n, SEED, 0, L=oracle, family="fs")
    nth = case.nth(n, w)
    a, b = _pair(monkeypatch, lambda: rr.FastSlam1(n, m, rr.FsConfig(q00=0.0, q11=0.0, nth=nth), seed=SEED))
    p = np.empty((n, 4))
    p[:, 0] = w
    p[:, 1] = np.arange(n) * 0.5 + 1.0
    p[:, 2] = -np.arange(n) * 0.25 - 1.0
    p[:, 3] = np.linspace(-3.0, 3.0, n)
    lm = np.zeros((n, m, 6))
    lm[:, :, 0] = np.arange(n)[:, None] + 1.0
    lm[:, :, 1] = np.arange(m)[None, :] + 2.0
    lm[:, :, 2] = lm[:, :, 5] = 1000.0
    for g in (a, b):
        g.set_state(p, lm)
    for t in range(2):
        da, db = a.fastslam_update([0.0, 0.0], []), b.fastslam_update([0.0, 0.0], [])
        _compare(a, b, t, da, db, best=case.name not in wc.NO_BEST)
