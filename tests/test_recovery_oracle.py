"""CPU tests of augmented MCL (DESIGN §3.8) on the oracle (tests/host/pf_recovery_oracle.c):
  - the glibc build reproduces tests/golden/recovery_golden.json (the Python restatement) bit for bit: particles, resample
    indices, w_slow / w_fast / p and the injected count of every step, with injected draws;
  - behaviour, with Philox draws: config 2's world at 2^14 particles with a kidnap (KidnapScenario: 30 steps of tracking, then the
    robot is carried 15 m and turned 0.5 rad, seed 7; filter seed 3; alpha_slow 0.01, alpha_fast 0.2, region = the 50 m box inside
    the landmark circle).  Without recovery the error stays above 5 m for the 60 steps after the kidnap; with it, it falls below
    1 m within them.  Global localisation from init_region gets within 1 m in its first steps (range beams do not observe the
    yaw, so a cloud that found the position can still hold wrong headings, which only driving resolves)."""
import json
import os

import numpy as np
import pytest

import _recovery_oracle as R
from rust_robotics_b200 import scenarios

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "recovery_golden.json")
ALPHAS = (0.01, 0.2)


def fx(v):
    if isinstance(v, list):
        return np.array([fx(a) for a in v])
    return float.fromhex(v)


def _cases():
    with open(GOLDEN) as f:
        return json.load(f)["cases"]


@pytest.mark.parametrize("case", _cases(), ids=lambda c: c["name"])
def test_oracle_reproduces_golden(case):
    o = R.OracleRecovery(case["n"], threshold=fx(case["threshold"]), range_noise=fx(case["sigma"]), velocity_noise=fx(case["sv"]),
                         yaw_rate_noise=fx(case["sw"]), dt=fx(case["dt"]), mode=case["mode"], max_particles=case["nmax"],
                         kld_epsilon=fx(case["eps"]), kld_z=fx(case["z"]), libm=True, fast_search=False)
    region = fx(case["region"])
    assert o.enable(fx(case["a_slow"]), fx(case["a_fast"]), region) == 0
    if "init_region_u3" in case:
        assert o.init_region(region, fx(case["init_region_u3"])) == 0
        assert np.array_equal(o.particles(), fx(case["init"]))
    else:
        o.upload(fx(case["init"]))
    for t, s in enumerate(case["steps"]):
        inj4 = fx(s["inj4"]) if s["inj4"] else np.zeros((len(s["zv"]), 4))      # (no draws: the predict is not armed)
        assert o.predict(fx(s["u"]), fx(s["zv"]), fx(s["zw"]), inj4) == 0
        assert o.state()[1] == s["injected"], f"step {t}"
        assert o.update(fx(s["obs"]).reshape(-1, 3)) == 0
        did = o.resample(fx(s["r"]))
        assert did == s["did_resample"], f"step {t}"
        w, _ = o.state()
        assert np.array_equal(w, [fx(s["w_slow"]), fx(s["w_fast"]), fx(s["p"])]), f"step {t}"
        if did:
            assert np.array_equal(o.last_indices(), np.array(s["indices"], dtype=np.uint32)), f"step {t}"
        assert o.count() == s["count"] and np.array_equal(o.estimate(), fx(s["est"])), f"step {t}"
    assert np.array_equal(o.particles(), fx(case["particles"]))


def test_golden_exercises_the_semantics():
    cases = {c["name"]: c for c in _cases()}
    pf = cases["pf_gate_some_steps_kidnap"]["steps"]
    assert any(not s["did_resample"] for s in pf) and any(s["did_resample"] for s in pf)
    for a, b in zip(pf, pf[1:]):                       # a closed gate never causes an injection in the next predict
        if not a["did_resample"]:
            assert b["injected"] == 0
    s0 = cases["mcl_kidnap_s_zero"]["steps"]
    assert any(fx(s["S"]) == 0.0 for s in s0) and any(s["injected"] for s in s0)
    kld = cases["mcl_kld_from_region"]["steps"]
    assert len({s["count"] for s in kld}) > 1


def test_validation_and_reset():
    o = R.OracleRecovery(32, mode=1, max_particles=32)
    box = [-1.0, 1.0, -1.0, 1.0]
    for a_s, a_f, reg in ((0.2, 0.1, box), (0.1, 0.1, box), (0.0, 0.1, box), (0.1, 1.5, box), (np.nan, 0.2, box), (0.1, 0.2, None),
                          (0.1, 0.2, [1.0, 1.0, 0.0, 1.0]), (0.1, 0.2, [0.0, 1.0, 2.0, 1.0]), (0.1, 0.2, [0.0, np.inf, 0.0, 1.0])):
        assert o.enable(a_s, a_f, reg) == -1
    assert o.enable(0.0, 0.0, None) == 0
    assert o.enable(0.1, 1.0, box) == 0
    assert o.init_region([0.0, 0.0, 0.0, 1.0]) == -1
    o.init_state([0.0, 0.0, 0.0, 0.0])
    o.update([[50.0, 0.0, 0.0]])                        # S = 0: the filter still runs
    w, _ = o.state()
    assert w[0] == 0.0 and w[1] == 0.0 and w[2] == 0.0


def _errors(sc, on, seed, init):
    n = 1 << 14
    o = R.OracleRecovery(n, mode=1, max_particles=n, range_noise=0.25, velocity_noise=0.05, yaw_rate_noise=0.02, seed=seed,
                         threads=min(8, os.cpu_count() or 1))
    if on:
        o.enable(*ALPHAS, sc.REGION)
    init(o)
    return [sc.error(k, o.step(sc.controls[k], sc.obs[k])[0]) for k in range(len(sc.controls))]


def test_kidnap_recovery_behaviour():
    sc = scenarios.KidnapScenario()
    for on in (False, True):
        err = _errors(sc, on, 3, lambda o: o.init_state(sc.init))
        assert max(err[:sc.before]) < 0.5                  # tracking before the kidnap, with or without recovery
        if on:
            assert min(err[sc.before:]) < 1.0 and err[-1] < 1.0
        else:
            assert min(err[sc.before:]) > 5.0              # plain MCL never recovers


def test_global_localisation_from_region():
    sc = scenarios.KidnapScenario(before=0, after=30)
    err = _errors(sc, True, 5, lambda o: o.init_region(sc.REGION))
    assert min(err[:5]) < 1.0                              # the first update finds the particles near the truth
