"""The landmark existence counters of the unknown-association oracle (tests/host/fs2_exist_oracle.c, DESIGN §3.7) against their
golden vectors (tests/golden/make_existence_golden.py), and the long-run behaviour they exist for, on the CPU."""
import json
import os

import numpy as np
import pytest

import _existence as E
from _exist_oracle import OracleFS2Exist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def unhex(v):
    if isinstance(v, list):
        return [unhex(a) for a in v]
    return float.fromhex(v) if isinstance(v, str) else v


def cases():
    with open(os.path.join(ROOT, "tests", "golden", "fs2_existence_golden.json")) as f:
        return json.load(f)["cases"]


def run_case(case, libm):
    n, m = case["n"], case["m"]
    cfg = {k: unhex(v) for k, v in case["cfg"].items()}
    o = OracleFS2Exist(n, m, libm=libm, **cfg)
    o.set_state(unhex(case["init_pose"]), unhex(case["init_lm"]))
    o.enable_existence(unhex(case["range"]))
    gate = unhex(case["gate"])
    for t, st in enumerate(case["steps"]):
        z1 = np.concatenate([unhex(st["z1"]), unhex(st["z2"])])
        did = o.step_unknown(unhex(st["u"]), unhex(st["obs"]), gate, unhex(st["z0"]), z1, unhex(st["u01"]))
        where = f"{case['name']} step {t}"
        assert did == st["did_resample"], where
        assert o.counts.tolist() == st["counts"] and o.removed == st["removed"], where
        if did:
            assert o.last_indices().tolist() == st["indices"], where
        assert o.existence_counts().tolist() == st["tau"], where
        p, l = o.state()
        wp, wl = np.array(unhex(st["pose"])), np.array(unhex(st["lm"]))
        if libm:
            assert o.last_neff() == unhex(st["neff"]), where
            assert np.array_equal(p, wp, equal_nan=True), where
            assert np.array_equal(l, wl, equal_nan=True), where
        else:                                                          # test_fs2_assoc_oracle.py's tolerances
            np.testing.assert_allclose(p, wp, rtol=1e-8, atol=1e-11, err_msg=where)
            np.testing.assert_allclose(l, wl, rtol=1e-7, atol=1e-10, err_msg=where)


@pytest.mark.parametrize("idx", range(5))
def test_existence_oracle_libm_bit_exact_vs_python(idx):
    run_case(cases()[idx], libm=True)


@pytest.mark.parametrize("idx", range(5))
def test_existence_oracle_contract_vs_python(idx):
    run_case(cases()[idx], libm=False)


def test_golden_cases_exercise_every_rule():
    cs = {c["name"]: c for c in cases()}
    assert sum(s["removed"] for c in cs.values() for s in c["steps"]) > 0
    assert any(s["did_resample"] for c in cs.values() for s in c["steps"])
    assert any(not s["obs"] for c in cs.values() for s in c["steps"])                       # k = 0 steps
    assert any(max(max(r) for r in s["tau"]) >= 3 for s in cs["seeded_map_dup_k0"]["steps"])
    # the range edge: d == r is decremented (1 -> 0 -> removed), one ulp beyond is not
    edge = [s["tau"][0] for s in cs["range_edge_k0"]["steps"]]
    assert edge == [[0, 1, 0, 0], [0, 1, 0, 0], [0, 1, 0, 0]]
    assert cs["range_edge_k0"]["steps"][1]["removed"] == 8
    # a birth into a slot an earlier step freed
    st = cs["full_map_drops_then_births"]["steps"]
    assert st[1]["removed"] > 0 and st[1]["counts"][2] > 0 and st[2]["counts"][1] > 0


def _oracle_run(r):
    sc = E.scenario()
    o = OracleFS2Exist(E.N, E.M, seed=E.SEED, nth=E.N / 1.5)
    o.L.orc_fs_set_threads(o.h, max(1, min(32, os.cpu_count() or 1)))
    o.set_state(np.tile([1.0 / E.N, *sc.start], (E.N, 1)), np.tile([0.0, 0.0, 1000.0, 0.0, 0.0, 1000.0], (E.N, E.M, 1)))
    o.enable_existence(r)

    def step(u, z):
        o.step_unknown(u, z)
        return int(o.counts[2]), o.removed
    return E.run(step, lambda: o.state()[1][o.best()], sc)


def test_long_run_maps_stop_filling():
    """1 000 steps on the config-3 grid from a fresh map of 64 slots: without counters the maps fill up (every slot of the best
    particle initialised although fewer landmarks have been seen) and observations are dropped; with them, none is dropped and the
    best particle keeps about one slot per landmark seen"""
    on, off = _oracle_run(E.RANGE), _oracle_run(0)
    E.check(on, off)
    assert on[-1, 0] == 49 and on[-1, 1] == 55 and on[:, 3].sum() == 16014   # the numbers of DESIGN §3.7
    assert off[-1, 2] == 1820
