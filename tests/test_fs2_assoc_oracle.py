"""The unknown-association oracle (tests/host/fs2_assoc_oracle.c) against its golden vectors (tests/golden/make_assoc_golden.py),
and the association metric the CUDA kernel evaluates (fs_assoc_d2, include/fs2_math.h) against the oracle's, on the CPU."""
import ctypes as C
import json
import math
import os
import subprocess

import numpy as np
import pytest

from _assoc_oracle import OracleFS2Assoc

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
dp = C.POINTER(C.c_double)


def unhex(v):
    if isinstance(v, list):
        return [unhex(a) for a in v]
    return float.fromhex(v) if isinstance(v, str) else v


def cases():
    with open(os.path.join(ROOT, "tests", "golden", "fs2_assoc_golden.json")) as f:
        return json.load(f)["cases"]


def run_case(case, libm):
    n, m = case["n"], case["m"]
    cfg = {k: unhex(v) for k, v in case["cfg"].items()}
    o = OracleFS2Assoc(n, m, libm=libm, **cfg)
    o.set_state(unhex(case["init_pose"]), unhex(case["init_lm"]))
    gate = unhex(case["gate"])
    for t, st in enumerate(case["steps"]):
        if st["zero_weights"]:
            p, l = o.state()
            p[:, 0] = 0.0
            o.set_state(p, l)
        z1 = np.concatenate([unhex(st["z1"]), unhex(st["z2"])])
        did = o.step_unknown(unhex(st["u"]), unhex(st["obs"]), gate, unhex(st["z0"]), z1, unhex(st["u01"]))
        where = f"{case['name']} step {t}"
        assert did == st["did_resample"], where
        assert o.counts.tolist() == st["counts"], where
        if did:
            assert o.last_indices().tolist() == st["indices"], where
        p, l = o.state()
        wp, wl = np.array(unhex(st["pose"])), np.array(unhex(st["lm"]))
        if libm:
            assert o.last_neff() == unhex(st["neff"]), where
            assert np.array_equal(p, wp, equal_nan=True), where
            assert np.array_equal(l, wl, equal_nan=True), where
        else:
            np.testing.assert_allclose(p, wp, rtol=1e-8, atol=1e-11, err_msg=where)
            np.testing.assert_allclose(l, wl, rtol=1e-7, atol=1e-10, err_msg=where)


@pytest.mark.parametrize("idx", range(5))
def test_assoc_oracle_libm_bit_exact_vs_python(idx):
    run_case(cases()[idx], libm=True)


@pytest.mark.parametrize("idx", range(5))
def test_assoc_oracle_contract_close_to_python(idx):
    run_case(cases()[idx], libm=False)


def test_golden_cases_exercise_every_outcome():
    tot = np.zeros(3, dtype=np.int64)
    for c in cases():
        for st in c["steps"]:
            tot += np.array(st["counts"])
    assert (tot > 0).all(), tot                                        # matches, births and drops all occur


@pytest.fixture(scope="module")
def probe():
    lib = os.path.join(ROOT, "tests", "host", "libfs_assoc_probe.so")
    subprocess.run(["/usr/bin/g++", "-O2", "-ffp-contract=off", "-fPIC", "-shared", "-o", lib,
                    os.path.join(ROOT, "tests", "host", "fs_assoc_probe.cpp"), "-lm"], check=True)
    L = C.CDLL(lib)
    L.fs_assoc_probe.argtypes = [dp, dp, C.c_double, C.c_double, C.c_double, C.c_double, dp]
    return L


def _p(a):
    return a.ctypes.data_as(dp)


def test_metric_equals_the_oracle(probe):
    rng = np.random.default_rng(91)
    o = OracleFS2Assoc(1, 1)
    skipped = nan = 0
    for t in range(4000):
        pose = np.array([rng.uniform(-30, 30), rng.uniform(-30, 30), rng.uniform(-math.pi, math.pi)])
        lm = np.array([pose[0] + rng.uniform(-20, 20), pose[1] + rng.uniform(-20, 20), 0, 0, 0, 0])
        a, b = 10 ** rng.uniform(-3, 1.5, 2)
        c = rng.uniform(-0.9, 0.9) * math.sqrt(a * b)
        lm[2:] = [a, c, c * rng.choice([1.0, 0.999]), b]
        z = np.array([rng.uniform(0.1, 25), rng.uniform(-4, 4)])
        r = (0.5, 0.0305)
        if t % 7 == 0:
            lm[:2] = pose[:2]                                          # d = 0: h is NaN, so is S
        if t % 11 == 0:
            lm[2] = math.nan                                           # NaN covariance
        if t % 13 == 0:
            lm[2:] = 0.0                                               # P = 0 and R = 0: det S = 0, the slot is skipped
            r = (0.0, 0.0)
        if t % 17 == 0:
            lm[:2] = pose[:2] + rng.uniform(-1e-6, 1e-6, 2)
        o.cfg.r00, o.cfg.r11 = r
        want = o.assoc_d2(lm, pose, z)
        got = np.zeros(1)
        ok = probe.fs_assoc_probe(_p(lm), _p(pose), float(z[0]), float(z[1]), r[0], r[1], _p(got))
        assert bool(ok) == (want is not None), (t, lm, pose, z)
        if want is None:
            skipped += 1
            continue
        if math.isnan(want):
            nan += 1
            assert math.isnan(got[0]), (t, got[0])
        else:
            assert got[0] == want, (t, lm, pose, z, got[0], want)
    assert skipped > 100 and nan > 100
