"""fsm_rcp / fsm_sqrt of include/fs_ekf_math.h on the GPU: the branch-free reciprocal and square root that the EKF fast
form runs must return the same bits as __drcp_rn / __dsqrt_rn (correctly rounded) on the window [2^-498, 2^498) where
the fast form uses them.  The probe (tests/host/fsm_probe.cu) is built by build() into build/libfsm_probe.so."""
import ctypes as C
import os

import pytest

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PROBE = os.path.join(ROOT, "build", "libfsm_probe.so")
CLASSES = ["random, every binade", "window ends", "powers of two / all-ones significands", "atan denominator", "2 pi sqrt(det)"]
LOG2_RANDOM = 28


def test_rcp_and_sqrt_equal_the_intrinsics():
    assert os.path.exists(PROBE), "build/libfsm_probe.so is missing: run __graft_entry__.build()"
    lib = C.CDLL(PROBE)
    lib.fsm_probe_run.argtypes = [C.c_int, C.c_uint, C.POINTER(C.c_ulonglong)]
    out = (C.c_ulonglong * (len(CLASSES) * 4))()
    err = lib.fsm_probe_run(0, LOG2_RANDOM, out)
    assert err == 0, f"CUDA error {err}"
    total = 0
    for c, name in enumerate(CLASSES):
        n, brcp, bsqrt, first = out[4 * c:4 * c + 4]
        assert n > 0, name
        assert brcp == 0 and bsqrt == 0, f"{name}: {brcp} reciprocal / {bsqrt} square-root mismatches of {n}, first operand bits {first:#018x}"
        total += n
    assert out[0] == 1 << LOG2_RANDOM
    assert total >= 1 << 28
