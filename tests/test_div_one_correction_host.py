"""The fast form's one-correction quotient (fsm_div, include/fs_ekf_math.h) equals IEEE a / b on the division window: the
finite region DESIGN §3.1 leaves to enumeration (both significands next to 2) exhaustively, plus significands near all-ones,
quotients at binade edges and next to rounding midpoints, operands at the window's ends and random pairs
(tests/host/divtest_one.c, on the CPU)."""
import os
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "host", "divtest_one.c")


def test_one_correction_quotient_is_ieee(tmp_path):
    exe = str(tmp_path / "divtest_one")
    subprocess.run(["/usr/bin/gcc", "-O2", "-ffp-contract=off", "-o", exe, SRC, "-lm"], check=True)
    r = subprocess.run([exe, "20000000"], capture_output=True, text=True)
    assert r.returncode == 0 and "mismatches=0" in r.stdout, r.stdout + r.stderr
