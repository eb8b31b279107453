"""The device finalize's Go math header (elprep_b200/csrc/gomath.hpp) built by g++, the way every host translation unit sees it, against the
oracle's restatement (oracle/gomath.c) bit for bit over a sweep of arguments: integer counts, every QUAL's error rate, the maxObs clamp,
random magnitudes from 1e-300 to 1e300, and Pow over reported qualities.  The header's device build (nvcc -fmad=false) is checked
against the oracle end to end by tests/test_gpu_finalize_device.py; this test catches a host/device split inside the header itself
(a bit cast, a classification or a constant that only one side gets right)."""
import os
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_header_matches_oracle(tmp_path):
    exe, obj = str(tmp_path / "gomath_check"), str(tmp_path / "gomath.o")
    subprocess.check_call(["gcc", "-O2", "-ffp-contract=off", "-c", os.path.join(ROOT, "oracle", "gomath.c"), "-o", obj])
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-Wall", "-Werror",
                           "-I", os.path.join(ROOT, "elprep_b200", "csrc"), "-I", os.path.join(ROOT, "oracle"),
                           os.path.join(ROOT, "tests", "c", "gomath_check.cpp"), obj, "-o", exe, "-lm"])
    out = subprocess.run([exe], capture_output=True, text=True)
    assert out.returncode == 0 and out.stdout.strip().endswith("OK"), out.stdout[-3000:]
