"""The in-process NCCL stand-in (tests/c/nccl_loopback.cpp) without a GPU: built with -DLOOPBACK_HOST_ONLY, where device copies are
memcpy and stream syncs do nothing, and driven from C++ threads by tests/c/nccl_loopback_check.cpp.  Pins the rendezvous, the
reductions, all-gather, grouped send / receive, the timeout and its text, the mismatch checks and the counters that
tests/test_gpu_comm_loopback.py relies on."""
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
C_DIR = os.path.join(ROOT, "tests", "c")

CASES = ["allreduce_sum_int64", "allreduce_max_int32", "allreduce_other_ops_refused", "allgather_uint32", "grouped_send_recv",
         "empty_group_on_one_rank", "mismatched_operation", "mismatch_counted", "mismatched_count", "mismatched_type",
         "send_recv_byte_mismatch", "p2p_mismatch_counted", "timeout_names_the_missing_rank", "timeout_counted", "stats"]


def cuda_include():
    """nccl.h includes cuda_runtime.h: the CUDA toolkit's include directory"""
    for base in (os.environ.get("CUDA_HOME"), os.environ.get("CUDA_PATH"), "/usr/local/cuda"):
        if base and os.path.exists(os.path.join(base, "include", "cuda_runtime.h")):
            return os.path.join(base, "include")
    pytest.skip("no CUDA toolkit headers")


def build_loopback(out_dir, host_only):
    """-> directory holding libnccl.so.2, the stand-in"""
    os.makedirs(out_dir, exist_ok=True)
    cmd = ["g++", "-std=c++17", "-O2", "-Wall", "-Wextra", "-Werror", "-fPIC", "-shared", "-Wl,-soname,libnccl.so.2", "-I", cuda_include(),
           os.path.join(C_DIR, "nccl_loopback.cpp"), "-o", os.path.join(out_dir, "libnccl.so.2"), "-lpthread"]
    if host_only:
        cmd.insert(1, "-DLOOPBACK_HOST_ONLY")
    else:
        cmd += ["-L", os.path.join(os.path.dirname(cuda_include()), "lib64"), "-lcudart"]
    subprocess.check_call(cmd)
    return out_dir


@pytest.fixture(scope="module")
def check_output(tmp_path_factory):
    d = build_loopback(str(tmp_path_factory.mktemp("loopback")), host_only=True)
    exe = os.path.join(d, "check")
    subprocess.check_call(["g++", "-std=c++17", "-O2", "-Wall", "-Wextra", "-Werror", "-I", cuda_include(), os.path.join(C_DIR, "nccl_loopback_check.cpp"),
                           "-o", exe, "-L", d, "-l:libnccl.so.2", "-Wl,-rpath," + d, "-lpthread"])
    p = subprocess.run([exe], capture_output=True, text=True, timeout=120, env=dict(os.environ, LOOPBACK_NCCL_TIMEOUT="1"))
    lines = dict(ln.split(" ", 1) for ln in p.stdout.splitlines())
    return p, lines


@pytest.mark.parametrize("case", CASES)
def test_loopback_case(check_output, case):
    p, lines = check_output
    assert case in lines, p.stdout + p.stderr
    assert lines[case] == "ok", lines[case]


def test_every_case_ran(check_output):
    p, lines = check_output
    assert sorted(lines) == sorted(CASES) and p.returncode == 0, p.stdout + p.stderr


def test_exports_the_calls_the_library_resolves(tmp_path):
    """the stand-in defines every ncclX the library looks up with dlsym (comm.cu, nccl_api), and nothing stands in for a symbol it lacks"""
    import re
    d = build_loopback(str(tmp_path), host_only=True)
    src = open(os.path.join(ROOT, "elprep_b200", "csrc", "comm.cu")).read()
    wanted = set(re.findall(r'sym\("(nccl[A-Za-z]+)"\)', src))
    assert len(wanted) == 10, wanted
    nm = subprocess.run(["nm", "-D", "--defined-only", os.path.join(d, "libnccl.so.2")], capture_output=True, text=True, check=True).stdout
    have = {ln.split()[-1] for ln in nm.splitlines() if ln.strip()}
    assert wanted <= have, wanted - have
    assert "loopback_stats" in have
    soname = subprocess.run(["objdump", "-p", os.path.join(d, "libnccl.so.2")], capture_output=True, text=True, check=True).stdout
    assert re.search(r"SONAME\s+libnccl\.so\.2\b", soname)
