"""CPU check of the team code of the device DEFLATE decoder and encoder: tests/c/team_check.cpp compiles inflate.cuh and deflate.cuh for host
teams of K lanes, one std::thread each (barriers for the syncs, atomic_ref for the atomics, a chain team of min(K, 32) lanes with its own
barrier), and compares every call with the team of one lane that test_inflate_cpu.py and test_deflate_cpu.py compare with zlib: every lane
returns the same status or length, and the bytes are the team of one's.  Built once with -O2 over the corpora, and once with
-fsanitize=thread over a subset, where any data race stops the run.  A lane that returns early leaves the others waiting at a barrier, so
a run that does not finish in time fails."""
import os
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def build(tmp_path, name, flags):
    exe = str(tmp_path / name)
    subprocess.check_call(["g++", *flags, "-std=c++20", "-pthread", "-I", os.path.join(ROOT, "elprep_b200", "csrc"), "-o", exe,
                           os.path.join(ROOT, "tests", "c", "team_check.cpp"), "-lz"])
    return exe


def run(exe, mode, timeout, env=None):
    try:
        out = subprocess.run([exe, mode], capture_output=True, text=True, timeout=timeout, env=env)
    except subprocess.TimeoutExpired as e:
        raise AssertionError(f"team_check {mode} did not finish in {timeout} s (a lane left the others at a barrier?)\n{e.stdout or ''}")
    print(out.stdout)
    assert out.returncode == 0 and out.stdout.strip().endswith("OK"), (out.stdout[-3000:], out.stderr[-5000:])


def test_teams_match_the_team_of_one(tmp_path):
    run(build(tmp_path, "team_check", ["-O2"]), "full", timeout=600)


def test_teams_do_not_race(tmp_path):
    exe = build(tmp_path, "team_check_tsan", ["-O1", "-g", "-fsanitize=thread"])
    run(exe, "tsan", timeout=600, env=dict(os.environ, TSAN_OPTIONS="halt_on_error=1"))
