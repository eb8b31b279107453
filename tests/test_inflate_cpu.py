"""CPU check of the device DEFLATE decoder: tests/c/inflate_check.cpp compiles the kernel's own decoder (elprep_b200/csrc/inflate.cuh) as
host C++ with AddressSanitizer and UndefinedBehaviorSanitizer and compares it with zlib, stream by stream: zlib levels 0-9 and its
strategies, BAM-like records, random bytes, runs, period-k data, distances up to 32768, many blocks per member, ISIZE of 0 to 65536, bit
flips, truncations and hand-built invalid streams -- the same accept / reject decision, the same bytes on accept -- and the per-lane
CRC-32 fold of bgzf_crc against zlib's crc32."""
import os
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_device_decoder_matches_zlib(tmp_path):
    exe = str(tmp_path / "inflate_check")
    subprocess.check_call(["g++", "-O1", "-g", "-std=c++17", "-fsanitize=address,undefined", "-fno-sanitize-recover=all",
                           "-I", os.path.join(ROOT, "elprep_b200", "csrc"), "-o", exe, os.path.join(ROOT, "tests", "c", "inflate_check.cpp"), "-lz"])
    env = dict(os.environ, ASAN_OPTIONS="detect_leaks=0")
    out = subprocess.run([exe], capture_output=True, text=True, env=env)
    assert out.returncode == 0 and out.stdout.strip().endswith("OK"), (out.stdout[-2000:], out.stderr[-3000:])
