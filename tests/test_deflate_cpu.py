"""CPU check of the device DEFLATE encoder: tests/c/deflate_check.cpp compiles the kernel's own encoder (elprep_b200/csrc/deflate.cuh) as host
C++ with AddressSanitizer and UndefinedBehaviorSanitizer.  Every stream of its corpus (empty, 1 and 0xff00 bytes, BAM-like records, random
bytes, runs, period-k data, distances of exactly 32768, literal-only input, a single literal value, Fibonacci histograms) must inflate back
with zlib and with inflate.cuh, every emitted Huffman code must be complete, and random bytes must take the stored path.  On synthetic BAM
records the encoder must be no larger than zlib level 1 on the same 0xff00-byte blocks."""
import os
import subprocess
import zlib

import numpy as np
import pytest

from elprep_b200 import synth

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ENV = dict(os.environ, ASAN_OPTIONS="detect_leaks=0")


@pytest.fixture(scope="module")
def exe(tmp_path_factory):
    exe = str(tmp_path_factory.mktemp("deflate") / "deflate_check")
    subprocess.check_call(["g++", "-O1", "-g", "-std=c++17", "-fsanitize=address,undefined", "-fno-sanitize-recover=all",
                           "-I", os.path.join(ROOT, "elprep_b200", "csrc"), "-o", exe, os.path.join(ROOT, "tests", "c", "deflate_check.cpp"), "-lz"])
    return exe


def test_device_encoder_round_trips(exe):
    out = subprocess.run([exe], capture_output=True, text=True, env=ENV)
    assert out.returncode == 0 and out.stdout.strip().endswith("OK"), (out.stdout[-2000:], out.stderr[-3000:])


def zlib_size(data, level):
    total = 0
    for off in range(0, len(data), 0xff00):
        co = zlib.compressobj(level, zlib.DEFLATED, -15)
        total += len(co.compress(data[off:off + 0xff00]) + co.flush())
    return total


def test_encoder_ratio_on_bam_records(exe, tmp_path):
    w = synth.make_workload(20_000, [("chr20", 2_000_000), ("chr21", 1_000_000), ("chrM", 16_569)], seed=20260924)
    raw, _ = synth.encode_bam(w.batch, w.header)
    data = np.ascontiguousarray(raw, dtype=np.uint8).tobytes()
    path = tmp_path / "records.bin"
    path.write_bytes(data)
    out = subprocess.run([exe, "size", str(path)], capture_output=True, text=True, env=ENV)
    assert out.returncode == 0, (out.stdout[-2000:], out.stderr[-3000:])
    ours = int(out.stdout.split()[-1])
    z1, z6 = zlib_size(data, 1), zlib_size(data, 6)
    print(f"{len(data)} bytes of records: encoder {ours} ({len(data) / ours:.3f}), zlib level 1 {z1} ({len(data) / z1:.3f}), "
          f"level 6 {z6} ({len(data) / z6:.3f})")
    assert ours <= z1
