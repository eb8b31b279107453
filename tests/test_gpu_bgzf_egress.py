"""elp_fetch_bgzf / elp_debug_deflate: the output records written as BGZF blocks deflated on the device, against elp_fetch_bam, host zlib
(elp_bgzf_inflate, gzip), elp_bgzf_deflate's block cut, the host build of the encoder (tests/c/deflate_check.cpp) and a round trip through
elp_append_bgzf."""
import ctypes as C
import gzip
import os
import struct
import subprocess

import numpy as np
import pytest

from elprep_b200 import _lib, bgzf, device, synth
from test_sam_text import HEADER, line
from util import encode_bam, host_encoder, set_side_inputs  # noqa: F401 (host_encoder: a fixture)

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SMALL = [("chr20", 600_000), ("chr21", 300_000), ("chrM", 16_569)]
EOF_BLOCK = bytes([0x1f, 0x8b, 8, 4, 0, 0, 0, 0, 0, 0xff, 6, 0, 0x42, 0x43, 2, 0, 0x1b, 0, 3, 0, 0, 0, 0, 0, 0, 0, 0, 0])
SQ_TAGS = [b"XAZabc\0", b"NMi\x01\x00\x00\x00"]


def blocks(data):
    """-> [(bsize, isize)] of a BGZF byte string, checking every header; the EOF marker counts as a block"""
    out, x = [], 0
    while x < len(data):
        assert data[x:x + 4] == b"\x1f\x8b\x08\x04" and data[x + 10:x + 16] == b"\x06\x00BC\x02\x00"
        bsize = struct.unpack_from("<H", data, x + 16)[0] + 1
        isize = struct.unpack_from("<I", data, x + bsize - 4)[0]
        out.append((bsize, isize))
        x += bsize
    assert x == len(data)
    return out


def inflate_all(data):
    """the bytes of a BGZF file by two host inflaters, which must agree (gzip checks every CRC-32 and ISIZE)"""
    a = bgzf.inflate(data).tobytes() if len(data) else b""
    assert gzip.decompress(data) == a if len(data) else True
    return a


def header_bytes(w, text=b"@HD\tVN:1.6\tSO:coordinate\n"):
    return b"BAM\1" + struct.pack("<i", len(text)) + text + struct.pack("<i", len(w.header.SQ)) + b"".join(
        struct.pack("<i", len(sq["SN"]) + 1) + sq["SN"].encode() + b"\0" + struct.pack("<i", int(sq["LN"])) for sq in w.header.SQ)


@pytest.fixture(scope="module")
def wl():
    w = synth.make_workload(3_000, SMALL, seed=29)
    raw, off = encode_bam(w.batch, w.header, np.random.default_rng(29), extra_tags=[SQ_TAGS[i % 2] for i in range(w.batch.n)])
    return w, raw, off


def corpus(raw):
    rng = np.random.default_rng(17)
    r = raw.tobytes()
    return [b"", b"x", r[:0xff00], r[:0xff00 + 1], r[:3 * 0xff00 - 7], rng.integers(0, 256, 0xff00 * 2 + 5, dtype=np.uint8).tobytes(),
            b"A" * 200_000, bytes((np.arange(100_000) % 37).astype(np.uint8)), r,
            rng.integers(0, 4, 70_000, dtype=np.uint8).tobytes(), bytes(rng.integers(0, 256, 32768, dtype=np.uint8)) * 3]


def test_debug_deflate_corpus(wl, host_encoder, tmp_path):
    w, raw, _ = wl
    ctx = device.Context(w.header)
    for data in corpus(raw):
        for eof in (True, False):
            z = ctx.debug_deflate(data, eof=eof).tobytes()
            bl = blocks(z)
            if eof:
                assert bl[-1] == (28, 0) and z.endswith(EOF_BLOCK)
            else:
                assert (bl[-1][1] > 0) if data else z == b""
            body = bl[:-1] if eof else bl
            assert all(b <= 65536 for b, _ in bl)
            assert [i for _, i in body] == [min(0xff00, len(data) - k) for k in range(0, len(data), 0xff00)]
            host = bytes(bgzf.deflate(np.frombuffer(data, np.uint8), level=1, write_eof=eof)) if data else (EOF_BLOCK if eof else b"")
            assert [i for _, i in blocks(host)] == [i for _, i in bl]                     # the ISIZE sequence of elp_bgzf_deflate
            assert inflate_all(z) == data
            assert z == host_encoder(data, eof, str(tmp_path))                             # byte for byte the host build of deflate.cuh
    ctx.close()


def pipeline_ctx(w, raw, off, out_filter=None, target=None, profile=False):
    ctx = device.Context(w.header, profile=profile)
    set_side_inputs(ctx, w)
    if out_filter:
        ctx.set_output_filter(**out_filter)
    ctx.append_bam(raw, off)
    ctx.sort_markdup(device.SO_COORDINATE, True)
    if target is not None:
        for ci, iv in target.items():
            ctx.set_bqsr_target_regions(ci, np.asarray(iv, np.int32).reshape(-1, 2))
        assert ctx.filter_target_regions() > 0
    ctx.bqsr_gather(); ctx.bqsr_finalize(None); ctx.bqsr_apply()
    return ctx


SETTINGS = {
    "none": dict(),
    "remove_duplicates": dict(out_filter=dict(mask=_lib.OUT_REMOVE_DUPLICATES)),
    "remove_field": dict(out_filter=dict(remove=("XA",))),
    "keep_field": dict(out_filter=dict(keep=("RG", "NM"))),
    "target_regions": dict(target={0: [[1000, 200_000], [300_000, 450_000]], 1: [[0, 100_000]]}),
}


@pytest.mark.parametrize("setting", sorted(SETTINGS))
def test_fetch_bgzf_equals_fetch_bam(wl, setting):
    w, raw, off = wl
    ctx = pipeline_ctx(w, raw, off, **SETTINGS[setting])
    hdr = header_bytes(w)
    n = ctx.n_output()
    assert 0 < n
    whole_records = ctx.fetch_bam()[0].tobytes()
    whole = ctx.fetch_bgzf(prefix=hdr, eof=True).tobytes()
    assert whole.endswith(EOF_BLOCK) and inflate_all(whole) == hdr + whole_records
    for first, m in ((0, 1), (n - 1, 1), (n // 3, n // 2), (7, n - 7)):                 # sub-ranges
        z = ctx.fetch_bgzf(first, m, eof=False).tobytes()
        assert inflate_all(z) == ctx.fetch_bam(first, m)[0].tobytes()
    cuts = [0, 1, n // 5, n // 2, n // 2 + 1, n]                                           # chunked calls, EOF on the last only
    parts = [ctx.fetch_bgzf(a, b - a, prefix=hdr if a == 0 else b"", eof=(b == n)).tobytes() for a, b in zip(cuts[:-1], cuts[1:])]
    assert inflate_all(b"".join(parts)) == inflate_all(whole)
    assert ctx.fetch_bgzf(0, 0, prefix=hdr, eof=False).tobytes() != b""                 # n == 0: prefix only, EOF only, nothing
    assert inflate_all(ctx.fetch_bgzf(0, 0, prefix=hdr, eof=False).tobytes()) == hdr
    assert ctx.fetch_bgzf(0, 0, eof=True).tobytes() == EOF_BLOCK
    assert ctx.fetch_bgzf(n, 0, eof=False).tobytes() == b""
    ctx.close()


def test_round_trip_through_append_bgzf(wl):
    w, raw, off = wl
    ctx = pipeline_ctx(w, raw, off)
    f = ctx.fetch_bgzf(prefix=header_bytes(w)).tobytes()
    want_n, want = ctx.n_output(), ctx.fetch_bam()[0].tobytes()
    ctx.close()
    ctx = device.Context(w.header)
    set_side_inputs(ctx, w)
    for a in range(0, len(f), 100_003):
        ctx.append_bgzf(f[a:a + 100_003])
    ctx.append_bgzf_end()
    assert ctx.n == want_n
    ctx.sort_markdup(device.SO_KEEP, False)                                              # the file's order, FLAG and QUAL as written
    got = ctx.fetch_bam()[0].tobytes()
    ctx.close()
    assert got == want


def _raw_fetch_bgzf(ctx, first, n, prefix, capacity):
    out = np.full(max(capacity, 1), 0x5a, np.uint8)
    got = C.c_uint64(12345)
    p = np.frombuffer(prefix, np.uint8) if prefix else None
    rc = ctx.L.elp_fetch_bgzf(ctx.h, first, n, p.ctypes.data if p is not None else None, len(prefix), 1, out.ctypes.data, capacity, C.byref(got))
    return rc, bool((out == 0x5a).all()) and got.value == 12345


def test_refusals(wl):
    w, raw, off = wl
    ctx = device.Context(w.header)
    set_side_inputs(ctx, w)
    ctx.append_bam(raw, off)
    assert _raw_fetch_bgzf(ctx, 0, 5, b"", 1 << 20) == (_lib.ESTATE, True)              # before the sort
    ctx.sort_markdup(device.SO_COORDINATE, True)
    n = ctx.n_output()
    for first, m in ((0, n + 1), (n, 1), (n - 3, 4)):                                    # past elp_n_output
        assert _raw_fetch_bgzf(ctx, first, m, b"", 1 << 24) == (_lib.EINVAL, True)
    nb = int(ctx.L.elp_fetch_bam_bytes(ctx.h, 10, 100))
    hdr = header_bytes(w)
    need = int(ctx.L.elp_bgzf_deflate_bound(nb + len(hdr)))
    assert _raw_fetch_bgzf(ctx, 10, 100, hdr, need - 1) == (_lib.EINVAL, True)            # one byte short of the bound
    rc, _ = _raw_fetch_bgzf(ctx, 10, 100, hdr, need)
    assert rc == 0
    ctx.close()
    # reads from elp_append_batch
    ctx = device.Context(w.header)
    set_side_inputs(ctx, w)
    ctx.append(w.batch)
    ctx.sort_markdup(device.SO_COORDINATE, True)
    assert _raw_fetch_bgzf(ctx, 0, 5, b"", 1 << 20) == (_lib.ESTATE, True)
    ctx.close()
    # after elp_clean_sam rewrote a CIGAR (chr2 of this header has 1000 bases)
    ctx = device.Context(HEADER)
    ctx.append_sam(line(POS=b"998"))
    assert ctx.clean_sam() == 1
    ctx.sort_markdup(device.SO_KEEP, False)
    assert _raw_fetch_bgzf(ctx, 0, 1, b"", 1 << 20) == (_lib.ESTATE, True)
    ctx.close()


def test_size_and_scale():
    """1 M reads of the bench workload (several scratch rounds): inflates to the records, no larger than zlib level 1, the same bytes twice"""
    w = synth.make_workload(500_000, synth.scaled_hg38(64.0), seed=20260924, want_reference=False)
    raw, off = synth.encode_bam(w.batch, w.header)
    ctx = device.Context(w.header, profile=True)
    ctx.append_bam(raw, off)
    ctx.sort_markdup(device.SO_COORDINATE, True)
    hdr = header_bytes(w)
    a = ctx.fetch_bgzf(prefix=hdr).tobytes()
    recs = ctx.fetch_bam()[0]
    st = ctx.kernel_stats()
    b = ctx.fetch_bgzf(prefix=hdr).tobytes()
    ctx.close()
    assert a == b
    data = np.concatenate([np.frombuffer(hdr, np.uint8), recs])
    assert data.size > 600 * 0xff00
    assert bgzf.inflate(a).tobytes() == data.tobytes()
    z1 = bytes(bgzf.deflate(data, level=1))
    print(f"{data.size} bytes: device {len(a)} ({data.size / len(a):.3f}), zlib level 1 {len(z1)} ({data.size / len(z1):.3f}); "
          f"bgzf_deflate {st['bgzf_deflate']['ms']:.1f} ms")
    assert len(a) <= len(z1)
    assert st["bgzf_deflate"]["launches"] >= 2 and st["bgzf_deflate_crc"]["alg_bytes"] == data.size


CPP_CLIENT = r"""
#include "elprep_b200.hpp"
#include <fstream>
#include <iterator>
#include <sstream>
// argv: header spec (lines "SQ name length" / "RG id lb pu", "-" for none), BGZF input, BAM header bytes, output file
static std::vector<uint8_t> slurp(const char* p) { std::ifstream s(p, std::ios::binary); return std::vector<uint8_t>(std::istreambuf_iterator<char>(s), {}); }
int main(int argc, char** argv) {
    if (argc != 5) return 2;
    elprep::Header h;
    std::ifstream spec(argv[1]);
    for (std::string kind; spec >> kind;) {
        if (kind == "SQ") { elprep::Header::SQ q; spec >> q.SN >> q.LN; h.sq.push_back(q); }
        else { elprep::Header::ReadGroup g; spec >> g.ID >> g.LB >> g.PU; g.hasLB = g.LB != "-"; g.hasPU = g.PU != "-"; h.rg.push_back(g); }
    }
    elprep::Options o; o.MarkDuplicates = true;
    elprep::DeviceSam d(h, o);
    const auto in = slurp(argv[2]), hdr = slurp(argv[3]);
    d.AppendBgzf(in.data(), in.size());
    d.AppendBgzfEnd();
    d.Finalize(elprep::SortingOrder::Coordinate);
    const auto out = d.FetchBgzf(0, elp_n_output(d.Context()), hdr, true);
    std::ofstream(argv[4], std::ios::binary).write(reinterpret_cast<const char*>(out.data()), (std::streamsize)out.size());
    return 0;
}
"""


def test_cpp_fetch_bgzf_matches_python(wl, tmp_path):
    """DeviceSam::FetchBgzf, through a small client compiled here, returns the bytes of the Python binding"""
    w, raw, _ = wl
    src, exe = tmp_path / "client.cpp", str(tmp_path / "client")
    src.write_text(CPP_CLIENT)
    libdir = os.path.join(ROOT, "elprep_b200", "lib")
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"), str(src), "-o", exe,
                           "-L", libdir, "-lelprep_b200", "-Wl,-rpath," + libdir])
    hdr = header_bytes(w)
    f = bytes(bgzf.deflate(np.concatenate([np.frombuffer(hdr, np.uint8), raw]), level=6))
    (tmp_path / "spec.txt").write_text("".join(f"SQ {q['SN']} {q['LN']}\n" for q in w.header.SQ) +
                                       "".join(f"RG {r['ID']} {r.get('LB') or '-'} {r.get('PU') or '-'}\n" for r in w.header.RG))
    (tmp_path / "in.bgzf").write_bytes(f)
    (tmp_path / "hdr.bin").write_bytes(hdr)
    subprocess.check_call([exe, str(tmp_path / "spec.txt"), str(tmp_path / "in.bgzf"), str(tmp_path / "hdr.bin"), str(tmp_path / "out.bgzf")])
    ctx = device.Context(w.header)
    ctx.append_bgzf(f)
    ctx.append_bgzf_end()
    ctx.sort_markdup(device.SO_COORDINATE, True)
    want = ctx.fetch_bgzf(prefix=hdr).tobytes()
    ctx.close()
    assert (tmp_path / "out.bgzf").read_bytes() == want
