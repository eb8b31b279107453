"""elp_fetch_sam: the stored records of a context as SAM text lines in output order.  Each line must equal FormatAlignment of
parseBamAlignment of the record elp_fetch_bam returns (tests/samformat.py), and for SAM input FormatAlignment(parseSamAlignment(line)),
the reference's own SAM -> SAM text."""
import ctypes as C
import struct

import numpy as np
import pytest

from elprep_b200 import device, synth, _lib
from samformat import bam_to_sam, format_alignment, parse_sam_alignment, sam_to_sam
from samtext import format_sam, sam_line_to_bam, sam_lines_to_bam, sam_text
from test_gpu_sam_ingest import NEG_POS, _tag_mix, _workload
from test_sam_format import LINES, NAMES, bam_record
from test_sam_text import HEADER, KAT, line
from util import gpu_phases, oracle_pipeline, set_side_inputs

pytestmark = pytest.mark.gpu

LOST = {"rname_unknown"}                                                  # RNAME chrZ with RNEXT '=': the record cannot give the names back
OUT_KERNELS = ("sam_out_measure", "sam_out_emit")


def _join(records):
    raw = b"".join(records)
    off = np.zeros(len(records) + 1, np.uint64)
    np.cumsum([len(r) for r in records], out=off[1:])
    return np.frombuffer(raw, np.uint8).copy(), off


def _line_off(lines):
    off = np.zeros(len(lines) + 1, np.uint64)
    np.cumsum([len(x) for x in lines], out=off[1:])
    return off


def test_kat_lines_round_trip():
    """every accepted known-answer line of the SAM ingest: SAM in, SAM out equals the reference's SAM -> SAM text"""
    lines = [k[1] for k in KAT if k[0] not in NEG_POS | LOST]
    ctx = device.Context(HEADER, profile=True)
    ctx.append_sam(b"\n".join(lines) + b"\n")
    ctx.sort_markdup(device.SO_KEEP, False)
    text, off = ctx.fetch_sam()
    want = [sam_to_sam(x) for x in lines]
    assert text.tobytes() == b"".join(want)
    assert np.array_equal(off, _line_off(want))
    assert all(k in ctx.kernel_stats() for k in OUT_KERNELS + ("sam_out_float",))
    ctx.close()


def _big_records():
    """a 100 kb read with a 65 535-operation CIGAR, and a record with more than 64 KB of optional fields"""
    rng = np.random.default_rng(5)
    L = 100_000
    cig = tuple((1, (0, 1)[i & 1]) for i in range(65534)) + ((L - 32767 - 32767, 0),)
    seq = rng.integers(0, 256, (L + 1) // 2, dtype=np.uint8).tobytes()
    qual = rng.integers(0, 94, L, dtype=np.uint8).tobytes()
    long_read = bam_record(qname=b"long", cigar=cig, seq=seq, lseq=L, qual=qual, tags=b"MDZ" + b"12A" * 5000 + b"\0")
    fl = rng.integers(0, 1 << 32, 3000, dtype=np.uint64).astype(np.uint32)
    fl[(fl & 0x7F800000) == 0x7F800000] = 0x7F800000                  # (keep NaN payload variety small: one infinity instead)
    tags = (b"XZZ" + bytes(rng.integers(33, 127, 70_000, dtype=np.uint8)) + b"\0" + b"XCBc" + struct.pack("<I", 20_000) + rng.integers(0, 256, 20_000, dtype=np.uint8).tobytes()
            + b"XIBi" + struct.pack("<I", 5000) + rng.integers(-(1 << 31), 1 << 31, 5000, dtype=np.int64).astype("<i4").tobytes()
            + b"XFBf" + struct.pack("<I", fl.size) + fl.astype("<u4").tobytes() + b"XHH" + b"0123456789ABCDEF" * 300 + b"\0")
    return [long_read, bam_record(qname=b"t" * 254, tags=tags)]


def test_bam_records():
    """hand-built records through elp_append_bam: every row of the field table, float specials and denormals, 254-byte QNAMEs, a 100 kb
    read, a 65 535-op CIGAR, more than 64 KB of tags, refID / next_refID -1, equal and different"""
    recs = [r for name, r, _ in LINES if name not in ("fixed_bounds", "qual_ff")]   # the phases refuse a negative POS and QUAL above 93
    recs.append(bam_record(flag=65535, mapq=255, pos=0, pnext=0x7FFFFFFF, tlen=-2147483648))
    specials = (0x7F800000, 0xFF800000, 0x7FC00000, 0xFFFFFFFF, 0x00000001, 0x007FFFFF, 0x80000001, 0x00800000, 0x7F7FFFFF, 0x80000000)
    recs.append(bam_record(tags=b"".join(b"F%df" % i + struct.pack("<I", v) for i, v in enumerate(specials))))
    recs += _big_records()
    raw, off = _join(recs)
    ctx = device.Context(HEADER)
    ctx.append_bam(raw, off)
    ctx.sort_markdup(device.SO_KEEP, False)
    text, loff = ctx.fetch_sam()
    want = [bam_to_sam(r, NAMES) for r in recs]
    got = [text[int(loff[i]):int(loff[i + 1])].tobytes() for i in range(len(recs))]
    bad = [i for i in range(len(recs)) if got[i] != want[i]]
    assert not bad, [(i, got[i][:200], want[i][:200]) for i in bad[:3]]
    assert text.tobytes() == b"".join(want)
    ctx.close()


def _lines_with_floats(w, rng):
    tags = _tag_mix(w.batch, rng)
    for i, t in enumerate(tags):
        t.append("ZF:B:f,1.5,-0.1,3e-40" if i % 3 else "ZF:B:f,2")
    return format_sam(w.batch, w.header, tags)


def test_full_path_and_sub_ranges():
    """sort + markdup + BQSR apply: the text carries the oracle's order, FLAG and QUAL; uneven sub-ranges concatenate to the whole"""
    w = _workload(seed=43)
    lines = _lines_with_floats(w, np.random.default_rng(8))
    ctx = device.Context(w.header, profile=True)
    set_side_inputs(ctx, w)
    ctx.append_sam(b"\n".join(lines))
    g = gpu_phases(ctx, profile=True)
    o = oracle_pipeline(w)
    assert np.array_equal(g["perm"], o["perm"]) and np.array_equal(g["flag"], o["flag"]) and np.array_equal(g["qual"], o["qual"])
    qo = g["qual_off"].astype(np.int64)
    want = []
    for k in range(ctx.n):
        a = parse_sam_alignment(lines[int(o["perm"][k])])
        a["FLAG"] = int(o["flag"][k])
        a["QUAL"] = o["qual"][qo[k]:qo[k + 1]].tobytes()
        want.append(format_alignment(a))
    text, off = ctx.fetch_sam()
    assert text.tobytes() == b"".join(want)
    assert np.array_equal(off, _line_off(want))
    n = ctx.n
    parts, offs = [], []
    for a, b in ((0, 7), (7, 8), (8, 1001), (1001, n - 3), (n - 3, n)):
        t, lo = ctx.fetch_sam(a, b - a)
        parts.append(t.tobytes())
        assert np.array_equal(lo, off[a:b + 1] - off[a]), (a, b)
    assert b"".join(parts) == text.tobytes()
    st = ctx.kernel_stats()
    assert all(k in st for k in OUT_KERNELS + ("sam_out_float",)), sorted(st)
    ctx.close()


def test_sam_and_bam_input_agree_and_round_trip():
    """the same reads through elp_append_sam and elp_append_bam give the same text; that text appended again reproduces fetch_bam"""
    w = _workload(900, seed=12)
    # (B:s 65535 is written back as -1, which parseSamNumericArray's ParseUint rejects: the reference cannot read that line of its own output)
    lines = [x.replace(b"ZB:B:s,1,2,65535", b"ZB:B:s,1,2,32767") for x in _lines_with_floats(w, np.random.default_rng(2))]
    raw, off = sam_lines_to_bam(lines, w.header)
    out = []
    for mode in ("sam", "bam"):
        ctx = device.Context(w.header)
        if mode == "sam":
            ctx.append_sam(b"\n".join(lines) + b"\n")
        else:
            ctx.append_bam(raw, off)
        ctx.sort_markdup()
        out.append((ctx.fetch_sam()[0].tobytes(), ctx.fetch_bam()[0].tobytes()))
        ctx.close()
    assert out[0] == out[1]
    again = device.Context(w.header)
    again.append_sam(out[0][0])
    again.sort_markdup(device.SO_KEEP, False)
    assert again.fetch_bam()[0].tobytes() == out[0][1]
    assert again.fetch_sam()[0].tobytes() == out[0][0]
    again.close()


def _raw_fetch_sam(ctx, first, n, cap):
    buf = np.full(max(cap, 1), 0xAA, np.uint8)
    off = np.full(n + 1, 7, np.uint64)
    rc = ctx.L.elp_fetch_sam(ctx.h, first, n, buf.ctypes.data_as(C.c_void_p), cap, off.ctypes.data_as(C.c_void_p))
    return rc, buf, off


def test_refusals():
    good = line(QNAME=b"ok")
    ctx = device.Context(HEADER)
    ctx.append_sam(good)
    rc, buf, off = _raw_fetch_sam(ctx, 0, 1, 1000)
    assert rc == _lib.ESTATE and np.all(buf == 0xAA) and np.all(off == 7)          # before elp_sort_markdup
    ctx.sort_markdup(device.SO_KEEP, False)
    need = int(ctx.L.elp_fetch_sam_bytes(ctx.h, 0, 1))
    assert need == len(sam_to_sam(good))
    for first, n, cap in ((0, 2, 1000), (1, 1, 1000), (0, 1, need - 1)):           # a range past n, a buffer too small
        rc, buf, off = _raw_fetch_sam(ctx, first, n, cap)
        assert rc == _lib.EINVAL and np.all(buf == 0xAA) and np.all(off == 7), (first, n, cap)
    rc, buf, off = _raw_fetch_sam(ctx, 0, 1, need)
    assert rc == 0 and buf[:need].tobytes() == sam_to_sam(good) and list(off) == [0, need]
    ctx.close()
    # a read that came in as columns
    w = synth.make_workload(50, [("chr1", 100_000)], seed=3)
    ctx = device.Context(w.header)
    ctx.append(w.batch)
    ctx.sort_markdup()
    with pytest.raises(device.ElprepError) as ei:
        ctx.fetch_sam()
    assert ei.value.code == _lib.ESTATE
    ctx.close()
    # elp_clean_sam rewrote a CIGAR (chr2 has 1000 bases)
    ctx = device.Context(HEADER)
    ctx.append_sam(line(POS=b"998"))
    assert ctx.clean_sam() == 1
    ctx.sort_markdup(device.SO_KEEP, False)
    with pytest.raises(device.ElprepError) as ei:
        ctx.fetch_sam()
    assert ei.value.code == _lib.ESTATE
    ctx.close()
    # a CIGAR operation code above 8
    raw, off = _join([bam_record(), bam_record(cigar=((4, 9),))])
    ctx = device.Context(HEADER)
    ctx.append_bam(raw, off)
    ctx.sort_markdup(device.SO_KEEP, False)
    with pytest.raises(device.ElprepError) as ei:
        ctx.fetch_sam()
    assert ei.value.code == _lib.EBAM
    assert ctx.fetch_sam(0, 1)[0].tobytes() == bam_to_sam(bam_record(), NAMES)
    ctx.close()
    # a context created without contig_names
    L = _lib.load()
    clen = np.array([1000], np.int32)
    cfg = _lib.ElpConfig(0, 1, None, clen.ctypes.data_as(C.c_void_p), 0, None, None, None, 500, 0, None, 0, b"GATK", 100, 0)
    h = C.c_void_p()
    assert L.elp_create(C.byref(cfg), C.byref(h)) == 0
    raw, off = _join([bam_record(refid=0, nref=0)])
    assert L.elp_append_bam(h, raw.ctypes.data_as(C.c_void_p), raw.size, off.ctypes.data_as(C.c_void_p), 1) == 0
    assert L.elp_sort_markdup(h, 0, 0) == 0
    buf = np.zeros(1000, np.uint8)
    assert L.elp_fetch_sam(h, 0, 1, buf.ctypes.data_as(C.c_void_p), 1000, None) == _lib.EINVAL
    L.elp_destroy(h)


@pytest.mark.parametrize("rname,rnext,lost", [(b"chrZ", b"=", True), (b"chr1", b"chrZ", True), (b"*", b"=", True), (b"chrZ", b"*", True), (b"", b"*", True),
                                              (b"*", b"*", False), (b"chr1", b"=", False), (b"chr1", b"chr1", False), (b"*", b"chr2", False)])
def test_lost_names(rname, rnext, lost):
    """lines whose RNAME / RNEXT the stored record cannot reproduce are counted; fetch_sam refuses them and names the count, fetch_bam is
    unchanged.  Lines the ingest filters drop do not count."""
    text = line(QNAME=b"a", RNAME=rname, RNEXT=rnext)
    ctx = device.Context(HEADER)
    ctx.append_sam(line(QNAME=b"ok") + b"\n" + text + b"\n" + text)
    ctx.sort_markdup(device.SO_KEEP, False)
    raw, _ = ctx.fetch_bam()
    assert raw.tobytes() == b"".join(sam_line_to_bam(x, HEADER) for x in (line(QNAME=b"ok"), text, text))
    if lost:
        with pytest.raises(device.ElprepError) as ei:
            ctx.fetch_sam()
        assert ei.value.code == _lib.ESTATE and "2 SAM lines" in str(ei.value), str(ei.value)
        assert int(ctx.L.elp_fetch_sam_bytes(ctx.h, 0, 1)) == 0
    else:
        assert ctx.fetch_sam()[0].tobytes() == b"".join(sam_to_sam(x) for x in (line(QNAME=b"ok"), text, text))
    ctx.close()
    if lost:                                                              # filtered out (unmapped), then the context can write SAM
        ctx = device.Context(HEADER)
        ctx.set_ingest_filter(_lib.FILTER_UNMAPPED, 0)
        ctx.append_sam(line(QNAME=b"ok") + b"\n" + line(QNAME=b"a", FLAG=b"4", RNAME=rname, RNEXT=rnext))
        assert ctx.n == 1
        ctx.sort_markdup(device.SO_KEEP, False)
        assert ctx.fetch_sam()[0].tobytes() == sam_to_sam(line(QNAME=b"ok"))
        ctx.close()
        ctx = device.Context(HEADER)                                      # kept by the filter: refused
        ctx.set_ingest_filter(_lib.FILTER_UNMAPPED, 0)
        ctx.append_sam(line(QNAME=b"ok", FLAG=b"4") + b"\n" + text)
        ctx.sort_markdup(device.SO_KEEP, False)
        with pytest.raises(device.ElprepError) as ei:
            ctx.fetch_sam()
        assert "1 SAM lines" in str(ei.value)
        ctx.close()


def test_c1_size():
    """2 M reads, fetched in a few chunks, against the vectorised SAM writer of the same reads in output order (multi-tile scan)"""
    w = synth.make_workload(1_000_000, synth.scaled_hg38(64.0), seed=78, want_reference=False)
    text = sam_text(w.batch, w.header)
    ctx = device.Context(w.header, profile=True)
    cut = int(np.nonzero(text[: text.size // 2] == 10)[0][-1]) + 1
    ctx.append_sam(text[:cut])
    ctx.append_sam(text[cut:])
    ctx.sort_markdup()
    idx, flag, qoff, qual = ctx.fetch()
    b = w.batch.take(idx.astype(np.int64))
    b.flag = flag.copy()
    assert np.array_equal(b.qual, qual[:int(qoff[-1])])
    want = sam_text(b, w.header)
    n = ctx.n
    cuts = [0, 333_333, 1_000_001, n]
    got = [ctx.fetch_sam(a, c - a)[0] for a, c in zip(cuts[:-1], cuts[1:])]
    assert np.array_equal(np.concatenate(got), want)
    st = ctx.kernel_stats()
    assert all(st[k]["launches"] >= 3 for k in OUT_KERNELS), sorted(st)
    assert "sam_out_float" not in st
    ctx.close()
