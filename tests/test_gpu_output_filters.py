"""The write-phase filters of elp_fetch_bam / elp_fetch_sam (elp_set_output_filter): record selection (RemoveDuplicateReads on the FLAG after
marking, RemoveOptionalReads), the optional-field filters against the restatement in tests/outfilter.py, and ClearDuplicateFlag at ingest."""
import ctypes as C
import struct

import numpy as np
import pytest

from elprep_b200 import device, synth, _lib
from outfilter import filter_record, split_records
from samformat import bam_to_sam
from samtext import sam_line_to_bam, sam_text
from test_gpu_sam_ingest import NEG_POS, _workload
from test_gpu_sam_output import LOST, _big_records, _join
from test_sam_format import LINES, NAMES, bam_record
from test_sam_text import HEADER, KAT, line
from util import encode_bam, gpu_phases, oracle_pipeline, set_side_inputs

pytestmark = pytest.mark.gpu

DUP, SR = _lib.OUT_REMOVE_DUPLICATES, _lib.OUT_REMOVE_OPTIONAL_READS
NEW_KERNELS = {"out_select", "bam_out_fields_measure", "bam_out_fields_emit"}
SR_TAG = b"sri\x01\x00\x00\x00"


def _dup_workload(seed):
    """duplicate-rich reads, every 11th flagged 0x400 on input, every 97th with the sr tag"""
    w = _workload(1500, seed=seed)
    w.batch.flag[5::11] |= 0x400
    raw, off = encode_bam(w.batch, w.header, np.random.default_rng(seed), extra_tags=[SR_TAG if o else b"" for o in w.batch.opt_flags])
    return w, raw, off


def _bam_ctx(w, raw, off, bqsr, ingest=0, profile=False):
    ctx = device.Context(w.header, profile=profile)
    set_side_inputs(ctx, w)
    ctx.set_ingest_filter(ingest, 0)
    ctx.append_bam(raw, off)
    g = gpu_phases(ctx, bqsr=bqsr)
    return ctx, g


def _rec_flags(recs):
    return np.array([struct.unpack_from("<H", r, 18)[0] for r in recs], np.uint16)


def test_no_filter_is_unchanged():
    """mask 0 with empty lists (and a remove list of strings that match nothing) gives the bytes of the unfiltered calls; no new kernel runs"""
    w, raw, off = _dup_workload(3)
    ctx, _ = _bam_ctx(w, raw, off, bqsr=False, profile=True)
    ctx.reset_stats()
    before = (ctx.fetch_bam(), ctx.fetch_sam())
    names = set(ctx.kernel_stats())
    for args in (dict(), dict(mask=0, remove=(), keep=None), dict(remove=("", "N", "XYZ"))):
        ctx.set_output_filter(**args)
        ctx.reset_stats()
        assert ctx.n_output() == ctx.n
        b, s = ctx.fetch_bam(), ctx.fetch_sam()
        assert b[0].tobytes() == before[0][0].tobytes() and np.array_equal(b[1], before[0][1])
        assert s[0].tobytes() == before[1][0].tobytes() and np.array_equal(s[1], before[1][1])
        assert set(ctx.kernel_stats()) == names and not names & NEW_KERNELS
    ctx.close()


@pytest.mark.parametrize("bqsr", [False, True])
def test_remove_duplicates_and_optional_reads(bqsr):
    w, raw, off = _dup_workload(17)
    o = oracle_pipeline(w, bqsr=bqsr)
    ctx, g = _bam_ctx(w, raw, off, bqsr=bqsr, profile=True)
    assert np.array_equal(g["perm"], o["perm"]) and np.array_equal(g["flag"], o["flag"])
    recs = split_records(*ctx.fetch_bam())
    lines = split_records(*ctx.fetch_sam())
    assert np.array_equal(_rec_flags(recs), o["flag"])
    optf = ctx.fetch_opt_flags()
    assert optf.sum() > 0
    is_dup = (o["flag"] & 0x400) != 0
    assert is_dup.sum() > 0 and (is_dup & (optf != 0)).sum() < optf.sum()
    for mask, drop in ((DUP, is_dup), (SR, optf != 0), (DUP | SR, is_dup | (optf != 0))):
        ctx.set_output_filter(mask)
        keep = np.nonzero(~drop)[0]
        assert ctx.n_output() == keep.size
        b, boff = ctx.fetch_bam()
        assert b.tobytes() == b"".join(recs[k] for k in keep)
        assert np.array_equal(np.diff(boff.astype(np.int64)), [len(recs[k]) for k in keep])
        s, _ = ctx.fetch_sam()
        assert s.tobytes() == b"".join(lines[k] for k in keep)
        m = keep.size                                                     # uneven sub-ranges concatenate to the whole
        cuts = [0, 1, 8, 501, m - 2, m]
        bp = [ctx.fetch_bam(a, c - a) for a, c in zip(cuts[:-1], cuts[1:])]
        sp = [ctx.fetch_sam(a, c - a)[0].tobytes() for a, c in zip(cuts[:-1], cuts[1:])]
        assert b"".join(x[0].tobytes() for x in bp) == b.tobytes() and b"".join(sp) == s.tobytes()
        for (a, c), (_, po) in zip(zip(cuts[:-1], cuts[1:]), bp):
            assert np.array_equal(po, boff[a:c + 1] - boff[a])
        if mask & DUP:                                                    # the survivors carry the oracle's FLAGs of a run on all reads
            assert np.array_equal(_rec_flags(split_records(b, boff)), o["flag"][keep])
    assert "out_select" in ctx.kernel_stats()
    ctx.close()
    # the ingest bit ELP_FILTER_DUPLICATES drops the reads flagged on input before marking, so other reads become duplicates or survive
    ctx2, _ = _bam_ctx(w, raw, off, bqsr=False, ingest=_lib.FILTER_DUPLICATES)
    ctx2.set_output_filter(DUP)
    ids = lambda rs: [(r[36:36 + r[12]], r[18:20]) for r in rs]          # QNAME and FLAG of every survivor
    assert ids(split_records(*ctx2.fetch_bam())) != ids(recs[k] for k in np.nonzero(~is_dup)[0])
    ctx2.close()


def _check_fields(ctx, shapes):
    """every shape (remove, keep) through fetch_bam and fetch_sam equals the restatement of the unfiltered records"""
    ctx.set_output_filter()
    recs = split_records(*ctx.fetch_bam())
    for remove, keep in shapes:
        ctx.set_output_filter(0, remove, keep)
        want = [filter_record(r, remove, keep) for r in recs]
        b, boff = ctx.fetch_bam()
        got = split_records(b, boff)
        bad = [i for i in range(len(recs)) if got[i] != want[i]]
        assert not bad, (remove, keep, bad[:5])
        s, soff = ctx.fetch_sam()
        wl = [bam_to_sam(r, NAMES) for r in want]
        gl = split_records(s, soff)
        bad = [i for i in range(len(recs)) if gl[i] != wl[i]]
        assert not bad, (remove, keep, [(gl[i][:200], wl[i][:200]) for i in bad[:3]])
    ctx.set_output_filter()


SHAPES = [(("XA", "a3", "B7", "MD", "XH", "XS", "XZ", "XF", "tag"), None),             # remove only
          ((), ("a1", "a6", "B3", "XC", "XT", "E2", "XI", "XF", "MD")),               # keep only
          ((), ()),                                                                # keep none
          (("a1", "XE", "B2", "XZ"), ("a1", "a2", "XE", "XI", "B2", "B4", "XV", "XZ", "XC", "XH", "F3"))]   # remove, then keep


def test_field_filters_on_hand_built_records():
    """every row of the field table, float specials, a 100 kb read, more than 64 KB of fields and large B arrays"""
    recs = [r for name, r, _ in LINES if name not in ("fixed_bounds", "qual_ff")]
    specials = (0x7F800000, 0xFF800000, 0x7FC00000, 0xFFFFFFFF, 0x00000001, 0x007FFFFF, 0x80000001, 0x00800000)
    recs.append(bam_record(tags=b"".join(b"F%df" % i + struct.pack("<I", v) for i, v in enumerate(specials)) + b"NMC\x01XAAq" + b"NMi\x02\x00\x00\x00"))
    recs += _big_records()
    raw, off = _join(recs)
    ctx = device.Context(HEADER, profile=True)
    ctx.append_bam(raw, off)
    ctx.sort_markdup(device.SO_KEEP, False)
    _check_fields(ctx, SHAPES + [(("NM",), None), ((), ("NM", "XA")), (("nm", "", "N", "NMX"), None), ((), ("nm",))])
    st = ctx.kernel_stats()
    assert {"bam_out_fields_measure", "bam_out_fields_emit"} <= set(st) and "out_select" not in st
    ctx.close()


def test_field_filters_on_sam_input():
    """the known-answer lines of the SAM ingest, and SAM text with tags, through both fetches"""
    lines = [k[1] for k in KAT if k[0] not in NEG_POS | LOST]
    ctx = device.Context(HEADER)
    ctx.append_sam(b"\n".join(lines) + b"\n")
    ctx.sort_markdup(device.SO_KEEP, False)
    _check_fields(ctx, SHAPES + [(("XF", "ZB"), None), ((), ("RG",))])
    ctx.close()


def test_float_slots():
    """f and B:f values that are dropped take no float slot; dropping every float of the call means no sam_out_float launch"""
    fl = lambda *v: struct.pack("<%df" % len(v), *v)
    recs = [bam_record(qname=b"q%d" % i, tags=b"XSf" + fl(1.5 + i) + b"ZFBf" + struct.pack("<I", 3) + fl(0.1, -2.5, 1e-40) + b"NMC\x01" + b"XTf" + fl(-0.25 * i)
                       + b"YFBf" + struct.pack("<I", 1) + fl(3.0))
            for i in range(40)]
    raw, off = _join(recs)
    ctx = device.Context(HEADER, profile=True)
    ctx.append_bam(raw, off)
    ctx.sort_markdup(device.SO_KEEP, False)
    _check_fields(ctx, [(("XS",), None), (("ZF",), None), ((), ("XT", "NM")), (("XS", "XT"), ("ZF", "XT", "XS", "YF"))])
    for remove, keep, floats in ((("XS", "ZF", "XT", "YF"), None, False), ((), ("NM",), False), ((), (), False), (("ZF",), None, True)):
        ctx.set_output_filter(0, remove, keep)
        ctx.reset_stats()
        s, _ = ctx.fetch_sam()
        assert s.tobytes() == b"".join(bam_to_sam(filter_record(r, remove, keep), NAMES) for r in recs)
        assert ("sam_out_float" in ctx.kernel_stats()) == floats, (remove, keep)
    ctx.close()


def test_clear_duplicate_flag():
    """ELP_FILTER_CLEAR_DUPLICATE_FLAG on BAM and SAM ingest, then marking: the FLAGs of the oracle run with input 0x400 cleared"""
    w, raw, off = _dup_workload(29)
    cleared = w.batch.copy()
    cleared.flag &= np.uint16(0xFBFF)
    o = oracle_pipeline(synth.Workload(w.header, cleared, w.contig_bases, w.sites, w.params), bqsr=False)
    o_in = oracle_pipeline(w, bqsr=False)
    assert not np.array_equal(o["flag"], o_in["flag"])
    ctx, g = _bam_ctx(w, raw, off, bqsr=False, ingest=_lib.FILTER_CLEAR_DUPLICATE_FLAG)
    assert np.array_equal(g["perm"], o["perm"]) and np.array_equal(g["flag"], o["flag"])
    assert np.array_equal(_rec_flags(split_records(*ctx.fetch_bam())), o["flag"])
    ctx.close()
    ctx = device.Context(w.header)
    ctx.set_ingest_filter(_lib.FILTER_CLEAR_DUPLICATE_FLAG | _lib.FILTER_UNMAPPED, 0)    # with a record filter: the clear still applies
    ctx.append_sam(sam_text(w.batch, w.header))
    ctx.sort_markdup()
    keep = np.nonzero((w.batch.flag & 4) == 0)[0]
    o2 = oracle_pipeline(synth.Workload(w.header, cleared.take(keep), w.contig_bases, w.sites, w.params), bqsr=False)
    _, flag, _, _ = ctx.fetch(want_qual=False)
    assert ctx.n == keep.size and np.array_equal(flag, o2["flag"])
    ctx.close()


def _raw_fetch(ctx, fn, first, n, cap):
    buf = np.full(max(cap, 1), 0xAA, np.uint8)
    off = np.full(n + 1, 7, np.uint64)
    rc = getattr(ctx.L, fn)(ctx.h, first, n, buf.ctypes.data_as(C.c_void_p), cap, off.ctypes.data_as(C.c_void_p))
    return rc, bool(np.all(buf == 0xAA) and np.all(off == 7))


def test_refusals_and_lifetime():
    ctx = device.Context(HEADER)
    for bad in (8, 0x80000000):
        with pytest.raises(device.ElprepError) as ei:
            ctx.set_output_filter(bad)
        assert ei.value.code == _lib.EINVAL
    arr = (C.c_char_p * 1)(b"NM")
    assert ctx.L.elp_set_output_filter(ctx.h, 0, None, 0, arr, 1) == _lib.EINVAL   # keep tags without ELP_OUT_KEEP_FIELDS
    assert ctx.L.elp_set_output_filter(ctx.h, 0, None, -1, None, 0) == _lib.EINVAL
    ctx.set_output_filter(DUP, remove=("XA",))
    T = [b"XA:A:q", b"NM:i:1"]
    ctx.append_sam(b"\n".join([line(QNAME=b"a", FLAG=b"1024", tags=T), line(QNAME=b"b", tags=T), line(QNAME=b"c", tags=T)]) + b"\n")
    assert ctx.n_output() == 0                                            # before elp_sort_markdup
    for fn in ("elp_fetch_bam", "elp_fetch_sam"):
        rc, untouched = _raw_fetch(ctx, fn, 0, 1, 10_000)
        assert rc == _lib.ESTATE and untouched
    with pytest.raises(device.ElprepError) as ei:
        ctx.fetch_bam()
    assert ei.value.code == _lib.ESTATE
    ctx.sort_markdup(device.SO_KEEP, False)
    assert ctx.n_output() == 2
    for fn in ("elp_fetch_bam", "elp_fetch_sam"):
        for first, n in ((0, 3), (2, 1), (1, 2)):                           # past n_output (but within the reads)
            rc, untouched = _raw_fetch(ctx, fn, first, n, 10_000)
            assert rc == _lib.EINVAL and untouched, (fn, first, n)
        assert int(getattr(ctx.L, fn + "_bytes")(ctx.h, 0, 3)) == 0
    want = [filter_record(sam_line_to_bam(line(QNAME=q, tags=T), HEADER), ("XA",)) for q in (b"b", b"c")]
    assert b"XA" not in b"".join(want) and ctx.fetch_bam()[0].tobytes() == b"".join(want)
    assert ctx.fetch_sam()[0].tobytes() == b"".join(bam_to_sam(r, NAMES) for r in want)
    # the setting survives elp_reset: a second data set in the same context
    ctx.reset()
    assert ctx.n_output() == 0
    ctx.append_sam(b"\n".join([line(QNAME=b"d", tags=T), line(QNAME=b"e", FLAG=b"1024"), line(QNAME=b"f", FLAG=b"1024")]) + b"\n")
    ctx.sort_markdup(device.SO_KEEP, False)
    assert ctx.n_output() == 1
    assert ctx.fetch_bam()[0].tobytes() == filter_record(sam_line_to_bam(line(QNAME=b"d", tags=T), HEADER), ("XA",))
    ctx.set_output_filter()
    assert ctx.n_output() == 3
    ctx.close()
    # after elp_clean_sam rewrote a CIGAR (chr2 has 1000 bases)
    ctx = device.Context(HEADER)
    ctx.set_output_filter(DUP)
    ctx.append_sam(line(POS=b"998"))
    assert ctx.clean_sam() == 1
    ctx.sort_markdup(device.SO_KEEP, False)
    for fn in ("elp_fetch_bam", "elp_fetch_sam"):
        rc, untouched = _raw_fetch(ctx, fn, 0, 1, 10_000)
        assert rc == _lib.ESTATE and untouched
    ctx.close()


def test_c1_size():
    """2 M reads of 150 bp, REMOVE_DUPLICATES plus keep RG, fetched in chunks of 2^18 records, against the unfiltered fetch with the
    duplicates and the MD / NM fields taken out (vectorised)"""
    w = synth.make_workload(1_000_000, synth.scaled_hg38(64.0), seed=91, want_reference=False)
    text = sam_text(w.batch, w.header, const_tags=b"MD:Z:75A74\tNM:i:1")           # (then RG:Z)
    K = len(sam_line_to_bam(line(tags=[b"MD:Z:75A74", b"NM:i:1"]), HEADER)) - len(sam_line_to_bam(line(), HEADER))
    ctx = device.Context(w.header, profile=True)
    cut = int(np.nonzero(text[: text.size // 2] == 10)[0][-1]) + 1
    ctx.append_sam(text[:cut])
    ctx.append_sam(text[cut:])
    del text
    ctx.sort_markdup()
    raw, off = ctx.fetch_bam()
    o = off.astype(np.int64)
    s, lens = o[:-1], np.diff(o)
    u16 = lambda x: raw[x].astype(np.int64) | (raw[x + 1].astype(np.int64) << 8)
    flag, ncig, lseq = u16(s + 18), u16(s + 16), u16(s + 20) | (u16(s + 22) << 16)
    t0 = 36 + raw[s + 12].astype(np.int64) + 4 * ncig + (lseq + 1) // 2 + lseq
    keep = (flag & 0x400) == 0
    assert 0 < keep.sum() < keep.size
    byte_keep = np.repeat(keep, lens)
    drop = ((s + t0)[keep][:, None] + np.arange(K)).ravel()
    byte_keep[drop] = False
    want = raw[byte_keep]
    nl = lens[keep] - K
    noff = np.zeros(nl.size + 1, np.int64)
    np.cumsum(nl, out=noff[1:])
    bs = (nl - 4).astype("<u4").view(np.uint8).reshape(-1, 4)
    for j in range(4):
        want[noff[:-1] + j] = bs[:, j]
    del raw, byte_keep
    ctx.set_output_filter(DUP, keep=("RG",))
    m = ctx.n_output()
    assert m == int(keep.sum())
    got, pos = [], 0
    for a in range(0, m, 1 << 18):
        c = min(m, a + (1 << 18))
        b, bo = ctx.fetch_bam(a, c - a)
        assert np.array_equal(bo.astype(np.int64), noff[a:c + 1] - noff[a])
        got.append(b)
    assert np.array_equal(np.concatenate(got), want)
    st = ctx.kernel_stats()
    assert st["bam_out_fields_emit"]["launches"] >= 2 and "out_select" in st
    ctx.close()
