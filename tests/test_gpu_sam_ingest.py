"""elp_append_sam: SAM text lines parsed on the device into BAM records, then the BAM ingest core.  Each record must equal what
formatBamAlignment(parseSamAlignment(line)) writes (tests/samtext.py), and the path computes what the column and BAM paths compute."""
import struct

import numpy as np
import pytest

from elprep_b200 import bgzf, device, sam, synth, _lib
from samtext import format_sam, sam_line_to_bam, sam_lines_to_bam, sam_text
from test_sam_text import ERRORS, HEADER, KAT, line
from util import encode_bam, gpu_phases, oracle_pipeline, oracle_tables_dense, set_side_inputs

pytestmark = pytest.mark.gpu

SMALL = [("chr20", 600_000), ("chr21", 300_000), ("chrM", 16_569)]
SAM_KERNELS = ("sam_lines", "sam_measure", "sam_emit")


def _tag_mix(b, rng):
    """per read: NM, MD, a negative AS, XS as f (some values the host rounds), B:s, A, and sr on a few reads"""
    out = []
    for i in range(b.n):
        t = [f"NM:i:{int(rng.integers(0, 9))}", "MD:Z:75A74", f"AS:i:{-int(rng.integers(1, 200))}",
             "XS:f:" + ("1.5" if i % 5 else "16777217"), "ZB:B:s,1,2,65535", "XA:A:q"]
        if b.opt_flags[i]:
            t.append("sr:i:1")
        out.append(t)
    return out


def _workload(n_pairs=1500, seed=41, sr=True):
    """a synthetic workload; with sr, every 97th read carries the sr tag (the oracle sees it through opt_flags)"""
    w = synth.make_workload(n_pairs, SMALL, seed=seed)
    if sr:
        w.batch.opt_flags[::97] = 1
    return w


def _fetch_expect(lines, header, ctx):
    """sam_line_to_bam of every line in output order, FLAG and QUAL patched from the context's result"""
    idx, flag, qoff, qual = ctx.fetch()
    out = []
    for k in range(ctx.n):
        r = bytearray(sam_line_to_bam(lines[int(idx[k])], header))
        r[18:20] = struct.pack("<H", int(flag[k]))
        ln, lname, ncig = struct.unpack_from("<i", r, 20)[0], r[12], struct.unpack_from("<H", r, 16)[0]
        q0 = 36 + lname + 4 * ncig + (ln + 1) // 2
        r[q0:q0 + ln] = bytes(qual[int(qoff[k]):int(qoff[k + 1])])
        out.append(bytes(r))
    return b"".join(out)


def test_path_parity():
    w = _workload()
    rng = np.random.default_rng(3)
    lines = format_sam(w.batch, w.header, _tag_mix(w.batch, rng))
    n = len(lines)
    a, b = n // 3, 2 * n // 3
    text1 = b"".join(x + b"\n" for x in lines[:a])
    text2 = b"".join(x + b"\r\n" for x in lines[a:b])
    text3 = b"\n".join(lines[b:])                                         # the last line without '\n'
    ctx = device.Context(w.header, profile=True)
    set_side_inputs(ctx, w)
    for t in (text1, text2, text3):
        ctx.append_sam(t)
    assert ctx.n == n
    g = gpu_phases(ctx, profile=True)
    o = oracle_pipeline(w)
    assert np.array_equal(g["perm"], o["perm"]) and np.array_equal(g["flag"], o["flag"])
    d, e = oracle_tables_dense(o["tables"])
    assert np.array_equal(g["tables"], d) and np.array_equal(g["emp"], e)
    assert np.array_equal(g["qual"], o["qual"])
    assert all(k in g["stats"] for k in SAM_KERNELS), sorted(g["stats"])
    assert np.array_equal(ctx.fetch_opt_flags(), w.batch.opt_flags[g["perm"].astype(np.int64)])
    raw, _ = ctx.fetch_bam()
    assert raw.tobytes() == _fetch_expect(lines, w.header, ctx)
    # the BAM path over the same reads
    extra = [b"srC\x01" if f else b"" for f in w.batch.opt_flags]
    braw, boff = encode_bam(w.batch, w.header, extra_tags=extra)
    ref = device.Context(w.header)
    set_side_inputs(ref, w)
    ref.append_bam(braw, boff)
    gb = gpu_phases(ref)
    for k in ("perm", "flag", "qual", "tables"):
        assert np.array_equal(g[k], gb[k]), k
    ctx.close(); ref.close()


NEG_POS = {"bin_negative_pos"}                                            # ingested, but the phases refuse a negative POS (ELP_ELIMIT)


@pytest.mark.parametrize("name,text,check", KAT, ids=[k[0] for k in KAT])
def test_quirk_lines(name, text, check):
    ctx = device.Context(HEADER)
    ctx.append_sam(text)
    assert ctx.n == 1
    if name in NEG_POS:
        with pytest.raises(device.ElprepError) as ei:
            ctx.sort_markdup(device.SO_KEEP, False)
        assert ei.value.code == _lib.ELIMIT
        return
    ctx.sort_markdup(device.SO_KEEP, False)
    raw, _ = ctx.fetch_bam()
    assert raw.tobytes() == sam_line_to_bam(text, HEADER)
    ctx.close()


def test_quirk_lines_in_one_call():
    lines = [k[1] for k in KAT if k[0] not in NEG_POS]
    ctx = device.Context(HEADER, profile=True)
    ctx.append_sam(b"\n".join(lines) + b"\n")
    ctx.sort_markdup(device.SO_KEEP, False)
    raw, _ = ctx.fetch_bam()
    assert raw.tobytes() == sam_lines_to_bam(lines, HEADER)[0].tobytes()
    assert "sam_fpatch" in ctx.kernel_stats()
    ctx.close()


def test_long_read():
    """a 100 kb read with thousands of CIGAR operations and a long MD tag: ingest and fetch"""
    rng = np.random.default_rng(9)
    L = 100_000
    seq = rng.choice(np.frombuffer(b"ACGT", np.uint8), L).tobytes()
    qual = bytes(rng.integers(35, 75, L).astype(np.uint8))
    ops, left = [], L
    while left > 0:
        m = min(left, int(rng.integers(5, 40)))
        ops.append(f"{m}M")
        left -= m
        if left > 0:
            ops.append(f"{int(rng.integers(1, 5))}D")
    cig = "".join(ops).encode()
    md = b"".join(b"%dA" % int(rng.integers(1, 50)) for _ in range(3000))
    text = line(QNAME=b"long", POS=b"1000", CIGAR=cig, SEQ=seq, QUAL=qual, tags=[b"MD:Z:" + md, b"NM:i:3000", b"XS:f:0.25"])
    ctx = device.Context(HEADER)
    ctx.append_sam(text)
    ctx.sort_markdup(device.SO_KEEP, False)
    raw, _ = ctx.fetch_bam()
    exp = sam_line_to_bam(text, HEADER)
    assert struct.unpack_from("<H", exp, 16)[0] > 2000
    assert raw.tobytes() == exp
    ctx.close()


@pytest.mark.parametrize("name,text,kind", ERRORS, ids=[e[0] for e in ERRORS])
def test_errors(name, text, kind):
    ctx = device.Context(HEADER)
    good = line(QNAME=b"ok")
    ctx.append_sam(good + b"\n")
    with pytest.raises(device.ElprepError) as ei:
        ctx.append_sam(good + b"\n" + text + b"\n" + good)
    assert ei.value.code == {"ESAM": _lib.ESAM, "ELIMIT": _lib.ELIMIT}[kind], str(ei.value)
    if kind == "ESAM":
        assert "line 1 " in str(ei.value), str(ei.value)
    assert ctx.n == 1
    ctx.append_sam(good)
    assert ctx.n == 2
    ctx.close()


def test_unknown_rg_and_missing_names():
    ctx = device.Context(HEADER)
    with pytest.raises(device.ElprepError) as ei:
        ctx.append_sam(line(tags=[b"RG:Z:nope"]))
    assert ei.value.code == _lib.EBAM and ctx.n == 0
    ctx.append_sam(line(tags=[b"RG:Z:g1"]))
    assert ctx.n == 1
    ctx.close()
    # a context created without contig_names cannot resolve RNAME
    import ctypes as C
    L = _lib.load()
    clen = np.array([1000], np.int32)
    cfg = _lib.ElpConfig(0, 1, None, clen.ctypes.data_as(C.c_void_p), 0, None, None, None, 500, 0, None, 0, b"GATK", 100, 0)
    h = C.c_void_p()
    assert L.elp_create(C.byref(cfg), C.byref(h)) == 0
    t = line()
    assert L.elp_append_sam(h, t, len(t)) == _lib.EINVAL
    L.elp_destroy(h)


def test_ingest_filters():
    """the cases of test_bam_ingest_filters plus strict exact-match and target regions, over SAM text"""
    w = synth.make_workload(2_500, SMALL, seed=29, unmapped_frac=0.1)
    b = w.batch
    b.flag[::17] |= 0x400
    rng = np.random.default_rng(1)
    strict = rng.random(b.n) < 0.5
    tags = [["X0:i:1", "X1:i:0", "XM:i:0", "XO:i:0", "XG:i:0"] if s else ["X0:i:2", "X1:i:0", "XM:i:0", "XO:i:0", "XG:i:0"] for s in strict]
    text = b"".join(x + b"\n" for x in format_sam(b, w.header, tags))
    ncig = (b.cigar_off[1:] - b.cigar_off[:-1]).astype(np.int64)
    ops_ok = np.ones(b.n, bool)
    for i in np.nonzero(ncig > 0)[0]:
        ops = b.cigar[int(b.cigar_off[i]):int(b.cigar_off[i + 1])] & 15
        ops_ok[i] = bool(np.all((ops == 0) | (ops == 4)))
    # target regions: one interval per contig; the reference's overlap of [POS, End()] (End from the CIGAR)
    regions = {0: (100_000, 300_000), 1: (50_000, 60_000)}
    end = b.pos.astype(np.int64).copy()
    for i in range(b.n):
        if not b.flag[i] & 4:
            cg = b.cigar[int(b.cigar_off[i]):int(b.cigar_off[i + 1])]
            rl = sum(int(c) >> 4 for c in cg if int(c) & 15 in (0, 1, 4, 7, 8))
            fl = sum(int(c) >> 4 for c in cg if int(c) & 15 in (0, 2, 3, 7, 8))
            if rl > 0:
                end[i] = int(b.pos[i]) + fl - 1
    in_reg = np.array([int(b.refid[i]) in regions and regions[int(b.refid[i])][0] <= end[i] - 1 and int(b.pos[i]) - 1 < regions[int(b.refid[i])][1]
                       for i in range(b.n)])
    preds = {
        _lib.FILTER_UNMAPPED: (b.flag & 4) == 0,
        _lib.FILTER_UNMAPPED_STRICT: ((b.flag & 4) == 0) & (b.pos != 0) & (b.refid >= 0),
        _lib.FILTER_NON_EXACT: ops_ok,
        _lib.FILTER_DUPLICATES: (b.flag & 0x400) == 0,
        _lib.FILTER_NON_EXACT_STRICT: strict,
        _lib.FILTER_TARGET_REGIONS: in_reg,
    }
    cases = [(m, 0) for m in preds] + [(0, 30), (_lib.FILTER_UNMAPPED | _lib.FILTER_NON_EXACT | _lib.FILTER_DUPLICATES, 20), (0, 300)]
    half = text.index(b"\n", len(text) // 2) + 1
    for mask, mq in cases:
        keep = b.mapq.astype(np.int64) >= mq
        for bit, p in preds.items():
            if mask & bit:
                keep &= p
        sub = b.take(np.nonzero(keep)[0])
        ctx = device.Context(w.header)
        ctx.set_ingest_filter(mask, mq)
        for c, (s, e) in regions.items():
            ctx.set_target_regions(c, [s, e])
        ctx.append_sam(text[:half])
        ctx.append_sam(text[half:])
        assert ctx.n == sub.n and ctx.n_filtered() == b.n - sub.n, (mask, mq)
        ref = device.Context(w.header)
        ref.append(sub)
        for c_ in (ctx, ref):
            c_.sort_markdup()
        a1, a2 = ctx.fetch(), ref.fetch()
        assert all(np.array_equal(x, y) for x, y in zip(a1[:3], a2[:3])), (mask, mq)
        assert np.array_equal(a1[3][:int(a1[2][-1])], a2[3][:int(a2[2][-1])]), (mask, mq)
        ctx.close(); ref.close()


def test_mixed_sam_then_bam():
    w = _workload(800, seed=7, sr=False)
    b = w.batch
    h = b.n // 2
    lines = format_sam(b.take(np.arange(h)), w.header)
    braw, boff = encode_bam(b.take(np.arange(h, b.n)), w.header)
    ctx = device.Context(w.header)
    set_side_inputs(ctx, w)
    ctx.append_sam(b"\n".join(lines))
    ctx.append_bam(braw, boff)
    g = gpu_phases(ctx)
    o = oracle_pipeline(w)
    assert np.array_equal(g["perm"], o["perm"]) and np.array_equal(g["flag"], o["flag"]) and np.array_equal(g["qual"], o["qual"])
    raw, off = ctx.fetch_bam()
    recs = [sam_line_to_bam(x, w.header) for x in lines] + [braw[int(boff[i]):int(boff[i + 1])].tobytes() for i in range(b.n - h)]
    idx, flag, qoff, qual = ctx.fetch()
    for k in range(b.n):
        r = bytearray(recs[int(idx[k])])
        r[18:20] = struct.pack("<H", int(flag[k]))
        ln, lname, ncig = struct.unpack_from("<i", r, 20)[0], r[12], struct.unpack_from("<H", r, 16)[0]
        q0 = 36 + lname + 4 * ncig + (ln + 1) // 2
        r[q0:q0 + ln] = bytes(qual[int(qoff[k]):int(qoff[k + 1])])
        assert raw[int(off[k]):int(off[k + 1])].tobytes() == bytes(r), k
    ctx.close()


def test_whole_sam_file():
    """SAM file bytes -> parse_sam_header -> Context -> append_sam -> path -> fetch_bam -> BGZF: the decoded result carries the oracle's FLAG and QUAL"""
    from util import decode_bam
    w = _workload(1000, seed=11, sr=False)
    hdr = b"@HD\tVN:1.6\tSO:unsorted\n" + b"".join(b"@SQ\tSN:%s\tLN:%d\n" % (s["SN"].encode(), int(s["LN"])) for s in w.header.SQ)
    hdr += b"".join(b"@RG\tID:%s\tSM:x\n" % r["ID"].encode() for r in w.header.RG) + b"@PG\tID:bwa\tPN:bwa\n@CO\tsynthetic\n"
    text = hdr + sam_text(w.batch, w.header).tobytes()
    h, n0 = sam.parse_sam_header(text)
    assert n0 == len(hdr)
    for k in ("LB", "PU"):
        for r, r0 in zip(h.RG, w.header.RG):
            if k in r0:
                r[k] = r0[k]
    ctx = device.Context(h)
    set_side_inputs(ctx, w)
    ctx.append_sam(np.frombuffer(text, np.uint8)[n0:])
    gpu_phases(ctx)
    raw, off = ctx.fetch_bam()
    d = decode_bam(bgzf.inflate(bgzf.deflate(raw)), off, h)
    o = oracle_pipeline(w)
    assert np.array_equal(d.flag, o["flag"]) and np.array_equal(d.qual, o["qual"])
    ctx.close()


def test_c1_size_matches_bam_path():
    """2 M reads of SAM text give the fetch_bam output of elp_append_bam of the same reads (multi-tile line finder and scan).  The BAM
    encoder writes a constant bin; the SAM path writes formatBamAlignment's, checked on a sample against the restatement."""
    w = synth.make_workload(1_000_000, synth.scaled_hg38(64.0), seed=77, want_reference=False)
    text = sam_text(w.batch, w.header, const_tags=b"NM:i:0")           # the BAM encoder writes NM:C:<edits> before RG:Z
    raw, offs = synth.encode_bam(w.batch, w.header)
    outs = []
    for mode in ("sam", "bam"):
        ctx = device.Context(w.header)
        if mode == "sam":
            cut = int(np.nonzero(text[: text.size // 2] == 10)[0][-1]) + 1
            ctx.append_sam(text[:cut])
            ctx.append_sam(text[cut:])
        else:
            ctx.append_bam(raw, offs)
        assert ctx.n == w.batch.n
        ctx.sort_markdup()
        outs.append(ctx.fetch_bam() + (ctx.fetch()[0].copy(),))
        ctx.close()
    (sr, so, sp), (br, bo, bp) = outs
    assert np.array_equal(sp, bp) and np.array_equal(so, bo)
    starts = so[:-1].astype(np.int64)
    bins = sr[starts + 14].astype(np.int64) | (sr[starts + 15].astype(np.int64) << 8)
    sr, br = sr.copy(), br.copy()
    assert {len(r["ID"]) for r in w.header.RG} == {3}
    nm = so[1:].astype(np.int64) - 8                                    # the NM value byte, in front of "RGZ" + 3-byte ID + NUL
    for pos in (starts + 14, starts + 15, nm):
        sr[pos] = 0
        br[pos] = 0
    assert np.array_equal(sr, br)
    lo = np.zeros(w.batch.n + 1, np.int64)
    nl = np.nonzero(text == 10)[0]
    lo[1:] = nl + 1
    for k in np.random.default_rng(0).integers(0, w.batch.n, 2000):
        i = int(sp[k])
        exp = sam_line_to_bam(text[lo[i]:nl[i]].tobytes(), w.header)
        assert int(bins[k]) == struct.unpack_from("<H", exp, 14)[0], k
