"""The ingest filters fused into elp_append_bam / elp_append_sam (bam_keep_kernel and the compaction after it) and elp_clean_sam, against
the restatement in tests/ingestfilter_ref.py, at their edges: region boundaries, MAPQ limits, every tag type of the strict filter, drops
around the 256-thread block edge, malformed records under every filter, CleanSam clip points in every operation and what the written
records say afterwards.  Every filter case is sent as BAM records and as SAM lines and asserts which reads arrived (FLAG, QNAME,
permutation), elp_n_filtered, the bytes elp_fetch_bam hands back and whether bam_keep ran."""
import struct

import numpy as np
import pytest

import ingestfilter_ref as R
from elprep_b200 import _lib, device, sam, synth
from samtext import sam_line_to_bam

pytestmark = pytest.mark.gpu
INT32_MAX = (1 << 31) - 1
H = sam.Header(sq=[{"SN": "c0", "LN": 1000}, {"SN": "c1", "LN": 1000}, {"SN": "c2", "LN": 1000}], rg=[{"ID": "g1", "LB": "l1"}])


def line(i, flag=0, rname="c0", pos=100, mapq=30, cigar="10M", tags=b"", lseq=None):
    c = R.parse_cigar(cigar) if cigar != "*" else []
    n = lseq if lseq is not None else (R.read_length(c) or 10)
    return b"\t".join([b"q%05d" % i, b"%d" % flag, rname.encode(), b"%d" % pos, b"%d" % mapq, cigar.encode(), b"*", b"0", b"0",
                       b"ACGT" * (n // 4) + b"ACGT"[:n % 4], b"I" * n]) + (b"\t" + tags if tags else b"")


def _records(lines, hdr=H):
    recs = [sam_line_to_bam(x, hdr) for x in lines]
    off = np.zeros(len(recs) + 1, np.uint64)
    np.cumsum([len(r) for r in recs], out=off[1:])
    return recs, np.frombuffer(b"".join(recs), np.uint8).copy(), off


def _ctx(mask, min_mapq, regions, hdr=H):
    ctx = device.Context(hdr, profile=True)
    for ci, iv in (regions or {}).items():
        ctx.set_target_regions(ci, np.asarray(iv, np.int32).reshape(-1, 2), already_flat=False)
    ctx.set_ingest_filter(mask, min_mapq)
    return ctx


def _fetched(ctx):
    ctx.sort_markdup(device.SO_KEEP, False)
    idx, flag, _, _ = ctx.fetch(want_qual=False)
    out, off = ctx.fetch_bam() if ctx.n else (np.zeros(0, np.uint8), np.zeros(1, np.uint64))
    return idx, flag, out, off


def check_filter(lines, pred, mask=0, min_mapq=0, regions=None, paths=("bam", "sam"), hdr=H):
    """lines through both ingest paths under (mask, min_mapq); pred: the restatement's keep predicate on a parsed record"""
    recs, raw, off = _records(lines, hdr)
    keep = [i for i, r in enumerate(recs) if pred(R.parse_bam(r))]
    # bam_keep runs for a record filter or a MAPQ threshold that can drop a read (byte(mq) == 0 keeps every read: no launch)
    active = mask & ~_lib.FILTER_CLEAR_DUPLICATE_FLAG or min_mapq > 255 or (min_mapq != 0 and min_mapq & 255 != 0)
    for path in paths:
        ctx = _ctx(mask, min_mapq, regions, hdr)
        try:
            if path == "bam":
                ctx.append_bam(raw, off)
            else:
                ctx.append_sam(b"\n".join(lines) + b"\n")
            assert ctx.n == len(keep) and ctx.n_filtered() == len(lines) - len(keep), (path, ctx.n, len(keep))
            assert ("bam_keep" in ctx.kernel_stats()) == bool(active), path
            idx, flag, out, o2 = _fetched(ctx)
            assert np.array_equal(idx, np.arange(len(keep))), path
            exp_flag = [struct.unpack_from("<H", recs[i], 18)[0] & (~0x400 if mask & _lib.FILTER_CLEAR_DUPLICATE_FLAG else 0xFFFF) for i in keep]
            assert flag.tolist() == exp_flag, path
            got = [bytes(out[int(o2[k]):int(o2[k + 1])]) for k in range(len(keep))]
            exp = [recs[i] if not mask & _lib.FILTER_CLEAR_DUPLICATE_FLAG else recs[i][:18] + struct.pack("<H", exp_flag[k]) + recs[i][20:]
                   for k, i in enumerate(keep)]
            assert [R.parse_bam(g).qname for g in got] == [R.parse_bam(recs[i]).qname for i in keep], path
            assert got == exp, path
        finally:
            ctx.close()
    return keep


# ---------------------------------------------------------------- target regions
def test_region_boundaries():
    cases = [(p, c) for p in (89, 90, 91, 92, 98, 99, 100, 101, 199, 200, 201, 202) for c in ("10M", "1M", "3S4M2D4M", "4M5I2M")]
    lines = [line(i, pos=p, cigar=c) for i, (p, c) in enumerate(cases)]
    lines += [line(len(lines) + k, flag=4, pos=p, cigar="500M") for k, p in enumerate((99, 100, 101, 200, 201))]   # placed unmapped: [POS, POS]
    lines += [line(len(lines) + k, pos=p, cigar="*") for k, p in enumerate((100, 101, 200, 201))]                  # no operations
    lines += [line(len(lines) + k, pos=p, cigar="5S3I") for k, p in enumerate((100, 101, 102, 201, 202))]          # I/S only: End() = POS - 1
    lines += [line(len(lines) + k, flag=4, rname="*", pos=0, cigar="*") for k in range(2)]                          # unplaced
    lines += [line(len(lines) + k, pos=p, cigar="10M", rname="c1") for k, p in enumerate((95, 150, 500))]           # c1 has no regions
    keep = check_filter(lines, R.remove_non_overlapping({0: [(100, 200)]}), _lib.FILTER_TARGET_REGIONS, regions={0: [[100, 200]]})
    assert 0 < len(keep) < len(lines)


def test_region_flattening_and_last_contig():
    raw_iv = [[500, 600], [100, 200], [100, 200], [120, 150], [200, 260], [261, 300], [700, 710], [705, 720]]
    flat = R.flatten_regions(raw_iv)
    assert flat == [(100, 260), (261, 300), (500, 600), (700, 720)]
    lines = [line(i, rname=rn, pos=p, cigar="10M") for i, (rn, p) in enumerate((rn, p) for rn in ("c0", "c2") for p in range(60, 760, 7))]
    check_filter(lines, R.remove_non_overlapping({2: flat}), _lib.FILTER_TARGET_REGIONS, regions={2: raw_iv})


def test_region_merge_decides():
    # contained and duplicated intervals where the binary search over the unmerged list lands on the inner interval and moves away from
    # the outer one: only the flattened list keeps these reads.  Regions [100, 200], [120, 150], [300, 400]: unmerged, a read at 160 meets
    # (120, 150) first, goes right to (300, 400) and is dropped; flattened to [100, 200], [300, 400] it overlaps.
    cases = [([[100, 200], [120, 150], [300, 400]], (160, 170, 190)),
             ([[300, 400], [100, 200], [100, 200], [120, 150], [130, 140], [500, 600]], (105, 160, 190, 395)),
             ([[10, 500], [20, 30], [40, 50], [60, 70], [700, 800]], (35, 55, 300, 490))]
    for raw_iv, poss in cases:
        flat = R.flatten_regions(raw_iv)
        unmerged = sorted(tuple(x) for x in raw_iv)
        lines = [line(i, pos=p, cigar="10M") for i, p in enumerate(poss)]
        recs = [R.parse_bam(sam_line_to_bam(x, H)) for x in lines]
        # the case must decide: the unmerged (sorted only) list drops a read the flattened one keeps
        assert any(R.remove_non_overlapping({0: flat})(r) and not R.remove_non_overlapping({0: unmerged})(r) for r in recs), raw_iv
        keep = check_filter(lines, R.remove_non_overlapping({0: flat}), _lib.FILTER_TARGET_REGIONS, regions={0: raw_iv})
        assert keep == list(range(len(lines))), raw_iv


def test_many_regions_every_search_depth():
    iv = [[10 + 50 * k, 20 + 50 * k] for k in range(5000)]          # 5000 disjoint regions on one contig: binary search depth 13
    rng = np.random.default_rng(4)
    rng.shuffle(iv)
    flat = R.flatten_regions(iv)
    hdr = sam.Header(sq=[{"SN": "c0", "LN": 1000}, {"SN": "c1", "LN": 300_000}], rg=H.RG)
    poss = [1, 5, 12, 20, 21, 29, 30, 31] + [10 + 50 * k + d for k in (1, 2, 2047, 2048, 2500, 4095, 4096, 4998, 4999) for d in (-9, -1, 0, 1, 10, 11, 12)]
    lines = [line(i, rname="c1", pos=p, cigar="10M") for i, p in enumerate(poss)]
    keep = check_filter(lines, R.remove_non_overlapping({1: flat}), _lib.FILTER_TARGET_REGIONS, regions={1: iv}, hdr=hdr)
    assert 10 < len(keep) < len(lines) - 10


def test_regions_replaced_between_appends_and_reset():
    lines = [line(i, pos=p) for i, p in enumerate(range(50, 400, 10))]
    recs, raw, off = _records(lines)
    ctx = _ctx(_lib.FILTER_TARGET_REGIONS, 0, {0: [[100, 150]]})
    try:
        exp = []
        for iv in ([[100, 150]], [[300, 320], [200, 210]], [[0, 1000]]):
            ctx.set_target_regions(0, np.array(iv, np.int32), already_flat=False)
            ctx.append_bam(raw, off)
            exp += [recs[i] for i, r in enumerate(recs) if R.remove_non_overlapping({0: R.flatten_regions(iv)})(R.parse_bam(r))]
        assert ctx.n == len(exp)
        _, _, out, o2 = _fetched(ctx)
        assert bytes(out) == b"".join(exp)
        ctx.reset()                                                   # the regions survive elp_reset, like the filter setting
        ctx.append_bam(raw, off)
        assert ctx.n == len(recs)
    finally:
        ctx.close()


def _raw(pos0, words, l_seq, qname=b"w"):
    body = struct.pack("<iiBBHHHiiii", 0, pos0, len(qname) + 1, 30, 0, len(words), 0, l_seq, -1, -1, 0) + qname + b"\0"
    body += struct.pack("<%dI" % len(words), *words) + b"\x11" * ((l_seq + 1) // 2) + b"\x1e" * l_seq
    return struct.pack("<I", len(body)) + body


def test_overlap_int32_wrap():
    # Overlap computes start - 1 and end - 1 in int32, and End() wraps: a read at POS -2^31 (BAM pos 2^31 - 1) whose D operations bring
    # End() back to 5, and a read whose End() passes 2^31 - 1.  Without the wrap both would overlap a region.
    big = (1 << 28) - 1
    recs = [_raw(INT32_MAX, [(1 << 4) | 0] + [(big << 4) | 2] * 8 + [(13 << 4) | 2], 1, b"a"),
            _raw(INT32_MAX - 5, [(10 << 4) | 0], 10, b"b"),
            _raw(149, [(10 << 4) | 0], 10, b"c")]
    parsed = [R.parse_bam(r) for r in recs]
    assert R.end(parsed[0]) == 5 and R.end(parsed[1]) == -(1 << 31) + 4
    iv = [(-5, 10), (100, 200), (INT32_MAX - 100, INT32_MAX)]
    exp = [i for i, r in enumerate(parsed) if R.remove_non_overlapping({0: iv})(r)]
    assert exp == [2]
    ctx = _ctx(_lib.FILTER_TARGET_REGIONS, 0, {0: iv})
    try:
        ctx.append_bam(np.frombuffer(b"".join(recs), np.uint8).copy())
        assert ctx.n == 1 and ctx.n_filtered() == 2
        _, _, out, _ = _fetched(ctx)
        assert bytes(out) == recs[2]
    finally:
        ctx.close()


# ---------------------------------------------------------------- MAPQ
@pytest.mark.parametrize("mq", [1, 254, 255, 256, INT32_MAX, 0, -1, -255, -256])
def test_mapq_threshold(mq):
    lines = [line(i, mapq=q) for i, q in enumerate((0, 1, 254, 255, 0, 255, 1, 254))]
    check_filter(lines, R.mapq_filter(mq) or (lambda r: True), 0, mq)


# ---------------------------------------------------------------- non-exact
def test_non_exact_ops():
    cigars = ["10M", "2M1I7M", "5M2D5M", "5M2N5M", "2S8M", "2H10M", "5M1P5M", "10=", "10X", "3S5M2S", "5M1X4M2S", "2S5=3M"]
    lines = [line(i, cigar=c) for i, c in enumerate(cigars)]
    keep = check_filter(lines, R.remove_non_exact, _lib.FILTER_NON_EXACT)
    assert [cigars[i] for i in keep] == ["10M", "2S8M", "3S5M2S"]


def test_non_exact_last_of_65535_ops():
    ops = "1M1S" * 32767 + "1M"
    lines = [line(0, cigar=ops, pos=1), line(1, cigar=ops[:-2] + "1X", pos=1), line(2, cigar="1I" + ops[2:], pos=1)]
    assert all(len(R.parse_bam(sam_line_to_bam(x, H)).cigar) == 65535 for x in lines)
    check_filter(lines, R.remove_non_exact, _lib.FILTER_NON_EXACT, paths=("bam",))


# ---------------------------------------------------------------- strict non-exact
def tag(name, ty, v):
    fmt = {"c": "<b", "C": "<B", "s": "<h", "S": "<H", "i": "<i", "I": "<I", "f": "<f"}
    if ty in fmt:
        return name + ty.encode() + struct.pack(fmt[ty], v)
    if ty == "A":
        return name + b"A" + bytes([v])
    if ty in "ZH":
        return name + ty.encode() + v + b"\0"
    sub, vals = ty[1], v                                             # "Bx"
    return name + b"B" + sub.encode() + struct.pack("<I", len(vals)) + struct.pack("<%d%s" % (len(vals), fmt[sub][1]), *vals)


GOOD = [(b"X0", 1), (b"X1", 0), (b"XM", 0), (b"XO", 0), (b"XG", 0)]


def _raw_lines(tag_blobs):
    """records with these optional-field bytes (built from a SAM line, the fields appended as raw BAM bytes)"""
    out = []
    for i, t in enumerate(tag_blobs):
        r = sam_line_to_bam(line(i), H) + t
        out.append(struct.pack("<I", len(r) - 4) + r[4:])
    return out


def check_raw(blobs, pred, mask, min_mapq=0):
    recs = _raw_lines(blobs)
    off = np.zeros(len(recs) + 1, np.uint64)
    np.cumsum([len(r) for r in recs], out=off[1:])
    keep = [i for i, r in enumerate(recs) if pred(R.parse_bam(r))]
    ctx = _ctx(mask, min_mapq, None)
    try:
        ctx.append_bam(np.frombuffer(b"".join(recs), np.uint8).copy(), off)
        assert ctx.n == len(keep) and ctx.n_filtered() == len(recs) - len(keep)
        _, _, out, _ = _fetched(ctx)
        assert bytes(out) == b"".join(recs[i] for i in keep)
    finally:
        ctx.close()
    return keep


def test_strict_integer_types_and_values():
    blobs, want = [], []
    for k, (name, good) in enumerate(GOOD):
        for ty in "cCsSiI":
            lim = {"c": (-128, 127), "C": (0, 255), "s": (-32768, 32767), "S": (0, 65535), "i": (-(1 << 31), INT32_MAX), "I": (0, (1 << 32) - 1)}[ty]
            for v in (0, 1, -1, 255, 65535, INT32_MAX, (1 << 32) - 1):
                if not lim[0] <= v <= lim[1]:
                    continue
                blobs.append(b"".join(tag(n, ty if n == name else "C", v if n == name else g) for n, g in GOOD))
                want.append(v == good)
    keep = check_raw(blobs, R.non_exact_strict, _lib.FILTER_NON_EXACT_STRICT)
    assert keep == [i for i, w in enumerate(want) if w]


def test_strict_repeats_types_positions():
    good = b"".join(tag(n, "C", g) for n, g in GOOD)
    blobs = [good,
             good + tag(b"X0", "C", 2), tag(b"X0", "C", 2) + good,                              # repeated: first occurrence counts
             good + tag(b"XM", "C", 0), tag(b"XG", "i", 5) + good]
    for n, _ in GOOD:                                                                           # each tag as f, A, Z, H, B: a mismatch
        for ty, v in (("f", 0.0), ("A", ord("0")), ("Z", b"0"), ("H", b"00"), ("Bc", [0]), ("Bi", [1])):
            blobs.append(b"".join(tag(m, ty, v) if m == n else tag(m, "C", g) for m, g in GOOD))
    for sub, vals in (("c", [1, -1]), ("C", [7]), ("s", [1, -300]), ("S", [65535]), ("i", [-5]), ("I", [7, 8]), ("f", [1.5])):
        blobs.append(tag(b"ZH", "H", b"0A1B") + tag(b"ZB", "B" + sub, vals) + good)                  # behind H strings and B arrays
        blobs.append(good[:-4] + tag(b"ZB", "B" + sub, vals) + good[-4:])                           # XG as the last field
    blobs += [tag(b"ZZ", "Z", b"X0C\x01") + good[4:],                                           # X0 only inside a Z value
              tag(b"x0", "C", 1) + good[4:]]                                                    # lowercase x0
    for k in range(5):                                                                          # one tag missing at a time
        blobs.append(b"".join(tag(n, "C", g) for j, (n, g) in enumerate(GOOD) if j != k))
    keep = check_raw(blobs, R.non_exact_strict, _lib.FILTER_NON_EXACT_STRICT)
    assert keep[:3] == [0, 1, 3] and len(keep) == 1 + 1 + 1 + 2 * 7


def test_strict_sam_text_matches_bam_types():
    good = b"X0:i:1\tX1:i:0\tXM:i:0\tXO:i:0\tXG:i:0"
    lines = [line(0, tags=good), line(1, tags=good.replace(b"X0:i:1", b"X0:i:2")), line(2, tags=good.replace(b"XM:i:0", b"XM:f:0")),
             line(3, tags=b"MD:Z:10\tAB:B:s,1,2\t" + good), line(4, tags=good.replace(b"XG:i:0", b"XG:Z:0")), line(5, tags=good + b"\tX0:i:3"),
             line(6, tags=good.replace(b"\tXO:i:0", b""))]
    keep = check_filter(lines, R.non_exact_strict, _lib.FILTER_NON_EXACT_STRICT)
    assert keep == [0, 3]                                              # SAM: a repeated tag replaces the value at its first position


# ---------------------------------------------------------------- unmapped, strict unmapped, duplicates
@pytest.mark.parametrize("extra", [0, _lib.FILTER_CLEAR_DUPLICATE_FLAG, _lib.FILTER_DUPLICATES])
def test_unmapped_clauses(extra):
    shapes = [(0, "c0", 100), (4, "c0", 100), (0, "c0", 0), (0, "*", 100), (4, "*", 0), (4, "c0", 0), (0, "*", 0), (0x404, "c0", 100),
              (0x400, "c0", 100), (0x400, "*", 0)]
    lines = [line(i, flag=f, rname=rn, pos=p, cigar="10M" if not f & 4 else "*") for i, (f, rn, p) in enumerate(shapes)]
    dup = (lambda r: True) if not extra & _lib.FILTER_DUPLICATES else R.remove_duplicates
    for mask, pred in ((_lib.FILTER_UNMAPPED, R.remove_unmapped), (_lib.FILTER_UNMAPPED_STRICT, R.remove_unmapped_strict),
                       (_lib.FILTER_UNMAPPED | _lib.FILTER_UNMAPPED_STRICT, R.remove_unmapped_strict)):
        check_filter(lines, lambda r, p=pred: p(r) and dup(r), mask | extra)


# ---------------------------------------------------------------- compaction
def test_compaction_edges():
    n = 700
    for name, drop in (("all", lambda i: True), ("first", lambda i: i == 0), ("last", lambda i: i == n - 1),
                       ("block edge", lambda i: 250 <= i < 262 or 508 <= i < 516), ("alternate", lambda i: i % 2 == 1)):
        lines = [line(i, flag=4 if drop(i) else 0, cigar="*" if drop(i) else "10M") for i in range(n)]
        keep = check_filter(lines, R.remove_unmapped, _lib.FILTER_UNMAPPED)
        assert keep == [i for i in range(n) if not drop(i)], name


def test_several_filtered_appends_then_fetch():
    ctx = _ctx(_lib.FILTER_UNMAPPED, 0, None)
    exp = []
    try:
        for call in range(5):
            lines = [line(1000 * call + i, flag=4 if (i * 7 + call) % 3 == 0 else 0) for i in range(300 + 37 * call)]
            recs, raw, off = _records(lines)
            ctx.append_bam(raw, off)
            exp += [r for r in recs if R.remove_unmapped(R.parse_bam(r))]
        assert ctx.n == len(exp)
        _, _, out, _ = _fetched(ctx)
        assert bytes(out) == b"".join(exp)
    finally:
        ctx.close()


def test_compaction_one_million_records():
    contigs = [("chr20", 2_000_000), ("chr21", 1_000_000)]
    w = synth.make_workload(500_000, contigs, seed=77, want_reference=False, unmapped_frac=0.05)
    raw, offs = synth.encode_bam(w.batch, w.header)
    b = w.batch
    assert b.n >= 1_000_000
    half = np.array([ln // 2 for _, ln in contigs], np.int32)
    # region [0, LN/2] per contig: [POS, End] overlaps iff POS <= LN/2 and End >= 1 (End = POS for unmapped reads; every mapped synthetic
    # read has M operations, so End >= POS)
    keep = (b.refid >= 0) & (b.pos >= 1) & (b.pos <= half[np.maximum(b.refid, 0)])
    assert 0.3 < keep.mean() < 0.7
    ctx = device.Context(w.header)
    try:
        for ci in range(len(contigs)):
            ctx.set_target_regions(ci, np.array([[0, half[ci]]], np.int32))
        ctx.set_ingest_filter(_lib.FILTER_TARGET_REGIONS, 0)
        ctx.append_bam(raw, offs)
        assert ctx.n == int(keep.sum()) and ctx.n_filtered() == b.n - int(keep.sum())
        _, _, out, o2 = _fetched(ctx)
        lens = np.diff(offs.astype(np.int64))
        assert np.array_equal(out, raw[np.repeat(keep, lens)])
        assert np.array_equal(np.diff(o2.astype(np.int64)), lens[keep])
    finally:
        ctx.close()


# ---------------------------------------------------------------- malformed records under filters
def _malformed():
    base = sam_line_to_bam(line(0, flag=0x404, mapq=0, cigar="5M1I4M", pos=900), H)   # unmapped, duplicate, MAPQ 0, non-exact, no X tags
    def with_tags(t):
        r = base + t
        return struct.pack("<I", len(r) - 4) + r[4:]
    lseq = bytearray(base); lseq[20:24] = struct.pack("<i", len(base))               # l_seq over block_size
    return {"l_seq": bytes(lseq), "B array": with_tags(b"ZBBs" + struct.pack("<I", 3) + struct.pack("<2h", 1, 2)),
            "type": with_tags(b"ZZq\x01"), "Z without NUL": with_tags(b"ZZZabc"),
            # well-formed, but beyond what the device holds: refused only in a record that passes the filters
            "RG:Z unknown": with_tags(b"RGZnone\0"), "CG:B": with_tags(b"CGBI" + struct.pack("<I", 1) + struct.pack("<I", (10 << 4) | 0))}


DROPPING = ((_lib.FILTER_UNMAPPED, 0), (_lib.FILTER_UNMAPPED_STRICT, 0), (_lib.FILTER_NON_EXACT, 0), (_lib.FILTER_DUPLICATES, 0),
            (_lib.FILTER_NON_EXACT_STRICT, 0), (_lib.FILTER_TARGET_REGIONS, 0), (0, 1), (0, 256))


@pytest.mark.parametrize("shape", ["l_seq", "B array", "type", "Z without NUL"])
def test_malformed_record_fails_under_every_filter(shape):
    bad = _malformed()[shape]
    with pytest.raises(R.Malformed):
        R.parse_bam(bad)
    good = sam_line_to_bam(line(1), H)
    raw = np.frombuffer(good + bad + good, np.uint8).copy()
    for mask, mq in ((0, 0),) + DROPPING:
        ctx = _ctx(mask, mq, {0: [[1, 10]]} if mask & _lib.FILTER_TARGET_REGIONS else None)
        try:
            with pytest.raises(device.ElprepError) as e:
                ctx.append_bam(raw)
            assert e.value.code == _lib.EBAM, (shape, mask, mq, str(e.value))
            assert ctx.n == 0 and ctx.n_filtered() == 0, (shape, mask, mq)
        finally:
            ctx.close()


@pytest.mark.parametrize("shape,code", [("RG:Z unknown", _lib.EBAM), ("CG:B", _lib.ELIMIT)])
def test_device_limits_only_in_kept_records(shape, code):
    rec = _malformed()[shape]
    R.parse_bam(rec)                                                  # well-formed: the reference reads it
    good = sam_line_to_bam(line(1), H)
    raw = np.frombuffer(good + rec + good, np.uint8).copy()
    ctx = _ctx(0, 0, None)
    try:
        with pytest.raises(device.ElprepError) as e:
            ctx.append_bam(raw)
        assert e.value.code == code and ctx.n == 0, str(e.value)
    finally:
        ctx.close()
    preds = {_lib.FILTER_UNMAPPED: R.remove_unmapped, _lib.FILTER_UNMAPPED_STRICT: R.remove_unmapped_strict, _lib.FILTER_NON_EXACT: R.remove_non_exact,
             _lib.FILTER_DUPLICATES: R.remove_duplicates, _lib.FILTER_NON_EXACT_STRICT: R.non_exact_strict,
             _lib.FILTER_TARGET_REGIONS: R.remove_non_overlapping({0: [(1, 10)]})}
    for mask, mq in DROPPING:                                         # dropped by the filter: the call gives the reference's result
        ctx = _ctx(mask, mq, {0: [[1, 10]]} if mask & _lib.FILTER_TARGET_REGIONS else None)
        try:
            ctx.append_bam(raw)
            pred = preds[mask] if mask else R.mapq_filter(mq)
            exp = [x for x in (good, rec, good) if pred(R.parse_bam(x))]
            assert rec not in exp
            assert ctx.n == len(exp) and ctx.n_filtered() == 3 - len(exp), (shape, mask, mq)
            _, _, out, _ = _fetched(ctx)
            assert bytes(out) == b"".join(exp)
        finally:
            ctx.close()


# ---------------------------------------------------------------- CleanSam on the device
CLEAN_CASES = [("100M", 951), ("100M", 901), ("100M", 902), ("10M20I10M", 988), ("5S100M", 951), ("5S100M", 996), ("10M20I70M", 990),
               ("100=", 951), ("30M70X", 951), ("10M10I10M10I10M", 975), ("10M10D10M10I10M", 965), ("50M10D50M", 949), ("10M10I10D100M", 970),
               ("5D100M", 1000), ("5D100M", 999), ("100M", 1100), ("100M", 1200), ("10M", 500), ("3S20M4I20M3S", 985)]


def _clean_expect(recs, lengths=(1000, 1000, 1000)):
    out = []
    for r in recs:
        cg, mq, rw = R.clean_sam(r, list(lengths))
        out.append((R.cigar_words(cg), mq, rw))
    return out


def _device_cigars(ctx):
    off, cg = ctx.debug_cigar()
    return [[int(x) for x in cg[int(off[i]):int(off[i + 1])]] for i in range(ctx.n)]


def _clean_lines(cases, start=0):
    return [line(start + i, pos=p, cigar=c, flag=16 * (i & 1)) for i, (c, p) in enumerate(cases)]


def test_clean_sam_clip_points_single_and_straddling():
    rng = np.random.default_rng(8)
    single = _clean_lines(CLEAN_CASES) + [line(100, rname="*", pos=5, cigar="10M")]           # RNAME * with FLAG 0x4 clear: length 0
    runs = []
    for k in range(900):                                                                      # rewrites across 256-thread block edges
        c, p = CLEAN_CASES[int(rng.integers(len(CLEAN_CASES)))] if rng.random() < 0.6 else ("4M2I4M", int(rng.integers(1, 900)))
        runs.append(line(200 + k, pos=p, cigar=c))
    for lines in (single, runs):
        recs, raw, off = _records(lines)
        parsed = [R.parse_bam(r) for r in recs]
        exp = _clean_expect(parsed)
        assert any(len(e[0]) > len(p.cigar) for e, p in zip(exp, parsed)) and any(len(e[0]) < len(p.cigar) for e, p in zip(exp, parsed))
        for path in ("bam", "sam"):
            ctx = device.Context(H)
            try:
                ctx.append_bam(raw, off) if path == "bam" else ctx.append_sam(b"\n".join(lines))
                n_rw = ctx.clean_sam()
                assert n_rw == sum(e[2] for e in exp)
                assert _device_cigars(ctx) == [e[0] for e in exp], path
            finally:
                ctx.close()


@pytest.mark.parametrize("cigar,pos", [("10M10I10D100M", 975), ("10M10I10N100M", 975), ("10D100M", 1100), ("10N100M", 1100)])
def test_clean_sam_panic_text(cigar, pos):
    with pytest.raises(R.CleanSamPanic):
        R.clean_sam(R.Rec(refid=0, pos=pos, cigar=R.parse_cigar(cigar)), [1000])
    ctx = device.Context(H)
    try:
        ctx.append_bam(np.frombuffer(sam_line_to_bam(line(0, pos=pos, cigar=cigar), H) + sam_line_to_bam(line(1), H), np.uint8).copy())
        with pytest.raises(device.ElprepError, match="Unexpected non-0 relative clipping position in CleanSam."):
            ctx.clean_sam()
    finally:
        ctx.close()


def test_clean_sam_twice_mixed_appends_and_reset():
    lines = _clean_lines(CLEAN_CASES)
    recs, raw, off = _records(lines)
    parsed = [R.parse_bam(r) for r in recs]
    once = _clean_expect(parsed)
    twice = _clean_expect([R.Rec(refid=p.refid, pos=p.pos, flag=p.flag, mapq=e[1], cigar=R.cigar_from_words(e[0])) for p, e in zip(parsed, once)])
    batch = sam.AlignmentBatch.from_records(H, [dict(QNAME=f"c{i}", FLAG=0, RNAME="c0", POS=p, MAPQ=30, CIGAR=c, SEQ="A" * R.read_length(R.parse_cigar(c)),
                                                     QUAL="I" * R.read_length(R.parse_cigar(c))) for i, (c, p) in enumerate(CLEAN_CASES)])
    ctx = device.Context(H)
    try:
        ctx.append_bam(raw, off)
        assert ctx.clean_sam() == sum(e[2] for e in once)
        ctx.clean_sam()
        assert _device_cigars(ctx) == [e[0] for e in twice]
        ctx.reset()
        ctx.append_bam(raw, off); ctx.append_sam(b"\n".join(lines)); ctx.append(batch)          # BAM, SAM and columns in one context
        ctx.clean_sam()
        assert _device_cigars(ctx) == [e[0] for e in once] * 3
    finally:
        ctx.close()


# ---------------------------------------------------------------- MAPQ after CleanSam in the byte outputs
@pytest.mark.parametrize("path", ["bam", "sam"])
@pytest.mark.parametrize("clean", [False, True])
@pytest.mark.parametrize("fields", [False, True])
def test_mapq_after_clean_sam(path, clean, fields):
    lines = [line(0, flag=4, mapq=7, cigar="10M", tags=b"XX:i:5"), line(1, flag=4, mapq=255, pos=200, cigar="*", tags=b"XX:i:5"),
             line(2, mapq=30, tags=b"XX:i:5"), line(3, flag=0x45, mapq=255, tags=b"XX:i:5\tYY:Z:a"), line(4, mapq=0, tags=b"XX:i:5")]
    recs, raw, off = _records(lines)
    ctx = device.Context(H)
    try:
        ctx.append_bam(raw, off) if path == "bam" else ctx.append_sam(b"\n".join(lines) + b"\n")
        if clean:
            assert ctx.clean_sam() == 0                                          # nothing runs past its contig: no CIGAR rewrite
        if fields:
            ctx.set_output_filter(0, remove=["XX"])
        ctx.sort_markdup(device.SO_KEEP, False)
        out, o2 = ctx.fetch_bam()
        txt, _ = ctx.fetch_sam()
        got = [bytes(out[int(o2[k]):int(o2[k + 1])]) for k in range(len(recs))]
        for k, r in enumerate(recs):
            p = R.parse_bam(r)
            mq = 0 if clean and p.flag & 4 else p.mapq
            assert got[k][13] == mq, (k, got[k][13], mq)
            if fields:                                                           # the fields path: XX dropped, everything else as stored
                q = R.parse_bam(got[k])
                assert q.tags == [t for t in p.tags if t[0] != b"XX"] and (q.refid, q.pos, q.flag, q.cigar, q.qname) == (p.refid, p.pos, p.flag, p.cigar, p.qname)
            else:
                assert got[k] == r[:13] + bytes([mq]) + r[14:], k
        cols = [ln.split(b"\t") for ln in bytes(txt).split(b"\n")[:-1]]
        assert [int(c[4]) for c in cols] == [0 if clean and f & 4 else m for f, m in ((4, 7), (4, 255), (0, 30), (0x45, 255), (0, 0))]
        if not clean and not fields:
            assert bytes(out) == b"".join(recs)
    finally:
        ctx.close()


# ---------------------------------------------------------------- the full path after CleanSam, against the oracle
def test_full_path_after_clean_sam_matches_oracle():
    from util import gpu_phases, oracle_pipeline, set_side_inputs
    contigs = [("chr20", 300_000), ("chr21", 200_000)]
    w = synth.make_workload(6000, contigs, seed=43)
    b = w.batch.copy()
    rng = np.random.default_rng(6)
    clen = np.array([ln for _, ln in contigs])
    sel = rng.choice(b.n, 600, replace=False)
    ok = sel[b.refid[sel] >= 0]
    b.pos[ok] = (clen[b.refid[ok]] - rng.integers(0, 160, ok.size)).astype(np.int32)
    # the restatement's cleaned batch for the oracle
    co = b.cigar_off.astype(np.int64)
    new, mapq, n_incons = [], b.mapq.copy(), 0
    for i in range(b.n):
        rec = R.Rec(refid=int(b.refid[i]), pos=int(b.pos[i]), flag=int(b.flag[i]), mapq=int(b.mapq[i]), cigar=R.cigar_from_words(b.cigar[co[i]:co[i + 1]]))
        cg, mq, rw = R.clean_sam(rec, list(clen))
        new.append(R.cigar_words(cg)); mapq[i] = mq
        n_incons += rw and R.read_length(cg) != int(b.lseq[i])
    assert n_incons > 50                                            # rewritten CIGARs whose read length is not l_seq
    cleaned = b.copy()
    cleaned.cigar = np.array([x for c in new for x in c], np.uint32)
    cleaned.cigar_off = np.concatenate([[0], np.cumsum([len(c) for c in new])]).astype(np.uint64)
    cleaned.mapq = mapq
    o = oracle_pipeline(synth.Workload(w.header, cleaned, w.contig_bases, w.sites, w.params))
    # of those, the reads recalibrateAln would take but for the CIGAR check (bqsr.go:225-244, on the FLAG after marking): the gather must
    # skip them, as the oracle's recalibrate_aln does
    f = np.empty_like(o["flag"]); f[o["perm"].astype(np.int64)] = o["flag"]
    elig = ((cleaned.opt_flags & 1) == 0) & (cleaned.mapq > 0) & (cleaned.mapq < 255) & ((f & (0x4 | 0x100 | 0x200 | 0x400)) == 0) & \
           (cleaned.refid >= 0) & (cleaned.pos > 0) & (cleaned.lseq > 0) & (cleaned.rg >= 0) & (cleaned.pos <= clen[np.maximum(cleaned.refid, 0)])
    rl = np.array([R.read_length(R.cigar_from_words(c)) for c in new])
    assert int((elig & (rl != cleaned.lseq)).sum()) > 20
    ctx = device.Context(w.header)
    try:
        set_side_inputs(ctx, w)
        ctx.append(b)
        ctx.clean_sam()
        off, cg = ctx.debug_cigar()
        assert np.array_equal(off, cleaned.cigar_off) and np.array_equal(cg, cleaned.cigar)
        g = gpu_phases(ctx, markdup=_lib.MARKDUP_OPTICAL)
    finally:
        ctx.close()
    from util import oracle_tables_dense
    assert np.array_equal(g["perm"], o["perm"]) and np.array_equal(g["flag"], o["flag"])
    d, e = oracle_tables_dense(o["tables"])
    assert np.array_equal(g["tables"], d) and np.array_equal(g["emp"], e)
    assert np.array_equal(g["qual"], o["qual"])
