"""The remaining per-record filters of SURVEY.md 8f row 4 against direct restatements of the reference functions:
RemoveNonExactMappingReadsStrict (filters/simple-filters.go:115-136), RemoveNonOverlappingReads (:310-328, intervals.Overlap
intervals/intervals.go:146-164) fused into elp_append_bam, and CleanSam (:292-306, softClipEndOfRead filters/utils.go:82-119) on the device."""
import struct

import numpy as np
import pytest

from elprep_b200 import device, filters, synth, _lib
from ingestfilter_ref import clean_cigar as _ref_clean_cigar
from util import encode_bam

pytestmark = pytest.mark.gpu
SMALL = [("chr20", 300_000), ("chr21", 200_000)]


def test_clean_sam_matches_reference_rule():
    w = synth.make_workload(3000, SMALL, seed=41, want_reference=False)
    b = w.batch.copy()
    # push a few hundred reads against / past the end of their contig
    rng = np.random.default_rng(3)
    sel = rng.choice(b.n, 400, replace=False)
    clen = np.array([ln for _, ln in SMALL])
    ok = b.refid[sel] >= 0
    b.pos[sel[ok]] = (clen[b.refid[sel[ok]]] - rng.integers(0, 160, ok.sum())).astype(np.int32)
    ctx = device.Context(w.header)
    ctx.append(b)
    changed = ctx.clean_sam()
    off, cg = ctx.debug_cigar()
    co = b.cigar_off.astype(np.int64)
    n_exp = 0
    for i in range(b.n):
        ops = [int(x) for x in b.cigar[co[i]:co[i + 1]]]
        unm = bool(b.flag[i] & 4)
        length = int(clen[b.refid[i]]) if b.refid[i] >= 0 else 0
        exp = _ref_clean_cigar(ops, int(b.pos[i]), length, unm)
        got = [int(x) for x in cg[int(off[i]):int(off[i + 1])]]
        assert got == exp, (i, ops, got, exp)
        n_exp += exp != ops or (not unm and int(b.pos[i]) + sum((o >> 4) for o in ops if (o & 15) in (0, 2, 3, 7, 8)) - 1 > length)
    assert changed == n_exp and changed > 50
    # the pipeline still runs on the cleaned reads
    ctx.sort_markdup(device.SO_COORDINATE, True)
    ctx.close()


def test_strict_exact_and_target_regions_on_bam_ingest():
    w = synth.make_workload(4000, SMALL, seed=42, want_reference=False)
    b = w.batch
    rng = np.random.default_rng(9)
    tags, exact = [], np.zeros(b.n, bool)
    for i in range(b.n):
        k = int(rng.integers(0, 6))
        t = b""
        if k == 0:                      # all five present and right, in mixed integer types
            t = b"X0C" + struct.pack("<B", 1) + b"X1c" + struct.pack("<b", 0) + b"XMS" + struct.pack("<H", 0) + b"XOi" + struct.pack("<i", 0) + b"XGI" + struct.pack("<I", 0); exact[i] = True
        elif k == 1:                    # XM wrong
            t = b"X0C\x01X1C\x00XMC\x02XOC\x00XGC\x00"
        elif k == 2:                    # XG missing
            t = b"X0C\x01X1C\x00XMC\x00XOC\x00"
        elif k == 3:                    # X0 != 1
            t = b"X0C\x02X1C\x00XMC\x00XOC\x00XGC\x00"
        elif k == 4:                    # behind a string and an array tag
            t = b"MDZ" + b"10A5\0" + b"ZBBs" + struct.pack("<I", 2) + struct.pack("<2h", 1, -1) + b"X0C\x01X1C\x00XMC\x00XOC\x00XGC\x00"; exact[i] = True
        tags.append(t)
    raw, offs = encode_bam(b, w.header, rng=np.random.default_rng(1), with_aux=False, extra_tags=tags)
    regions = [np.array([[1000, 5000], [4000, 9000], [100_000, 100_500], [250_000, 299_000]], np.int32), np.array([[50_000, 60_000]], np.int32)]
    flt = filters.RemoveNonOverlappingReads(regions)(w.header)
    kept_regions = set(map(int, np.nonzero(np.isin(np.arange(b.n), _kept_indices(flt, b)))[0]))
    for mask, expect in ((_lib.FILTER_NON_EXACT_STRICT, set(map(int, np.nonzero(exact)[0]))), (_lib.FILTER_TARGET_REGIONS, kept_regions),
                         (_lib.FILTER_NON_EXACT_STRICT | _lib.FILTER_TARGET_REGIONS, set(map(int, np.nonzero(exact)[0])) & kept_regions)):
        ctx = device.Context(w.header)
        for ci, iv in enumerate(regions):
            ctx.set_target_regions(ci, iv)
        ctx.set_ingest_filter(mask, 0)
        ctx.append_bam(raw, offs)
        assert ctx.n == len(expect) and ctx.n_filtered() == b.n - len(expect)
        # which reads arrived: compare QNAME+FLAG multiset through the output of an unsorted fetch
        ctx.sort_markdup(device.SO_KEEP, False)
        idx, flag, _, _ = ctx.fetch(want_qual=False)
        assert np.array_equal(np.sort(flag), np.sort(b.flag[sorted(expect)]))
        ctx.close()


def _kept_indices(flt, batch):
    """indices of the reads a column filter keeps (the filter returns the filtered batch; reads are identified by position)"""
    tagged = batch.copy()
    tagged.tlen = np.arange(batch.n, dtype=np.int32)          # carry the index through the filter in a column it does not look at
    return flt(tagged).tlen
