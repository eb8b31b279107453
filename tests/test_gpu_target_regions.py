"""elp_filter_target_regions (`--target-regions`: RemoveNonOverlappingReads after duplicate marking, before the BQSR gather) against the
reference's order composed in tests/targetregions_ref.py: oracle marking and sort over every read, the restated predicate over the output
order, the oracle gather / finalize / apply over the kept reads.  Each case compares the output permutation, FLAG, elp_n_sorted, the number
removed, table counters, EmpiricalQuality, report text and QUAL bytes, and the BAM / SAM bytes where the reads came in as records."""
import os
import tempfile

import numpy as np
import pytest

import ingestfilter_ref as R
import targetregions_ref as T
from elprep_b200 import _lib, device, sam, synth
from util import bqsr_paths, encode_bam, oracle_tables_dense, set_side_inputs

pytestmark = pytest.mark.gpu
CONTIGS = [("chr20", 300_000), ("chr21", 150_000)]
SORTS = {"coordinate": device.SO_COORDINATE, "queryname": _lib.SO_QUERYNAME, "keep": device.SO_KEEP}
NEW_KERNELS = ("target_keep", "target_compact", "target_pack_rows", "target_gather_cols", "target_summary")


@pytest.fixture(scope="module")
def exome():
    return synth.make_workload(3000, CONTIGS, seed=11, exome=True)


def _set_regions(ctx, regions, already_flat=False):
    for ci, iv in regions.items():
        ctx.set_bqsr_target_regions(ci, np.asarray(iv, np.int32).reshape(-1, 2), already_flat=already_flat)


def run(w, regions, sort="coordinate", markdup=True, bqsr=True, max_cycle=500, batch=None, filt=True, already_flat=False, mark=None):
    """device: append, sort + mark, [set regions + filter], gather, finalize, apply, fetch -> dict like targetregions_ref.mark_then_filter"""
    ctx = device.Context(w.header, max_cycle=max_cycle, profile=True)
    try:
        if bqsr:
            set_side_inputs(ctx, w)
        ctx.append(batch if batch is not None else w.batch)
        ctx.sort_markdup(SORTS[sort], mark if mark is not None else int(markdup))
        res = {}
        if filt:
            _set_regions(ctx, regions, already_flat)
            res["n_removed"] = ctx.filter_target_regions()
        res["n_sorted"] = ctx.n_sorted
        assert ctx.n == (batch if batch is not None else w.batch).n
        if bqsr:
            ctx.bqsr_gather()
            res["tables"] = ctx.tables_get()
            with tempfile.TemporaryDirectory() as d:
                p = os.path.join(d, "g.recal")
                ctx.bqsr_finalize(p)
                res["report"] = open(p).read()
            res["emp"] = ctx.empirical_get()
            ctx.bqsr_apply()
        idx, flag, qoff, qual = ctx.fetch()
        res.update(perm=idx, flag=flag, qual_off=qoff, qual=qual[:int(qoff[-1])], stats=ctx.kernel_stats())
        return res
    finally:
        ctx.close()


def compare(g, o, bqsr=True, max_cycle=500):
    assert g["n_removed"] == o["n_removed"] and g["n_sorted"] == o["perm"].size
    assert np.array_equal(g["perm"], o["perm"]), "output order differs"
    assert np.array_equal(g["flag"], o["flag"]), "FLAG differs"
    assert np.array_equal(g["qual_off"], o["qual_off"])
    if bqsr:
        d, e = oracle_tables_dense(o["tables"], max_cycle)
        assert np.array_equal(g["tables"], d), "BQSR table counters differ"
        assert np.array_equal(g["emp"], e), "EmpiricalQuality differs"
        assert g["report"] == o["report"], "recalibration report text differs"
    assert np.array_equal(g["qual"], o["qual"]), "QUAL bytes differ"


def _regions(pad, contigs=(0, 1)):
    ex = synth.exome_regions(CONTIGS, seed=11, pad=pad)
    return {c: ex[c] for c in contigs}


# ---------------------------------------------------------------- full paths against the reference order
@pytest.mark.parametrize("sort", ["coordinate", "queryname", "keep"])
@pytest.mark.parametrize("pad", [0, 150])
def test_exome_full_path(exome, sort, pad):
    regions = _regions(pad)
    g = run(exome, regions, sort=sort)
    o = T.mark_then_filter(exome, regions, sort=sort)
    assert 0 < o["n_removed"] < exome.batch.n
    compare(g, o)
    assert all(k in g["stats"] for k in ("target_keep", "target_compact", "target_summary")), sorted(g["stats"])


def test_regions_on_last_contig_only_and_unsorted_overlapping_lists(exome):
    ex = synth.exome_regions(CONTIGS, seed=11, pad=40)[1]
    # the same regions given unsorted, split into overlapping pieces: flattened inside to the same set
    pieces = np.concatenate([np.stack([ex[:, 0], ex[:, 0] + 200], 1), np.stack([ex[:, 0] + 150, ex[:, 1]], 1)])[::-1]
    o = T.mark_then_filter(exome, {1: ex})
    compare(run(exome, {1: pieces}), o)
    compare(run(exome, {1: ex}, already_flat=True), o)


def test_5000_regions_on_one_contig(exome):
    rng = np.random.default_rng(3)
    s = np.sort(rng.choice(np.arange(0, 300_000, 60), 5000, replace=False)).astype(np.int64)
    iv = np.stack([s, s + 20], 1)
    compare(run(exome, {0: iv}, already_flat=True), T.mark_then_filter(exome, {0: iv}))


# ---------------------------------------------------------------- predicate edges on hand-built reads, through BAM and SAM bytes
H = sam.Header(sq=[{"SN": "c0", "LN": 1000}, {"SN": "c1", "LN": 1000}], rg=[{"ID": "g1", "LB": "l1"}])


def _rec(name, pos, cigar="10M", flag=0, rname="c0"):
    n = R.read_length(R.parse_cigar(cigar)) if cigar != "*" else 10
    n = n or 10
    return dict(QNAME=name, FLAG=flag, RNAME=rname, POS=pos, MAPQ=30, CIGAR=cigar, RNEXT="*", PNEXT=0, SEQ="ACGT" * (n // 4) + "ACGT"[:n % 4],
                QUAL=[30] * n, RG="g1")


EDGE_RECS = [_rec("a", 90), _rec("b", 91), _rec("c", 92), _rec("d", 200), _rec("e", 201), _rec("f", 150, flag=4), _rec("g", 100, flag=4),
             _rec("h", 150, rname="*", flag=4), _rec("i", 150, cigar="*"), _rec("j", 150, cigar="4H"), _rec("k", 95, cigar="2S3M20D3M"),
             _rec("l", 150, rname="c1"), _rec("m", 991, cigar="15M")]


def test_predicate_edges_bam_and_sam_bytes():
    b = sam.AlignmentBatch.from_records(H, EDGE_RECS)
    regions = {0: [(100, 200), (1000, 1010)]}
    w = type("W", (), {"header": H})()
    o = T.mark_then_filter(w, regions, sort="coordinate", markdup=True, bqsr=False, batch=b)
    raw, off = encode_bam(b, H)
    for path in ("bam", "sam"):                       # the records as elp_fetch_bam and as elp_fetch_sam write them
        outs = []
        for filt in (False, True):
            ctx = device.Context(H, profile=True)
            try:
                ctx.append_bam(raw, off)
                ctx.sort_markdup(device.SO_COORDINATE, 1)
                if filt:
                    _set_regions(ctx, regions)
                    assert ctx.filter_target_regions() == o["n_removed"]
                idx, flag, _, _ = ctx.fetch(want_qual=False)
                by, bo = ctx.fetch_bam() if path == "bam" else ctx.fetch_sam()
                outs.append((idx, flag, by, bo, ctx.n_output(), ctx.n_sorted))
            finally:
                ctx.close()
        (i0, f0, b0, o0, n0, s0), (i1, f1, b1, o1, n1, s1) = outs
        assert np.array_equal(i1, o["perm"]) and np.array_equal(f1, o["flag"]) and s1 == n1 == o["perm"].size and s0 == n0 == b.n
        keep = np.nonzero(o["keep"])[0]
        assert [bytes(b1[int(o1[k]):int(o1[k + 1])]) for k in range(keep.size)] == [bytes(b0[int(o0[k]):int(o0[k + 1])]) for k in keep], path


def test_cigar_rewritten_by_clean_sam_counts():
    # "m" runs past c0's end: CleanSam soft-clips it to [991, 1000], which ends on the region start 1000 -- no longer an overlap
    b = sam.AlignmentBatch.from_records(H, EDGE_RECS)
    regions = {0: [(100, 200), (1000, 1010)]}
    ctx = device.Context(H)
    try:
        ctx.append(b)
        assert ctx.clean_sam() == 1
        ctx.sort_markdup(device.SO_COORDINATE, 1)
        _set_regions(ctx, regions)
        ctx.filter_target_regions()
        idx, flag, _, _ = ctx.fetch(want_qual=False)
    finally:
        ctx.close()
    cb = b.copy()
    co = cb.cigar_off.astype(np.int64)
    words = [R.clean_cigar(cb.cigar[co[i]:co[i + 1]].tolist(), int(cb.pos[i]), 1000, bool(cb.flag[i] & 4)) if cb.refid[i] == 0 else cb.cigar[co[i]:co[i + 1]].tolist()
             for i in range(cb.n)]
    cb = sam.AlignmentBatch(**{**{f: getattr(cb, f) for f in sam.AlignmentBatch.FIELDS}, "cigar": np.array(sum(words, []), np.uint32),
                               "cigar_off": np.concatenate([[0], np.cumsum([len(x) for x in words])]).astype(np.uint64)})
    w = type("W", (), {"header": H})()
    o = T.mark_then_filter(w, regions, bqsr=False, batch=cb)
    assert np.array_equal(idx, o["perm"]) and np.array_equal(flag, o["flag"])
    assert 12 not in idx.tolist()


# ---------------------------------------------------------------- marking before filtering
def test_marking_sees_every_read_and_metrics_stay(exome):
    regions = _regions(0)
    ctx = device.Context(exome.header, profile=True)
    try:
        ctx.append(exome.batch)
        ctx.sort_markdup(device.SO_COORDINATE, _lib.MARKDUP_OPTICAL)
        before = ctx.optical_metrics()
        with tempfile.TemporaryDirectory() as d:
            ctx.print_duplicates_metrics(os.path.join(d, "a"), "cmd", "t0")
            _set_regions(ctx, regions)
            ctx.filter_target_regions()
            ctx.print_duplicates_metrics(os.path.join(d, "b"), "cmd", "t0")
            assert open(os.path.join(d, "a")).read() == open(os.path.join(d, "b")).read()
        assert repr(ctx.optical_metrics()) == repr(before)          # (repr: percent_duplication may be NaN)
        idx, flag, _, _ = ctx.fetch(want_qual=False)
    finally:
        ctx.close()
    o = T.mark_then_filter(exome, regions, bqsr=False)
    assert np.array_equal(idx, o["perm"]) and np.array_equal(flag, o["flag"])
    # the ingest filter's order gives other FLAGs on this workload: pairs with one mate off target
    i2, f2 = T.ingest_then_mark(exome.header, exome.batch, regions)
    common = np.intersect1d(i2, o["perm"])
    fa = dict(zip(o["perm"].tolist(), o["flag"].tolist())); fb = dict(zip(i2.tolist(), f2.tolist()))
    assert any(fa[k] != fb[k] for k in common.tolist())


def test_ingest_and_target_regions_in_one_context(exome):
    ingest = _regions(400)                              # --filter-non-overlapping-reads A.bed
    target = _regions(0)                                # --target-regions B.bed
    raw, off = encode_bam(exome.batch, exome.header)
    ctx = device.Context(exome.header)
    try:
        for ci, iv in ingest.items():
            ctx.set_target_regions(ci, iv)
        ctx.set_ingest_filter(_lib.FILTER_TARGET_REGIONS)
        ctx.append_bam(raw, off)
        ctx.sort_markdup(device.SO_COORDINATE, 1)
        _set_regions(ctx, target)
        nr = ctx.filter_target_regions()
        idx, flag, _, _ = ctx.fetch(want_qual=False)
    finally:
        ctx.close()
    first = np.nonzero(T.keep_mask(exome.batch, ingest))[0]
    o = T.mark_then_filter(exome, target, bqsr=False, batch=exome.batch.take(first))
    assert nr == o["n_removed"] > 0
    assert np.array_equal(idx, o["perm"]) and np.array_equal(flag, o["flag"])


# ---------------------------------------------------------------- order and write phase
def test_write_phase_filters_and_uneven_fetch_ranges(exome):
    regions = _regions(50)
    raw, off = encode_bam(exome.batch, exome.header)
    o = T.mark_then_filter(exome, regions, bqsr=False)
    ctx = device.Context(exome.header)
    try:
        ctx.append_bam(raw, off)
        ctx.sort_markdup(device.SO_COORDINATE, 1)
        ctx.set_output_filter(_lib.OUT_REMOVE_DUPLICATES, remove=["NM"])
        n_out0 = ctx.n_output()
        _set_regions(ctx, regions)
        ctx.filter_target_regions()
        nd = int(((o["flag"] & 0x400) == 0).sum())
        assert ctx.n_output() == nd and n_out0 > nd
        whole, woff = ctx.fetch_bam()
        parts, k = [], 0
        for step in (1, 7, 300, 10 ** 9):
            m = min(step, nd - k)
            if m <= 0:
                break
            p, _ = ctx.fetch_bam(k, m)
            parts.append(bytes(p)); k += m
        assert b"".join(parts) == bytes(whole)
        i1, f1, _, _ = ctx.fetch(0, 5, want_qual=False)
        i2, f2, _, _ = ctx.fetch(5, ctx.n_sorted - 5, want_qual=False)
        assert np.array_equal(np.concatenate([i1, i2]), o["perm"]) and np.array_equal(np.concatenate([f1, f2]), o["flag"])
        with pytest.raises(device.ElprepError):
            ctx.fetch(0, ctx.n_sorted + 1, want_qual=False)
        s, soff = ctx.fetch_sam()
        assert soff.size == nd + 1
    finally:
        ctx.close()
    rows = [bytes(whole[int(woff[k]):int(woff[k + 1])]) for k in range(nd)]
    assert [r[36:36 + r[12] - 1] for r in rows] == [bytes(exome.batch.qname[int(exome.batch.qname_off[i]):int(exome.batch.qname_off[i + 1])])
                                                    for i, f in zip(o["perm"], o["flag"]) if not f & 0x400]


# ---------------------------------------------------------------- dropped reads must not matter
def _extras(w, recs):
    """a copy of w's reads with extra unpaired reads on the second contig (which gets no regions) appended"""
    return sam.AlignmentBatch.concat([w.batch, sam.AlignmentBatch.from_records(w.header, recs)])


def _extra(name, pos, L, q=30, quals=None):
    qual = quals if quals is not None else [q] * L
    return dict(QNAME=name, FLAG=0, RNAME="chr21", POS=pos, MAPQ=60, CIGAR=f"{L}M", RNEXT="*", PNEXT=0, SEQ="ACGT" * (L // 4) + "ACGT"[:L % 4],
                QUAL=qual, RG=None)


@pytest.mark.parametrize("case", ["long_2000", "qual_alphabet", "past_max_cycle", "past_contig_end", "qual_above_93"])
def test_dropped_reads_do_not_matter(case):
    w = synth.make_workload(1500, CONTIGS, seed=5, L=150)
    rg = w.header.RG[0]["ID"]
    max_cycle, markdup = 500, True
    if case == "long_2000":
        # kept reads of 500 bases: the general gather kernels stop at 512 bases per read (bqsr_gather.cu MAXIT); one read group keeps
        # their compact apply table in shared memory
        recs = [_extra("x", 5000, 2000)]
        w = synth.make_workload(1500, CONTIGS, seed=5, L=500, n_rg=1)
    elif case == "qual_alphabet":
        recs = [_extra("x", 5000, 150, q=50), _extra("y", 6000, 150, q=60)]
    elif case == "past_max_cycle":
        max_cycle, recs = 200, [_extra("x", 5000, 300)]
    elif case == "past_contig_end":
        recs = [_extra("x", 150_000 - 20, 150)]
    else:
        markdup, recs = False, [_extra("x", 5000, 150, q=100)]
    for r in recs:
        r["RG"] = rg
    batch = _extras(w, recs)
    regions = {0: np.array([[0, 300_001]], np.int32)}        # every read on chr20; nothing on chr21
    o = T.mark_then_filter(w, regions, markdup=markdup, max_cycle=max_cycle, batch=batch)
    g = run(w, regions, markdup=markdup, max_cycle=max_cycle, batch=batch)
    compare(g, o, max_cycle=max_cycle)
    clean = run(w, regions, markdup=markdup, max_cycle=max_cycle)    # the same kept reads in a context that never held the extra ones
    assert bqsr_paths(g["stats"]) == bqsr_paths(clean["stats"])
    assert np.array_equal(g["tables"], clean["tables"]) and np.array_equal(g["qual"], clean["qual"])
    try:                                                              # without the filter the extra reads fail a phase or pick other kernels
        nf = run(w, regions, markdup=markdup, max_cycle=max_cycle, batch=batch, filt=False)
        assert bqsr_paths(nf["stats"]) != bqsr_paths(clean["stats"]), case
    except device.ElprepError:
        pass


# ---------------------------------------------------------------- extremes, phase order, lifecycle
def test_nothing_dropped_is_byte_identical(exome):
    everything = {0: [(0, 400_000)], 1: [(0, 400_000)]}
    w1 = synth.make_workload(1500, CONTIGS, seed=8, unmapped_frac=0.0, mate_unmapped_frac=0.0, exome=True)
    g = run(w1, everything)
    n = run(w1, everything, filt=False)
    assert g["n_removed"] == 0 and not any(k in g["stats"] for k in NEW_KERNELS[1:])
    for k in ("perm", "flag", "qual_off", "qual", "tables", "emp", "report"):
        assert np.array_equal(g[k], n[k]) if k != "report" else g[k] == n[k], k


def test_everything_dropped(exome):
    g = run(exome, {})
    assert g["n_removed"] == exome.batch.n and g["n_sorted"] == 0 and g["perm"].size == 0 and g["qual"].size == 0
    assert not g["tables"].any()


def test_phase_errors_second_call_and_reset(exome):
    regions = _regions(0)
    ctx = device.Context(exome.header)
    try:
        set_side_inputs(ctx, exome)
        ctx.append(exome.batch)
        with pytest.raises(device.ElprepError) as e:
            ctx.filter_target_regions()
        assert e.value.code == _lib.ESTATE
        ctx.sort_markdup(device.SO_COORDINATE, 1)
        _set_regions(ctx, _regions(150))
        first = ctx.filter_target_regions()
        _set_regions(ctx, regions)                               # narrower regions: a second call drops what they drop
        second = ctx.filter_target_regions()
        o = T.mark_then_filter(exome, regions, bqsr=False)
        assert first + second == o["n_removed"] and second > 0
        idx, flag, _, _ = ctx.fetch(want_qual=False)
        assert np.array_equal(idx, o["perm"]) and np.array_equal(flag, o["flag"])
        ctx.bqsr_gather()
        with pytest.raises(device.ElprepError) as e:
            ctx.filter_target_regions()
        assert e.value.code == _lib.ESTATE
        # the regions survive elp_reset
        ctx.reset()
        ctx.append(exome.batch)
        ctx.sort_markdup(device.SO_COORDINATE, 1)
        assert ctx.n_sorted == exome.batch.n
        assert ctx.filter_target_regions() == o["n_removed"]
        idx, flag, _, _ = ctx.fetch(want_qual=False)
        assert np.array_equal(idx, o["perm"])
        ctx.reset()
        ctx.append(exome.batch)
        ctx.sort_markdup(device.SO_COORDINATE, 1)
        ctx.tables_put(np.zeros(ctx.table_shape(), np.int64))
        with pytest.raises(device.ElprepError) as e:
            ctx.filter_target_regions()
        assert e.value.code == _lib.ESTATE
    finally:
        ctx.close()


def test_tables_only_worker(exome, tmp_path):
    regions = _regions(0)
    o = T.mark_then_filter(exome, regions)
    ctx = device.Context(exome.header)
    try:
        set_side_inputs(ctx, exome)
        ctx.append(exome.batch)
        ctx.sort_markdup(device.SO_COORDINATE, 1)
        _set_regions(ctx, regions)
        ctx.filter_target_regions()
        ctx.bqsr_gather()
        ctx.write_elrecal(str(tmp_path / "w.elrecal"))
    finally:
        ctx.close()
    merge = device.Context(exome.header)
    try:
        merge.tables_clear()
        merge.add_elrecal(str(tmp_path / "w.elrecal"))
        d, _ = oracle_tables_dense(o["tables"])
        assert np.array_equal(merge.tables_get(), d)
    finally:
        merge.close()


def test_no_new_launches_without_the_call(exome):
    g = run(exome, {}, filt=False)
    assert not any(k in g["stats"] for k in NEW_KERNELS), sorted(g["stats"])


def test_exome_two_million_reads():
    w = synth.make_workload(1_000_000, [("chr1", 60_000_000), ("chr2", 40_000_000)], seed=21, exome=True)
    ex = synth.exome_regions([("chr1", 60_000_000), ("chr2", 40_000_000)], seed=21, pad=30)
    regions = {0: ex[0], 1: ex[1]}
    g = run(w, regions)
    o = T.mark_then_filter(w, regions)
    assert 0 < o["n_removed"] < w.batch.n
    compare(g, o)
