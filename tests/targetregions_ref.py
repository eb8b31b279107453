"""The reference's phase order for `--target-regions`, composed from the oracle and the ingest-filter restatement, as expected results for
elp_filter_target_regions:

  1. duplicate marking (and the coordinate / queryname sort) over EVERY read           oracle.mark_duplicates, oracle.*_sort
  2. RemoveNonOverlappingReads(bedRegions) over the output order                        ingestfilter_ref.remove_non_overlapping
     (filters/simple-filters.go:308-328; runBestPracticesPipelineIntermediateSam, cmd/filter.go:171-180)
  3. BQSR gather, finalize and apply over the kept reads only                           oracle.bqsr_*

``ingest_then_mark`` is the other order -- the reads dropped before marking, as `--filter-non-overlapping-reads` does -- so that tests can
show where the two give different FLAGs."""
from __future__ import annotations

import os
import tempfile

import numpy as np

import ingestfilter_ref as R


def recs_of(batch):
    """ingestfilter_ref.Rec of every read of an AlignmentBatch (the fields RemoveNonOverlappingReads looks at)"""
    co = batch.cigar_off.astype(np.int64)
    return [R.Rec(refid=int(batch.refid[i]), pos=int(batch.pos[i]), flag=int(batch.flag[i]), cigar=R.cigar_from_words(batch.cigar[co[i]:co[i + 1]]),
                  lseq=int(batch.lseq[i])) for i in range(batch.n)]


def flatten(regions):
    """{contig: (start, end) pairs} -> {contig: flattened pairs}, as elp_set_bqsr_target_regions stores them"""
    return {int(c): R.flatten_regions(np.asarray(iv, np.int64).reshape(-1, 2).tolist()) for c, iv in regions.items()}


def keep_mask(batch, regions):
    """RemoveNonOverlappingReads(regions) of every read of ``batch``; regions: {contig: (start, end) pairs}, not yet flattened"""
    keep = R.remove_non_overlapping(flatten(regions))
    return np.array([keep(r) for r in recs_of(batch)], dtype=bool)


def _order(b, sort):
    import oracle
    if sort == "coordinate":
        return oracle.coordinate_sort(b, n_threads=4)
    if sort == "queryname":
        return oracle.queryname_sort(b)
    return np.arange(b.n, dtype=np.int64)


def mark_then_filter(w, regions, sort="coordinate", markdup=True, bqsr=True, max_cycle=500, batch=None):
    """the reference order.  w: a synth.Workload (header, reference, known sites; batch overrides its reads).  Returns perm (arrival index of
    every kept output record), flag, qual_off and qual (recalibrated when bqsr), n_removed, keep (mask over the full output order), and with
    bqsr the oracle tables and report text."""
    import oracle
    b = (batch if batch is not None else w.batch).copy()
    if markdup:
        oracle.mark_duplicates(b, w.header, n_threads=1)
    perm = _order(b, sort)
    srt = b.take(perm)
    keep = keep_mask(srt, regions)
    kept = srt.take(np.nonzero(keep)[0])
    res = dict(perm=perm[keep].astype(np.uint64), flag=kept.flag.copy(), qual_off=kept.qual_off.copy(), qual=kept.qual.copy(),
               n_removed=int((~keep).sum()), keep=keep, flag_all=srt.flag.copy())
    if bqsr:
        ref = oracle.Reference(w.header, w.contig_bases, w.sites)
        t = oracle.bqsr_gather(kept, w.header, ref, max_cycle=max_cycle, n_threads=4)
        oracle.bqsr_finalize(t)
        with tempfile.TemporaryDirectory() as d:
            p = os.path.join(d, "o.recal")
            oracle.bqsr_report(t, oracle.OracleHeader(w.header).cov_names, p)
            res["report"] = open(p).read()
        oracle.bqsr_apply(kept, w.header, t, n_threads=4)
        res["qual"] = kept.qual.copy()
        res["tables"] = t
    return res


def ingest_then_mark(header, batch, regions, sort="coordinate"):
    """`--filter-non-overlapping-reads`: the reads dropped before marking -> (arrival indices of the kept reads in output order, FLAG)"""
    import oracle
    idx = np.nonzero(keep_mask(batch, regions))[0]
    b = batch.take(idx)
    oracle.mark_duplicates(b, header, n_threads=1)
    perm = _order(b, sort)
    return idx[perm].astype(np.uint64), b.flag[perm].copy()
