"""Parity at the BASELINE.json sizes (SURVEY.md 8d): C1 = 2 M reads on one contig, C2 = 30 M reads on an hg38/20-shaped genome.
The CUDA path (through the C ABI) is compared record by record with the oracle: output permutation, FLAG (u16) of every
record, the BQSR tables, EmpiricalQuality and every recalibrated QUAL byte.  C2 crosses 2^32 bytes in the QUAL arena and
thousands of onesweep tiles / look-back steps per radix pass -- the first size at which a 32-bit offset or a look-back bug
would show.  Oracle time at 30 M reads: ~25-60 s on the GPU box's host cores."""
import os

import numpy as np
import pytest

from elprep_b200 import synth
from util import bqsr_paths, fast_plan, oracle_tables_dense, with_qual_alphabet

pytestmark = pytest.mark.gpu
THREADS = min(os.cpu_count() or 1, 64)


def _run_gpu(w, sort, markdup, bqsr, n_batches, profile=False):
    from elprep_b200 import device
    ctx = device.Context(w.header, profile=profile)
    try:
        if bqsr:
            for ci in range(len(w.header.SQ)):
                ctx.set_reference(ci, w.contig_bases[ci])
                ctx.set_known_sites(ci, w.sites[ci], already_flat=True)
        n = w.batch.n
        bounds = [n * i // n_batches for i in range(n_batches + 1)]
        for a, b in zip(bounds[:-1], bounds[1:]):
            ctx.append(synth.take(w.batch, np.arange(a, b), threads=THREADS) if n_batches > 1 else w.batch)
        ctx.sort_markdup(device.SO_COORDINATE if sort else device.SO_KEEP, markdup)
        res = {}
        if bqsr:
            ctx.bqsr_gather()
            res["tables"] = ctx.tables_get()
            ctx.bqsr_finalize(None)
            res["emp"] = ctx.empirical_get()
            ctx.bqsr_apply()
        idx, flag, qoff, qual = ctx.fetch()
        res.update(perm=idx, flag=flag, qual=qual[:int(qoff[-1])], qual_off=qoff)
        if profile:
            res["stats"] = ctx.kernel_stats()
        return res
    finally:
        ctx.close()


def _run_oracle(w, sort, markdup, bqsr):
    """in place on w.batch (run the GPU first)"""
    import oracle
    b = w.batch
    if markdup:
        oracle.mark_duplicates(b, w.header, n_threads=THREADS)
    perm = oracle.coordinate_sort(b, n_threads=THREADS) if sort else np.arange(b.n, dtype=np.int64)
    srt = synth.take(b, perm, threads=THREADS)
    res = dict(perm=perm.astype(np.uint64), flag=srt.flag, qual=srt.qual)
    if bqsr:
        ref = oracle.Reference(w.header, w.contig_bases, w.sites)
        t = oracle.bqsr_gather(srt, w.header, ref, n_threads=THREADS)
        oracle.bqsr_finalize(t)
        oracle.bqsr_apply(srt, w.header, t, n_threads=THREADS)
        res["qual"] = srt.qual
        res["tables"], res["emp"] = oracle_tables_dense(t)
    return res


def _compare(g, o, bqsr):
    assert np.array_equal(g["perm"], o["perm"]), "output order differs"
    assert np.array_equal(g["flag"], o["flag"]), f"FLAG differs in {int((g['flag'] != o['flag']).sum())} records"
    if bqsr:
        assert np.array_equal(g["tables"], o["tables"]), "BQSR table counters differ"
        assert np.array_equal(g["emp"], o["emp"]), "EmpiricalQuality differs"
    assert g["qual"].shape == o["qual"].shape and np.array_equal(g["qual"], o["qual"]), "QUAL bytes differ"


def test_c1_2m_sort_only():
    """configs[0]: chr20-only, 2 M reads, --sorting-order coordinate"""
    w = synth.make_workload(1_000_000, [("chr20", 64_444_167)], seed=20260924, want_reference=False, threads=THREADS)
    g = _run_gpu(w, True, False, False, 4)
    o = _run_oracle(w, True, False, False)
    _compare(g, o, False)


def _c1_full_path(quals=None):
    w = synth.make_workload(1_000_000, [("chr20", 64_444_167)], seed=20260925, threads=THREADS)
    if quals:
        w = with_qual_alphabet(w, quals, seed=25)
    g = _run_gpu(w, True, True, True, 3, profile=True)
    o = _run_oracle(w, True, True, True)
    _compare(g, o, True)
    assert int(((g["flag"] & 0x400) != 0).sum()) > 100_000
    assert bqsr_paths(g["stats"])[0] == "fast"


def test_c1_2m_full_path():
    """the generator's four QUAL levels: count kernel S = 3"""
    _c1_full_path()


def test_c1_2m_full_path_s4_alphabet():
    """a five-value alphabet (count kernel S = 4, classifier shift 3): every read-group class runs many 255-pass segments through a
    contended work queue"""
    quals = (2, 10, 18, 26, 34)
    assert fast_plan(quals, 4, 150) == (4, 3)
    _c1_full_path(quals)


def test_c2_30m_full_path():
    """configs[1] (+ the BQSR half of configs[2]): 30 M reads, hg38/20-shaped genome, 25 contigs; > 2^32 QUAL bytes"""
    w = synth.make_workload(15_000_000, synth.scaled_hg38(20.0), seed=20260924, threads=THREADS)
    assert int(w.batch.qual.size) > 1 << 32
    g = _run_gpu(w, True, True, True, 1)
    o = _run_oracle(w, True, True, True)
    _compare(g, o, True)
    assert int(((g["flag"] & 0x400) != 0).sum()) > 2_000_000
