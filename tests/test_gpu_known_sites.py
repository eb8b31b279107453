"""GPU parity of the known-sites masking (calculateSkipSlice, filters/bqsr.go:389-414) on every device path a read can take, chosen by
the number of site ranges its clipped alignment overlaps:

  0-2 ranges, no indel     bqsr_prep2_kernel packs them into the 32-byte work record; bqsr_count_kernel turns them into range planes
  3-4 ranges, or any range on an indel read     handed to the general kernels: ReadDesc.skip[4], bqsr_chunk_kernel<false / true>
  5 or more                a 512-bit mask per read (DF_SKIP_OVF), read by bqsr_general_kernel (warp per read)

Every case runs through the device and the oracle and compares bit for bit (order, FLAG, table counters, EmpiricalQuality, report
text, QUAL bytes), and asserts from kernel_stats() that the kernels it is meant to exercise ran.  Site lists also go in raw, the way
callers hand them over (elp_set_known_sites with already_flat = 0); the oracle then gets the restatement's flattened list."""
import ctypes as C
import os
import tempfile

import numpy as np
import pytest

import knownsites_cases as kc
import knownsites_ref as ks
from elprep_b200 import synth
from util import (apply_plan, bqsr_paths, compare_bqsr, fast_plan, gpu_phases, gpu_pipeline, oracle_pipeline, oracle_tables_dense,
                  set_side_inputs, with_qual_alphabet)

pytestmark = pytest.mark.gpu

HISEQ_X = (2, 6, 15, 22, 27, 33, 37, 40)       # seven slots: the general kernels
ALPHABETS = [(2, 30), (2, 11, 25, 37, 40), HISEQ_X]   # bqsr_count_kernel S = 1, S = 4, and the general kernels
FAST_ALPHABETS = ALPHABETS[:2]


def _qid(v):
    return "q" + "-".join(str(x) for x in v)


def _run(cases, values, n_rg, expect, max_cycle=500, seed=0):
    """expect: "count" (every read stays in bqsr_count_kernel on the fast path), "skip4" (the general kernels with <= 4 ranges per read)
    or "ovf" (some read needs an overflow mask)"""
    w, _ = kc.build(cases, values, n_rg=n_rg, seed=seed)
    assert np.unique(w.batch.qual).tolist() == sorted(values)
    L = int(w.batch.lseq.max())
    fast = fast_plan(values, n_rg, L) is not None
    # bqsr_apply_kernel (the apply when the compact table does not fit) stops at 512 bases: longer reads are compared up to finalize
    whole = L <= 512 or apply_plan(values, n_rg, L, max_cycle) == "v2"
    g = gpu_pipeline(w, max_cycle=max_cycle, profile=True) if whole else _gather_only(w, max_cycle)
    st = g["stats"]
    assert bqsr_paths(st)[0] == ("fast" if fast else "general"), sorted(st)
    if expect == "count":
        assert ("bqsr_g_prep" not in st) if fast else ("bqsr_g_chunk" in st), sorted(st)
    if expect in ("count", "skip4"):
        assert "bqsr_g_warp_per_read" not in st, sorted(st)
    if expect == "skip4":
        assert "bqsr_g_prep" in st and ("bqsr_g_chunk_list" in st or "bqsr_g_chunk" in st), sorted(st)
    if expect == "ovf":
        assert "bqsr_g_prep" in st and "bqsr_g_warp_per_read" in st, sorted(st)
    o = oracle_pipeline(w, max_cycle=max_cycle)
    if whole:
        compare_bqsr(g, o, max_cycle)
    else:
        d, e = oracle_tables_dense(o["tables"], max_cycle)
        assert np.array_equal(g["perm"], o["perm"]) and np.array_equal(g["flag"], o["flag"])
        assert np.array_equal(g["tables"], d), "BQSR table counters differ"
        assert np.array_equal(g["emp"], e) and g["report"] == o["report"]
    return g


def _gather_only(w, max_cycle):
    """sort + duplicate marking + gather + finalize on the device, without apply"""
    from elprep_b200 import device
    ctx = device.Context(w.header, max_cycle=max_cycle, profile=True)
    try:
        set_side_inputs(ctx, w)
        ctx.append(w.batch)
        ctx.sort_markdup()
        ctx.bqsr_gather()
        g = dict(tables=ctx.tables_get())
        with tempfile.TemporaryDirectory() as dname:
            p = os.path.join(dname, "g.recal")
            ctx.bqsr_finalize(p)
            g["report"] = open(p).read()
        g["emp"] = ctx.empirical_get()
        idx, flag, _, _ = ctx.fetch(want_qual=False)
        g.update(perm=idx, flag=flag, stats=ctx.kernel_stats())
        return g
    finally:
        ctx.close()


# ---- 0-2 ranges: bqsr_count_kernel
@pytest.mark.parametrize("n_rg", [1, 4])
@pytest.mark.parametrize("L", [32, 33, 64, 151])
@pytest.mark.parametrize("values", ALPHABETS, ids=_qid)
def test_count_kernel_ranges(values, L, n_rg):
    _run(kc.count_cases(L) + kc.adaptor_cases(L), values, n_rg, "count", seed=L + n_rg)


@pytest.mark.parametrize("n_rg", [1, 4])
@pytest.mark.parametrize("values", FAST_ALPHABETS, ids=_qid)
def test_count_kernel_ranges_1024(values, n_rg):
    """32 lanes per read; only the count kernel takes 1024 bases (the general kernels stop at 512).  Where the compact apply table does
    not fit (S = 4, or 4 read groups) the comparison ends at finalize, since the global-table apply also stops at 512"""
    _run(kc.count_cases(1024) + kc.adaptor_cases(1024), values, n_rg, "count", max_cycle=1024, seed=1024 + n_rg)


# ---- hand-off: 3-4 ranges, and sites on indel reads
@pytest.mark.parametrize("n_rg", [1, 4])
@pytest.mark.parametrize("values", ALPHABETS, ids=_qid)
def test_handoff_skip4(values, n_rg):
    g = _run(kc.handoff_cases(151), values, n_rg, "skip4", seed=20 + n_rg)
    assert "bqsr_g_chunk_list" in g["stats"]                          # the indel reads, on both paths


# ---- more than four ranges: the overflow masks
@pytest.mark.parametrize("n_rg", [1, 4])
@pytest.mark.parametrize("values", ALPHABETS, ids=_qid)
def test_overflow_masks(values, n_rg):
    _run(kc.overflow_cases(151), values, n_rg, "ovf", seed=30 + n_rg)


@pytest.mark.parametrize("n_rg", [1, 4])
@pytest.mark.parametrize("values", ALPHABETS, ids=_qid)
def test_overflow_masks_512(values, n_rg):
    """512-base reads with ranges in bases 480-511: the last word of the mask"""
    _run(kc.overflow_cases(512), values, n_rg, "ovf", max_cycle=512, seed=40 + n_rg)


# ---- getReadCoordinateForReferenceCoordinate's quirks on the general path
@pytest.mark.parametrize("n_rg", [1, 4])
@pytest.mark.parametrize("values", ALPHABETS, ids=_qid)
def test_read_coordinate_quirks(values, n_rg):
    _run(kc.quirk_cases(60), values, n_rg, "ovf", seed=50 + n_rg)


# ---- site lists as callers pass them (already_flat = 0)
CONTIGS = [("chr20", 300_000), ("chr21", 100_000)]


def _raw_sites(n, lo, hi, seed):
    """n raw intervals in [lo, hi): random short ones with duplicates, contained, touching and adjacent neighbours, unsorted"""
    rng = np.random.default_rng(seed)
    s = rng.integers(lo, hi - 40, size=n)
    e = s + rng.integers(0, 20, size=n) * (rng.random(n) < 0.3)
    iv = np.stack([s, e], 1)
    k = n // 8
    extra = [iv[:k],                                                                  # duplicates
             np.stack([iv[k:2 * k, 0] + (iv[k:2 * k, 1] - iv[k:2 * k, 0]) // 2] * 2, 1),   # contained
             np.stack([iv[2 * k:3 * k, 1], iv[2 * k:3 * k, 1] + 3], 1),              # touching: merge
             np.stack([iv[3 * k:4 * k, 1] + 1, iv[3 * k:4 * k, 1] + 2], 1)]          # adjacent: stay apart
    out = np.concatenate([iv] + extra).astype(np.int32)
    return out[rng.permutation(len(out))]


def _context_run(ctx, w, raw, values):
    """raw site list per contig into the context (already_flat = 0), then the pipeline; the oracle gets the restatement's flattening"""
    for ci in range(len(w.header.SQ)):
        ctx.set_known_sites(ci, raw[ci], already_flat=False)
    ctx.append(w.batch)
    g = gpu_phases(ctx, profile=True)
    flat = [ks.sort_and_flatten(r) for r in raw]
    o = oracle_pipeline(synth.Workload(w.header, w.batch, w.contig_bases, flat, w.params))
    return g, o


@pytest.mark.parametrize("values", ALPHABETS, ids=_qid)
def test_raw_site_lists(values):
    """more than 4096 unsorted intervals on one contig (duplicated, contained, touching, adjacent) next to a contig without sites"""
    from elprep_b200 import device
    w = with_qual_alphabet(synth.make_workload(4_000, CONTIGS, seed=60, L=151), values)
    raw = [_raw_sites(6_000, 1, CONTIGS[0][1], seed=61), np.zeros((0, 2), np.int32)]
    flat = ks.sort_and_flatten(raw[0])
    assert len(raw[0]) > 4096 and len(flat) < len(raw[0]) and not np.array_equal(np.sort(raw[0], 0), raw[0])
    assert ((flat[1:, 0] - flat[:-1, 1]) == 1).any()                  # adjacent intervals survived the flattening
    ctx = device.Context(w.header, profile=True)
    try:
        for ci in range(len(CONTIGS)):
            ctx.set_reference(ci, w.contig_bases[ci])
        g, o = _context_run(ctx, w, raw, values)
    finally:
        ctx.close()
    assert "bqsr_g_warp_per_read" in g["stats"], sorted(g["stats"])
    compare_bqsr(g, o)


def test_sites_replaced_across_reset():
    """one context, two gathers: the second list is uploaded again after elp_reset (the table is dirty), and the tables follow it"""
    from elprep_b200 import device
    values = (2, 11, 25, 37, 40)
    w = with_qual_alphabet(synth.make_workload(3_000, CONTIGS, seed=70, L=151), values)
    lists = [[_raw_sites(3_000, 1, CONTIGS[0][1], seed=71), _raw_sites(500, 1, CONTIGS[1][1], seed=72)],
             [np.zeros((0, 2), np.int32), _raw_sites(5_000, 1, CONTIGS[1][1], seed=73)]]
    ctx = device.Context(w.header, profile=True)
    tables = []
    try:
        for ci in range(len(CONTIGS)):
            ctx.set_reference(ci, w.contig_bases[ci])
        for k, raw in enumerate(lists):
            if k:
                ctx.reset()
                ctx.reset_stats()
            g, o = _context_run(ctx, w, raw, values)
            compare_bqsr(g, o)
            tables.append(g["tables"])
    finally:
        ctx.close()
    assert not np.array_equal(tables[0], tables[1])


# ---- dense sites at size: more reads with > 4 ranges than the first guess of overflow slots
def _overflowing_reads(w):
    """eligible reads (recalibrateAln, after duplicate marking) whose clipped alignment overlaps more than four site ranges; the clipping
    is the oracle's (orc_probe_clip), the range count the restatement's Intersect"""
    import oracle
    b = w.batch.copy()
    oracle.mark_duplicates(b, w.header, n_threads=1)
    L = oracle.lib()
    co = b.cigar_off.astype(np.int64)
    clen = w.header.contig_lengths()
    elig = ((b.opt_flags & 1) == 0) & (b.mapq > 0) & (b.mapq < 255) & ((b.flag & (0x100 | 0x400 | 0x200 | 0x4)) == 0) & (b.refid >= 0) & \
           (b.pos > 0) & (b.lseq > 0) & (b.rg >= 0)
    cpos, cend, keep = [], [], []
    lo, hi, npos = C.c_int32(), C.c_int32(), C.c_int32()
    out = np.zeros(64, np.uint32)
    for i in np.nonzero(elig)[0]:
        if b.pos[i] > clen[b.refid[i]]:
            continue
        cg = np.ascontiguousarray(b.cigar[co[i]:co[i + 1]])
        if ((cg & 15) == 3).any() or int(sum(int(x) >> 4 for x in cg if (int(x) & 15) in (0, 1, 4, 7, 8))) != int(b.lseq[i]):
            continue
        n = L.orc_probe_clip(C.c_int32(int(b.pos[i])), C.c_uint16(int(b.flag[i])), C.c_int32(int(b.pnext[i])), C.c_int32(int(b.tlen[i])),
                             C.c_int32(int(b.refid[i])), C.c_int32(int(b.nref[i])), cg.ctypes.data_as(C.c_void_p), C.c_int32(len(cg)),
                             C.c_int32(int(b.lseq[i])), C.byref(lo), C.byref(hi), C.byref(npos), out.ctypes.data_as(C.c_void_p), C.c_int(64))
        if n <= 0:
            continue
        reflen = sum(int(x) >> 4 for x in out[:n] if (int(x) & 15) in (0, 2, 3, 7, 8))
        cpos.append(npos.value); cend.append(npos.value + reflen - 1); keep.append(int(b.refid[i]))
    cpos, cend, keep = np.array(cpos), np.array(cend), np.array(keep)
    total = 0
    for ci, s in enumerate(w.sites):
        m = keep == ci
        if not m.any() or not len(s):
            continue
        first = np.searchsorted(s[:, 1], cpos[m], side="left")
        last = np.searchsorted(s[:, 0], cend[m], side="right")
        total += int(((last - first) > 4).sum())
    return total


@pytest.mark.parametrize("values", [(2, 11, 25, 37, 40), HISEQ_X], ids=_qid)
@pytest.mark.parametrize("every", [50, 3])
def test_dense_sites(every, values):
    """~200 k reads of 151 bases, 4 read groups, random 1-bp sites at one per ``every`` bases plus a few 2-30 bp intervals: more eligible
    reads need an overflow mask than the n/16 + 4096 slots the gather reserves at first, and none of them may fail it"""
    contigs = [("chr20", 3_000_000)]
    w = with_qual_alphabet(synth.make_workload(100_000, contigs, seed=80, L=151, n_rg=4, cross_contig_frac=0.0), values)
    rng = np.random.default_rng(81 + every)
    ln = contigs[0][1]
    one = np.sort(rng.choice(np.arange(1, ln + 1, dtype=np.int32), size=ln // every, replace=False))
    s = rng.integers(1, ln - 40, size=300).astype(np.int32)
    raw = np.concatenate([np.stack([one, one], 1), np.stack([s, s + rng.integers(1, 30, size=300).astype(np.int32)], 1)])
    w = synth.Workload(w.header, w.batch, w.contig_bases, [ks.sort_and_flatten(raw)], w.params)
    n = w.batch.n
    n_over = _overflowing_reads(w)
    assert n_over > n // 16 + 4096, (n_over, n)
    g = gpu_pipeline(w, profile=True)
    assert "bqsr_g_warp_per_read" in g["stats"], sorted(g["stats"])
    compare_bqsr(g, oracle_pipeline(w))
