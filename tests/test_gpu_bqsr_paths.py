"""GPU parity for every specialisation of the BQSR gather and apply kernels.

The host picks the gather kernels from the QUAL values present in the arena (bqsr_count_kernel<S, INDEL> with S = 1..4 slots and a
classifier shift, or the general bqsr_prep / bqsr_chunk / bqsr_general kernels), from the read length (lanes per read), from the
number of read-group covariates, and the apply kernel from the size of the compact table (bqsr_apply2_kernel, or bqsr_apply_kernel
over the global table).  Every case here compares with the oracle bit for bit (order, FLAG, table counters, EmpiricalQuality,
report text, QUAL bytes) AND asserts, from kernel_stats(), that the kernels it is meant to exercise are the ones that ran."""
import numpy as np
import pytest

from elprep_b200 import synth
from util import (SYNTH_QUALS, apply_plan, bqsr_paths, fast_plan, gpu_phases, gpu_pipeline, oracle_pipeline, oracle_tables_dense,
                  set_side_inputs, with_qual_alphabet)

pytestmark = pytest.mark.gpu

CONTIGS = [("chr20", 300_000), ("chr21", 100_000)]
HISEQ_X = (2, 6, 15, 22, 27, 33, 37, 40)       # seven slots: the general kernels

# (QUAL alphabet, bqsr_count_kernel instance (S, classifier shift) it selects, or None for the general kernels)
ALPHABETS = [
    ((2, 30), (1, 0)),                     # smallest classifier
    ((30,), (1, 0)),                       # no tail values at all
    ((5, 6), (1, 0)),                      # 5 is below the first slot, 6 is the first slot
    ((3, 9, 41), (2, 3)),                  # shifted classifier
    ((2, 11, 25, 37, 40), (4, 0)),
    ((2, 10, 18, 26, 34), (4, 3)),
    ((2, 12, 23, 37, 93), (4, 2)),         # largest legal QUAL
    ((0, 1, 2, 3, 4, 13, 22, 31), (3, 0)),  # eight values, 0..5 inside the count kernel
    (HISEQ_X, None),                       # HiSeq X binning: the fall-back must agree too
]


def _qid(v):
    return "q" + "-".join(str(x) for x in v)


def _compare(g, o, max_cycle=500):
    assert np.array_equal(g["perm"], o["perm"]), "output order differs"
    assert np.array_equal(g["flag"], o["flag"]), "FLAG differs"
    assert np.array_equal(g["qual_off"], o["qual_off"])
    d, e = oracle_tables_dense(o["tables"], max_cycle)
    assert np.array_equal(g["tables"], d), "BQSR table counters differ"
    assert np.array_equal(g["emp"], e), "EmpiricalQuality differs"
    assert g["report"] == o["report"], "recalibration report text differs"
    assert np.array_equal(g["qual"], o["qual"]), "QUAL bytes differ"


def _expected(values, n_cov, L, max_cycle=500):
    return ("fast" if fast_plan(values, n_cov, L) else "general"), apply_plan(values, n_cov, L, max_cycle)


def _check(w, paths, max_cycle=500, n_batches=2):
    g = gpu_pipeline(w, n_batches=n_batches, max_cycle=max_cycle, profile=True)
    assert bqsr_paths(g["stats"]) == paths, sorted(g["stats"])
    _compare(g, oracle_pipeline(w, max_cycle=max_cycle), max_cycle)
    return g


# ---- a. QUAL alphabet x read length x read groups
@pytest.mark.parametrize("n_rg", [1, 4])
@pytest.mark.parametrize("L", [20, 32, 33, 151, 300])            # 1, 1, 2, 5 and 10 lanes of 32 bases per read
@pytest.mark.parametrize("values,plan", ALPHABETS, ids=[_qid(v) for v, _ in ALPHABETS])
def test_alphabet_by_read_length(values, plan, L, n_rg):
    assert fast_plan(values, n_rg, L) == plan
    w = with_qual_alphabet(synth.make_workload(1_500, CONTIGS, seed=1000 + 10 * L + n_rg, L=L, n_rg=n_rg), values, seed=L)
    assert int(w.batch.lseq.max()) == L
    _check(w, _expected(values, n_rg, L))


# ---- b. read-length limits
def _without_known_sites(w):
    return synth.Workload(w.header, w.batch, w.contig_bases, [np.zeros((0, 2), np.int32) for _ in w.contig_bases], w.params)


def _count_kernel_only(w):
    """the reads of ``w`` that bqsr_count_kernel takes whole, without known sites: no indel (an adaptor boundary inside an indel read,
    or a known site on one, sends the read to the general kernels) and not past the contig end"""
    b = w.batch
    co = b.cigar_off.astype(np.int64)
    keep = np.ones(b.n, bool)
    for i in range(b.n):
        ops = b.cigar[co[i]:co[i + 1]]
        reflen = int(sum(int(x) >> 4 for x in ops if (int(x) & 15) in (0, 2, 3, 7, 8)))
        keep[i] = not any((int(x) & 15) in (1, 2) for x in ops) and (b.refid[i] < 0 or b.pos[i] - 1 + reflen <= w.contig_bases[b.refid[i]].size)
    return _without_known_sites(synth.Workload(w.header, b.take(np.nonzero(keep)[0]), w.contig_bases, w.sites, w.params))


def test_read_length_1024():
    """the longest read the fast gather (32 lanes, one read per warp) and bqsr_apply2_kernel (~36 KB compact table) accept, on reads
    the count kernel takes whole"""
    values = (2, 30)
    w = with_qual_alphabet(_count_kernel_only(synth.make_workload(500, CONTIGS, seed=1024, L=1024, n_rg=1)), values)
    assert int(w.batch.lseq.max()) == 1024 and w.batch.n > 900
    g = _check(w, ("fast", "v2"), max_cycle=1024)
    assert "bqsr_g_prep" not in g["stats"]


@pytest.mark.parametrize("n_pairs,seed,L,n_rg,values,whole,phase", [
    (300, 2026, 1024, 4, SYNTH_QUALS, True, "apply"),   # fast gather; the compact table does not fit, and bqsr_apply_kernel stops at 512 bases
    (500, 1024, 1024, 1, (2, 30), False, "gather"),     # fast gather, but some reads go on to the general kernels: 512 bases
    (300, 600, 600, 4, HISEQ_X, False, "gather"),       # general gather: 512 bases
    (300, 1025, 1025, 4, SYNTH_QUALS, False, "gather"),  # longer than any gather kernel
], ids=["1024-gmem-apply", "1024-handed-to-general", "600-general-gather", "1025"])
def test_read_length_limits(n_pairs, seed, L, n_rg, values, whole, phase):
    """whole: only reads the count kernel takes whole (_count_kernel_only), else the workload as generated"""
    from elprep_b200 import device
    w = synth.make_workload(n_pairs, CONTIGS, seed=seed, L=L, n_rg=n_rg)
    assert int(w.batch.pos.min()) >= 0                                 # (a negative POS is refused by sort_markdup)
    if values != SYNTH_QUALS:
        w = with_qual_alphabet(w, values)
    if whole:
        w = _count_kernel_only(w)
    ctx = device.Context(w.header, max_cycle=L, profile=True)       # max_cycle >= L, or the cycle check fails first
    try:
        set_side_inputs(ctx, w)
        ctx.append(w.batch)
        ctx.sort_markdup()
        if phase == "apply":
            ctx.bqsr_gather()
            ctx.bqsr_finalize(None)
            assert bqsr_paths(ctx.kernel_stats())[0] == "fast"
            assert apply_plan(values, n_rg, L, L) == "gmem"
        with pytest.raises(device.ElprepError) as ei:
            ctx.bqsr_apply() if phase == "apply" else ctx.bqsr_gather()
        assert ei.value.code == -15 and "read longer than the device kernel supports" in str(ei.value)
        if phase == "gather":
            assert ("bqsr_g_count" in ctx.kernel_stats()) == (fast_plan(values, n_rg, L) is not None)
            with pytest.raises(device.ElprepError) as ei:                  # no tables were produced
                ctx.bqsr_finalize(None)
            assert ei.value.code == -16
    finally:
        ctx.close()


# ---- c. read-group covariates
@pytest.mark.parametrize("n_rg,gather", [(32, "fast"), (33, "general")])
def test_read_group_covariates(n_rg, gather):
    """32 read groups = 64 classes, the count kernel's limit (mismatch tables in global memory); 33 must take the general kernels"""
    values = (2, 11, 25, 37, 40)
    w = with_qual_alphabet(synth.make_workload(4_000, CONTIGS, seed=3000 + n_rg, L=151, n_rg=n_rg), values)
    assert np.unique(w.batch.rg[w.batch.rg >= 0]).size == n_rg
    _check(w, (gather, apply_plan(values, n_rg, 151)))


@pytest.mark.parametrize("case", ["no_second_of_pair", "read_group_without_reads"])
def test_empty_class(case):
    w = synth.make_workload(2_000, CONTIGS, seed=3100, L=151)
    b = w.batch
    if case == "no_second_of_pair":
        b = b.take(np.nonzero((b.flag & 0x80) == 0)[0])
    else:
        b = b.copy()
        b.rg[b.rg == 2] = 1
    w = synth.Workload(w.header, b, w.contig_bases, w.sites, w.params)
    _check(w, _expected(SYNTH_QUALS, 4, 151))


# ---- e. the QUAL presence bitmap built at ingest
def _pick(b, where, arena_pad=64):
    """(read, byte) of the QUAL arena that gets the new value: the first byte of the middle append, the last byte of the last one,
    or a byte of the middle append 7 bytes past a 16-byte boundary of the arena (which starts with ``arena_pad`` bytes of padding)"""
    n = b.n
    bounds = [0, n // 3, 2 * n // 3, n]
    qo = b.qual_off.astype(np.int64)
    if where == "first":
        at = int(qo[bounds[1]])
    elif where == "last":
        at = int(qo[n]) - 1
    else:
        at = int(qo[bounds[1]]) + 1000
        at += (7 - (arena_pad + at)) % 16
    r = int(np.searchsorted(qo, at, side="right")) - 1
    assert bounds[1] <= r < bounds[2] or where == "last"
    return bounds, r, at


@pytest.mark.parametrize("how", ["append", "append_async", "append_bam", "append_bam_filtered"])
@pytest.mark.parametrize("where", ["first", "last", "unaligned"])
def test_qual_presence_bitmap(where, how):
    """one byte of a QUAL value nothing else carries; if ingest missed it, the count kernel would classify it as another value
    (45 shares q & 7 with 37) or as a low-quality tail (40 lands in an empty classifier entry)"""
    from elprep_b200 import device
    w = synth.make_workload(1_500, CONTIGS, seed=4500, L=151)
    b = w.batch.copy()
    bounds, r, at = _pick(b, where)
    new = 40 if where == "last" else 45
    b.qual[at] = new
    b.mapq[r] = 60                                                     # the read survives the mapping-quality filter
    values = sorted(SYNTH_QUALS + (new,))
    assert fast_plan(values, 4, 151) == ((4, 0) if new == 40 else (4, 3))
    min_mapq = 30 if how == "append_bam_filtered" else 0
    keep = np.nonzero(b.mapq.astype(np.int64) >= min_mapq)[0]
    kept = synth.Workload(w.header, b.take(keep), w.contig_bases, w.sites, w.params)
    assert np.unique(kept.batch.qual).tolist() == values
    ctx = device.Context(w.header, profile=True)
    try:
        set_side_inputs(ctx, w)
        parts = [b.take(np.arange(lo, hi)) for lo, hi in zip(bounds[:-1], bounds[1:])]
        if how == "append":
            for p in parts:
                ctx.append(p)
        elif how == "append_async":
            import bench
            pinned = [bench.pinned(p) for p in parts]
            ctx.append_async(pinned[0])
            ctx.append_async(pinned[1])                                   # two uploads in flight
            ctx.append_wait()
            ctx.append_async(pinned[2])
            ctx.append_wait()
        else:
            ctx.set_ingest_filter(0, min_mapq)
            raw, offs = synth.encode_bam(b, w.header)
            for lo, hi in zip(bounds[:-1], bounds[1:]):
                ctx.append_bam(raw[int(offs[lo]):int(offs[hi])], (offs[lo:hi + 1] - offs[lo]) if hi != b.n else None)
            assert ctx.n_filtered() == b.n - keep.size
        assert ctx.n == keep.size
        g = gpu_phases(ctx, profile=True)
    finally:
        ctx.close()
    assert bqsr_paths(g["stats"]) == ("fast", apply_plan(values, 4, 151)), sorted(g["stats"])
    _compare(g, oracle_pipeline(kept))


# ---- f. one context across elp_reset, and an apply-only worker whose reads arrive after finalize
def test_context_reuse_across_reset():
    """three rounds in one context: S=3 at 151 bases -> seven slots (general) at 100 -> S=1 at 300, reads in 4, 1 and 2 read groups"""
    from elprep_b200 import device
    header = synth.make_header(CONTIGS, 4)
    base = synth.make_workload(10, CONTIGS, seed=600)                 # reference and known sites of genome 600
    rounds = [(151, 4, SYNTH_QUALS), (100, 1, HISEQ_X), (300, 2, (2, 30))]
    ctx = device.Context(header, profile=True)
    try:
        set_side_inputs(ctx, base)
        for k, (L, n_rg, values) in enumerate(rounds):
            w0 = synth.make_workload(1_500, CONTIGS, seed=610 + k, L=L, n_rg=n_rg, genome_seed=600, want_reference=False)
            w = synth.Workload(header, w0.batch, base.contig_bases, base.sites, w0.params)
            if values != SYNTH_QUALS:
                w = with_qual_alphabet(w, values, seed=k)
            if k:
                ctx.reset()
            ctx.reset_stats()
            half = w.batch.n // 2
            ctx.append(w.batch.take(np.arange(0, half)))
            ctx.append(w.batch.take(np.arange(half, w.batch.n)))
            g = gpu_phases(ctx, profile=True)
            assert bqsr_paths(g["stats"]) == _expected(values, 4, L), (k, sorted(g["stats"]))
            _compare(g, oracle_pipeline(w))
    finally:
        ctx.close()


@pytest.mark.parametrize("n_rg", [1, 4])
def test_apply_only_worker_late_reads(n_rg):
    """tables_put -> finalize (no reads yet) -> append reads that are longer and carry a QUAL value the tables never saw -> sort -> apply:
    the apply table and its compact form are rebuilt for them"""
    import oracle
    from elprep_b200 import device
    a = synth.make_workload(1_500, CONTIGS, seed=700, L=100, n_rg=n_rg)
    values = SYNTH_QUALS + (45,)
    bw = with_qual_alphabet(synth.make_workload(1_500, CONTIGS, seed=701, L=151, n_rg=n_rg, genome_seed=700, want_reference=False), values)
    t = oracle_pipeline(a)["tables"]                                  # finalized tables of workload a
    dense, emp = oracle_tables_dense(t)
    bb = bw.batch.copy()
    oracle.mark_duplicates(bb, bw.header, n_threads=1)
    perm = oracle.coordinate_sort(bb, n_threads=4)
    srt = bb.take(perm)
    oracle.bqsr_apply(srt, bw.header, t, n_threads=4)
    ctx = device.Context(bw.header, profile=True)
    try:
        ctx.tables_put(dense)
        ctx.bqsr_finalize(None)
        assert np.array_equal(ctx.empirical_get(), emp)
        half = bw.batch.n // 2
        ctx.append(bw.batch.take(np.arange(0, half)))
        ctx.append(bw.batch.take(np.arange(half, bw.batch.n)))
        ctx.sort_markdup()
        ctx.bqsr_apply()
        idx, flag, qoff, qual = ctx.fetch()
        assert bqsr_paths(ctx.kernel_stats())[1] == apply_plan(values, n_rg, 151)
    finally:
        ctx.close()
    assert np.array_equal(idx, perm.astype(np.uint64)) and np.array_equal(flag, srt.flag)
    assert np.array_equal(qoff, srt.qual_off) and np.array_equal(qual[:int(qoff[-1])], srt.qual), "QUAL bytes differ"


# ---- g. --max-cycle
@pytest.mark.parametrize("max_cycle", [151, 200])
def test_max_cycle(max_cycle):
    w = synth.make_workload(1_500, CONTIGS, seed=5000 + max_cycle, L=151)
    _check(w, _expected(SYNTH_QUALS, 4, 151, max_cycle), max_cycle=max_cycle)


def test_max_cycle_exceeded_then_reset():
    """a 151-base read with --max-cycle 150 is the reference's cycle error; the context stays usable after elp_reset"""
    from elprep_b200 import device
    w = synth.make_workload(1_500, CONTIGS, seed=5100, L=151)
    with pytest.raises(ValueError, match="cycle value exceeds maximum cycle value"):
        oracle_pipeline(w, max_cycle=150)
    w2 = synth.make_workload(1_500, CONTIGS, seed=5101, L=150, genome_seed=5100, want_reference=False)
    w2 = synth.Workload(w.header, w2.batch, w.contig_bases, w.sites, w2.params)
    ctx = device.Context(w.header, max_cycle=150, profile=True)
    try:
        set_side_inputs(ctx, w)
        ctx.append(w.batch)
        ctx.sort_markdup()
        with pytest.raises(device.ElprepError) as ei:
            ctx.bqsr_gather()
        assert ei.value.code == -12 and "cycle value exceeds maximum cycle value" in str(ei.value)
        ctx.reset()
        ctx.reset_stats()
        ctx.append(w2.batch)
        g = gpu_phases(ctx, profile=True)
    finally:
        ctx.close()
    assert bqsr_paths(g["stats"]) == _expected(SYNTH_QUALS, 4, 150, 150)
    _compare(g, oracle_pipeline(w2, max_cycle=150), 150)
