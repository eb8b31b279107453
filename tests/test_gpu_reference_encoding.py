"""GPU parity of the BQSR gather on references that are not upper-case ACGTN.

The device keeps one copy of the reference, as one-hot nibbles (A/a/* 1, C/c 2, G/g 4, T/t 8, every other byte 0), and every gather
kernel takes its mismatches from it; baseToIntMap (filters/bqsr.go:247-252) is the rule they must follow: a lower-case base counts as
its upper-case one, `*` as A, and any other byte mismatches every read base.  Each case overwrites part of every contig (its first and
last 40 bases included) with lower-case bases, `*`, `N`, `=`, every IUPAC code and arbitrary bytes 0-255, adds reads that start on a
contig's first base or end on its last, runs the device and the oracle and compares bit for bit (order, FLAG, table counters,
EmpiricalQuality, report text, QUAL bytes), and asserts from kernel_stats() which gather kernels ran."""
import numpy as np
import pytest

import knownsites_cases as kc
from elprep_b200 import _lib, sam, synth
from util import SYNTH_QUALS, bqsr_paths, compare_bqsr, gpu_phases, gpu_pipeline, oracle_pipeline, with_qual_alphabet

pytestmark = pytest.mark.gpu

CONTIGS = [("chr20", 300_000), ("chr21", 100_000)]
HISEQ_X = (2, 6, 15, 22, 27, 33, 37, 40)       # seven slots: the general kernels
IUPAC = b"RYSWKMBDHVN"
ODD = np.frombuffer(b"acgt*N=" + IUPAC + IUPAC.lower(), np.uint8)


def _qid(v):
    return "q" + "-".join(str(x) for x in v)


def _scramble(bases, seed):
    """a copy of one contig: the first and last 40 bases and 10 % of the others become random bytes of ODD or 0-255, another 5 % the
    lower-case form of their base, and 2 % of the A bases `*`"""
    rng = np.random.default_rng(seed)
    out = np.array(bases, dtype=np.uint8, copy=True)
    n = out.size
    pool = np.concatenate([ODD, np.arange(256, dtype=np.uint8)])
    pick = rng.random(n)
    odd = (pick < 0.10) | (np.arange(n) < 40) | (np.arange(n) >= n - 40)
    out[odd] = pool[rng.integers(0, pool.size, size=int(odd.sum()))]
    low = (pick >= 0.10) & (pick < 0.15)
    out[low] = np.frombuffer(bytes(out[low]).lower(), np.uint8)
    star = (pick >= 0.15) & (pick < 0.17) & (out == ord("A"))
    out[star] = ord("*")
    assert np.isin(pool, out).all()
    return out


def _edge_reads(header, contig_bases, quals, n_rg, seed, L=151):
    """unpaired reads on both strands that start on each contig's first bases or end on its last ones: one M run, and with an insertion
    or a deletion; SEQ from ``contig_bases`` with 5 % substitutions"""
    rng = np.random.default_rng(seed)
    recs = []
    for ci, (name, ln) in enumerate(zip(header.contig_names(), (len(b) for b in contig_bases))):
        ref = contig_bases[ci]
        for k, (cg, reflen) in enumerate(((f"{L}M", L), (f"30M2I{L - 32}M", L - 2), (f"30M3D{L - 30}M", L + 3))):
            for pos in (1 + 3 * k, ln - reflen + 1 - 3 * k):          # distinct 5' ends: no read is a duplicate of another
                for flag in (0, 0x10):
                    seq = [chr(b) for b in ref[pos - 1:pos - 1 + reflen]]
                    if "D" in cg:
                        del seq[30:33]
                    if "I" in cg:
                        seq[30:30] = ["ACGT"[int(x)] for x in rng.integers(0, 4, size=2)]
                    seq = [("ACGT"[int(rng.integers(0, 4))] if rng.random() < 0.05 else s) for s in seq]
                    recs.append(dict(QNAME=f"edge{len(recs):04d}", FLAG=flag, RNAME=name, POS=pos, MAPQ=60, CIGAR=cg, RNEXT="*", PNEXT=0,
                                     TLEN=0, SEQ="".join(seq), QUAL=[int(x) for x in rng.choice(quals, size=L)], RG=f"rg{len(recs) % n_rg + 1}"))
    return sam.AlignmentBatch.from_records(header, recs)


def _with_edges(w, quals, n_rg, seed):
    """``w`` plus its edge reads, on the scrambled reference"""
    batch = sam.AlignmentBatch.concat([w.batch, _edge_reads(w.header, w.contig_bases, quals, n_rg, seed)])
    return synth.Workload(w.header, batch, [_scramble(b, seed + ci) for ci, b in enumerate(w.contig_bases)], w.sites, w.params)


def _synth_case(values, seed, n_rg=4):
    w = _with_edges(synth.make_workload(1_500, CONTIGS, seed=seed, L=151, n_rg=n_rg), SYNTH_QUALS, n_rg, seed)
    return with_qual_alphabet(w, values, seed=seed) if values != SYNTH_QUALS else w


def _run(w):
    g = gpu_pipeline(w, n_batches=2, profile=True)
    compare_bqsr(g, oracle_pipeline(w))
    return g["stats"]


# ---- bqsr_count_kernel (S = 1 and S = 4): reads without and with an indel
@pytest.mark.parametrize("n_rg", [1, 4])
@pytest.mark.parametrize("values", [(2, 30), (2, 11, 25, 37, 40)], ids=_qid)
def test_count_kernel(values, n_rg):
    st = _run(_synth_case(values, 100 + n_rg, n_rg))
    assert bqsr_paths(st)[0] == "fast" and st["bqsr_g_count"]["launches"] and st["bqsr_g_count_indel"]["launches"], sorted(st)


# ---- the general kernels over every read: bqsr_chunk_kernel<false> (one M run) and <true> (indel reads)
@pytest.mark.parametrize("n_rg", [1, 4])
def test_chunk_kernels(n_rg):
    st = _run(_synth_case(HISEQ_X, 200 + n_rg, n_rg))
    assert bqsr_paths(st)[0] == "general" and "bqsr_g_chunk" in st and "bqsr_g_chunk_list" in st, sorted(st)


# ---- reads the fast path hands to the general kernels: known sites on indel reads (bqsr_chunk_kernel<true> over a list), more than
# four site ranges (bqsr_general_kernel, warp per read)
@pytest.mark.parametrize("values", [(2, 30), HISEQ_X], ids=_qid)
@pytest.mark.parametrize("cases,kernel", [(kc.handoff_cases(151), "bqsr_g_chunk_list"), (kc.overflow_cases(151), "bqsr_g_warp_per_read")],
                         ids=["handoff", "overflow"])
def test_handed_off_reads(cases, kernel, values):
    w, _ = kc.build(cases, values, n_rg=4, seed=300)
    st = _run(_with_edges(w, values, 4, 300))
    assert "bqsr_g_prep" in st and kernel in st, sorted(st)


# ---- the reference replaced: before the first gather, and after elp_reset
def test_reference_replaced():
    from elprep_b200 import device
    values = (2, 11, 25, 37, 40)
    w = _synth_case(values, 400)
    refs = [w.contig_bases, [_scramble(b, 410 + ci) for ci, b in enumerate(w.contig_bases)]]
    ctx = device.Context(w.header, profile=True)
    tables = []
    try:
        for ci, b in enumerate(w.contig_bases):
            ctx.set_reference(ci, np.full(len(b) // 2, ord("T"), np.uint8))   # shorter and different: the next call must replace it
            ctx.set_known_sites(ci, w.sites[ci])
        for k, ref in enumerate(refs):
            if k:
                ctx.reset()
                ctx.reset_stats()
            for ci, b in enumerate(ref):
                ctx.set_reference(ci, b)
            ctx.append(w.batch)
            g = gpu_phases(ctx, profile=True)
            assert bqsr_paths(g["stats"])[0] == "fast", sorted(g["stats"])
            compare_bqsr(g, oracle_pipeline(synth.Workload(w.header, w.batch, ref, w.sites, w.params)))
            tables.append(g["tables"])
    finally:
        ctx.close()
    assert not np.array_equal(tables[0], tables[1])


def test_known_sites_null_pointer():
    from elprep_b200 import device
    ctx = device.Context(synth.make_header(CONTIGS))
    try:
        assert ctx.L.elp_set_known_sites(ctx.h, 0, None, 3, 0) == _lib.EINVAL
        assert "null interval array" in ctx.L.elp_last_error(ctx.h).decode()
        assert ctx.L.elp_set_known_sites(ctx.h, 0, None, 0, 0) == 0
    finally:
        ctx.close()
