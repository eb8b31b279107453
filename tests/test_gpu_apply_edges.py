"""BQSR apply at its edges, on both kernels: bqsr_apply2_kernel (compact table in shared memory, stats "bqsr_apply") and
bqsr_apply_kernel (global table, stats "bqsr_apply_gmem", forced with ELPREP_B200_APPLY=v1).

Every case of apply_cases.py goes through append -> sort (no duplicate marking) -> apply -> fetch, with tables gathered from the cases
and with crafted tables loaded through tables_put; the QUAL bytes are compared with the restatement (apply_ref.py) and with the oracle,
and kernel_stats() must name the kernel the case is meant for."""
import numpy as np
import pytest

import apply_cases as AC
import apply_ref
from elprep_b200 import sam, synth
from util import apply_plan, bqsr_paths, decode_bam

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ref():
    return AC.genome()


def _device(w, max_cycle, dense=None, bam=False, levels=0, sqq=None):
    """-> dict(perm, qoff, qual, stats[, tables][, bam_qual]) of one context run through the library"""
    from elprep_b200 import device
    ctx = device.Context(w.header, max_cycle=max_cycle, quantize_levels=levels, sqq=sqq, profile=True)
    try:
        if dense is not None:
            ctx.tables_put(dense)
            ctx.bqsr_finalize(None)
        else:
            ctx.set_reference(0, w.contig_bases[0])
            ctx.set_known_sites(0, w.sites[0])
        if bam:
            raw, offs = synth.encode_bam(w.batch, w.header)
            ctx.append_bam(raw, offs)
        else:
            ctx.append(w.batch)
        ctx.sort_markdup(device.SO_COORDINATE, False)
        res = {}
        if dense is None:
            ctx.bqsr_gather()
            res["tables"] = ctx.tables_get()
            ctx.bqsr_finalize(None)
        ctx.bqsr_apply()
        idx, _, qoff, qual = ctx.fetch()
        res.update(perm=idx.astype(np.int64), qoff=qoff, qual=qual[:int(qoff[-1])].copy(), stats=ctx.kernel_stats())
        if bam:
            raw, offs = ctx.fetch_bam()
            res["bam_qual"] = decode_bam(raw, offs, w.header).qual
        return res
    finally:
        ctx.close()


def _expect(w, max_cycle, dense=None, levels=0, sqq=None):
    """(output order, sorted batch, oracle QUAL, restatement QUAL, finalized tables) of the reference path"""
    import oracle
    perm = oracle.coordinate_sort(w.batch, n_threads=4)
    srt = w.batch.take(perm)
    if dense is None:
        t = oracle.bqsr_gather(srt, w.header, oracle.Reference(w.header, w.contig_bases, w.sites), max_cycle=max_cycle, n_threads=4)
        oracle.bqsr_finalize(t)
    else:
        t = AC.oracle_tables(dense, max_cycle)
    got, err = apply_ref.apply(srt, w.header, t, quantize_levels=levels, sqq=sqq)
    assert err is None, err
    b = srt.copy()
    oracle.bqsr_apply(b, w.header, t, quantize_levels=levels, sqq=sqq, n_threads=4)
    return perm, srt, b.qual, got, t


def _kernel(stats):
    return bqsr_paths(stats)[1]


def _no_quirks(w):
    b = w.batch
    qo = b.qual_off.astype(np.int64)
    for i in range(b.n):
        assert not apply_ref.context_quirk(apply_ref.bases_of(b, i), [int(x) for x in b.qual[qo[i]:qo[i + 1]]], int(b.flag[i])), i


# (name, specs(ref), header read groups, QUAL alphabet of the generated reads)
CONTEXTS = {
    "len32": (lambda r: AC.lengths_context(32), 4, (12, 23, 37)),
    "len33": (lambda r: AC.lengths_context(33), 4, (12, 23, 37)),
    "len100": (lambda r: AC.lengths_context(100), 4, (12, 23, 37)),
    "len512": (lambda r: AC.lengths_context(512), 4, (12, 23, 37)),
    "len1024": (lambda r: AC.lengths_context(1024), 1, (12, 37)),
    "short_in_1024": (lambda r: AC.many_short_in_long(), 1, (12, 37)),
    "tails": (lambda r: AC.tail_context(), 4, (12, 23, 37)),
    "bases": (lambda r: AC.base_context(r), 4, (12, 23, 37)),
    "quals": (lambda r: AC.qual_context(), 4, (12, 23, 37)),
    "quals_above_93": (lambda r: AC.qual_context(every_value=False), 4, (12, 23, 37)),
    "read_groups": (lambda r: AC.read_group_context(), 4, (12, 23, 37)),
}


def _context(name, ref):
    mk, n_rg, quals = CONTEXTS[name]
    specs = mk(ref)
    w, _ = AC.build(specs, AC.header(n_rg), ref, quals=quals)
    _no_quirks(w)
    return w, max(1, int(w.batch.lseq.max()))


def _phases(qoff, rpw):
    """16-byte phases at which the warp passes of bqsr_apply2_kernel start in the output stream"""
    return {int(qoff[k]) & 15 for k in range(0, len(qoff) - 1, rpw)}


@pytest.mark.parametrize("kernel", ["default", "v1"])
@pytest.mark.parametrize("tables", ["gathered", "crafted"])
@pytest.mark.parametrize("name", sorted(CONTEXTS))
def test_cases(name, tables, kernel, ref, monkeypatch):
    w, L = _context(name, ref)
    if kernel == "v1":
        if L > 512:
            pytest.skip("bqsr_apply_kernel refuses reads over 512 bases (test_v1_refuses_long_reads)")
        monkeypatch.setenv("ELPREP_B200_APPLY", "v1")
    n_cov = len(w.header.rg_cov_ids()[1])
    values = np.unique(w.batch.qual).tolist()
    dense = AC.crafted_dense(n_cov, L, [q for q in values if 6 <= q <= 93], empty_covs=(2,) if n_cov == 3 else (), longest=L) if tables == "crafted" else None
    g = _device(w, L, dense)
    perm, srt, oq, rq, _ = _expect(w, L, dense)
    want = "gmem" if kernel == "v1" else apply_plan(values, n_cov, L, L)
    assert _kernel(g["stats"]) == want, sorted(g["stats"])
    assert np.array_equal(g["perm"], perm), "output order differs"
    assert np.array_equal(g["qoff"], srt.qual_off)
    assert np.array_equal(rq, oq), "restatement and oracle differ"
    bad = np.nonzero(g["qual"] != rq)[0]
    assert bad.size == 0, f"{bad.size} QUAL bytes differ, first at output byte {bad[:8].tolist()}"
    assert np.count_nonzero(rq != srt.qual) > 0.2 * np.count_nonzero(srt.qual >= 6)   # apply changed many bases
    if name.startswith("len") and want == "v2":
        rpw = 32 // min(32, (L + 31) // 32)
        assert len(_phases(g["qoff"], rpw)) >= 14 or rpw == 1, "warp passes start at too few 16-byte phases"


def test_kernels_chosen_by_default(ref):
    """the contexts meant for bqsr_apply2_kernel do take it"""
    for name in ("len32", "len33", "len100", "len1024", "short_in_1024", "tails", "bases", "quals_above_93", "read_groups"):
        w, L = _context(name, ref)
        assert apply_plan(np.unique(w.batch.qual).tolist(), len(w.header.rg_cov_ids()[1]), L, L) == "v2", name
    w, L = _context("quals", ref)
    assert apply_plan(np.unique(w.batch.qual).tolist(), 3, L, L) == "gmem"


def test_bam_records(ref):
    """the same QUAL through elp_append_bam and elp_fetch_bam"""
    w, L = _context("quals_above_93", ref)
    dense = AC.crafted_dense(3, L, (12, 23, 37), empty_covs=(2,), longest=L)
    g = _device(w, L, dense, bam=True)
    _, srt, oq, rq, _ = _expect(w, L, dense)
    assert np.array_equal(g["qual"], rq) and np.array_equal(g["bam_qual"], rq)
    assert _kernel(g["stats"]) == "v2"


@pytest.mark.parametrize("levels,sqq", [(16, None), (0, [10, 20, 30]), (3, [7, 41])])
def test_quantization(levels, sqq, ref):
    w, L = _context("len100", ref)
    dense = AC.crafted_dense(3, L, (12, 23, 37), empty_covs=(2,), longest=L)
    g = _device(w, L, dense, levels=levels, sqq=sqq)
    _, _, oq, rq, _ = _expect(w, L, dense, levels=levels, sqq=sqq)
    assert np.array_equal(rq, oq) and np.array_equal(g["qual"], rq)


def test_crafted_tables_discriminate(ref):
    """the crafted tables tell the right key from a mirrored cycle, a forward-strand context on a reverse read, and a context shifted by
    one base: the restatement with each of these mistakes predicts another byte for at least 40 % of the recalibrated bases"""
    w, L = _context("len100", ref)
    dense = AC.crafted_dense(3, L, (12, 23, 37), empty_covs=(2,), longest=L)
    _, srt, _, _, t = _expect(w, L, dense)
    T = apply_ref.Tables(t)
    _, names = w.header.rg_cov_ids()
    cov_of = {n: k for k, n in enumerate(names)}
    n = {"mirrored": [0, 0], "forward": [0, 0], "shifted": [0, 0]}
    qo = srt.qual_off.astype(np.int64)
    for i in range(srt.n):
        cov = cov_of[apply_ref.read_group_covariate(w.header, int(srt.rg[i]))]
        if T.comb[cov] is None:
            continue
        f, bases, q = int(srt.flag[i]), apply_ref.bases_of(srt, i), [int(x) for x in srt.qual[qo[i]:qo[i + 1]]]
        keys = apply_ref.context_covariates(bases, q, f)
        fkeys = apply_ref.context_covariates(bases, q, f & ~sam.Reversed)
        cf, inc = apply_ref.cycle_covariates(f, len(q))
        for j, x in enumerate(q):
            if x < 6:
                continue
            cyc = cf + j * inc
            right = T.recalibrated(cov, x, cyc, keys[j])
            for k, alt in (("mirrored", T.recalibrated(cov, x, -cyc, keys[j])), ("shifted", T.recalibrated(cov, x, cyc, keys[j - 1] if j else -1)),
                           ("forward", T.recalibrated(cov, x, cyc, fkeys[j]) if f & sam.Reversed else None)):
                if alt is not None:
                    n[k][0] += alt != right
                    n[k][1] += 1
    for k, (d, tot) in n.items():
        assert tot > 1000 and d >= 0.4 * tot, (k, d, tot)


@pytest.mark.parametrize("L,values,above93,want", [(235, (12, 23, 37), False, "v2"), (236, (12, 23, 37), False, "gmem"),
                                                  (235, (12, 37), True, "v2"), (236, (12, 37), True, "gmem")])
def test_compact_table_size_switch(L, values, above93, want, ref):
    """3 covariates x 3 slots: the compact table is 81 856 bytes with reads of 235 bases and 82 176 with 236 (limit 80 KB); QUAL above
    93 counts as one more slot"""
    specs = [AC.spec(L, f) for f in AC.FLAGS.values()] + [AC.spec(int(x), 0x10) for x in range(1, 200, 7)]
    if above93:
        specs.append(AC.spec(50, 0x10, qual=[200, 12] * 25, kind="unmapped"))
    w, _ = AC.build(specs, AC.header(), ref, quals=values)
    vals = np.unique(w.batch.qual).tolist()
    assert apply_plan(vals, 3, L, L) == want
    dense = AC.crafted_dense(3, L, [q for q in vals if 6 <= q <= 93], empty_covs=(2,), longest=L)
    g = _device(w, L, dense)
    _, _, oq, rq, _ = _expect(w, L, dense)
    assert _kernel(g["stats"]) == want and np.array_equal(g["qual"], rq) and np.array_equal(rq, oq)


def test_v1_refuses_long_reads(ref, monkeypatch):
    from elprep_b200 import device
    monkeypatch.setenv("ELPREP_B200_APPLY", "v1")
    w, L = _context("len1024", ref)
    with pytest.raises(device.ElprepError) as ei:
        _device(w, L, AC.crafted_dense(1, L, (12, 37), longest=L))
    assert ei.value.code == -15 and "read longer than the device kernel supports" in str(ei.value)


# ---- errors: a read without RG (empty ones too), --max-cycle; what a fetch returns after a failed apply
def _fail(w, L, dense, code, text, kernel, monkeypatch, fetch_before=True):
    from elprep_b200 import device
    if kernel == "v1":
        monkeypatch.setenv("ELPREP_B200_APPLY", "v1")
    ctx = device.Context(w.header, max_cycle=L, profile=True)
    try:
        ctx.tables_put(dense)
        ctx.bqsr_finalize(None)
        raw, offs = synth.encode_bam(w.batch, w.header)
        ctx.append_bam(raw, offs)
        ctx.sort_markdup(device.SO_COORDINATE, False)
        if fetch_before:
            ctx.fetch()                                         # materialises the output QUAL stream first
        with pytest.raises(device.ElprepError) as ei:
            ctx.bqsr_apply()
        assert ei.value.code == code and text in str(ei.value), str(ei.value)
        # (reads longer than --max-cycle leave the compact table: it covers the cycles up to --max-cycle only)
        assert _kernel(ctx.kernel_stats()) == ("gmem" if kernel == "v1" else apply_plan(np.unique(w.batch.qual).tolist(), 3, int(w.batch.lseq.max()), L))
        idx, _, qoff, qual = ctx.fetch()
        srt = w.batch.take(idx.astype(np.int64))
        assert np.array_equal(qual[:int(qoff[-1])], srt.qual), "a fetch after a failed apply returns other than the original QUAL"
        raw, offs = ctx.fetch_bam()
        assert np.array_equal(decode_bam(raw, offs, w.header).qual, srt.qual)
    finally:
        ctx.close()


ERROR_CASES = {
    "no_rg": ([AC.spec(20), AC.spec(20, rg=None)] + [AC.spec(30, 0x10)] * 40, "ENORG"),
    "no_rg_empty_read": ([AC.spec(20)] * 40 + [AC.spec(0, qual=[], seq="", rg=None)] + [AC.spec(25, 0x10)] * 40, "ENORG"),
    "cycle_fwd": ([AC.spec(40)] * 10 + [AC.spec(41, 0x1 | 0x40)] + [AC.spec(40)] * 10, "ECYCLE"),
    "cycle_rev": ([AC.spec(40)] * 10 + [AC.spec(41, 0x80 | 0x10, qual=[6] + [30] * 40)] + [AC.spec(40)] * 10, "ECYCLE"),
    "cycle_last_base_low_fwd": ([AC.spec(40)] * 10 + [AC.spec(41, 0x1 | 0x80, qual=[30] * 40 + [5])], None),
    "cycle_last_base_low_rev": ([AC.spec(40)] * 10 + [AC.spec(41, 0x10, qual=[5] + [30] * 40)], None),
    "cycle_equal_max": ([AC.spec(40, f) for f in AC.FLAGS.values()], None),
}
CODES = {"ENORG": (-11, "requires input with read groups"), "ECYCLE": (-12, "cycle value exceeds maximum cycle value")}


@pytest.mark.parametrize("kernel", ["default", "v1"])
@pytest.mark.parametrize("name", sorted(ERROR_CASES))
def test_errors(name, kernel, ref, monkeypatch):
    """--max-cycle 40: a 41-base read fails where its base of cycle +-41 has QUAL >= 6, on either strand"""
    specs, err = ERROR_CASES[name]
    w, _ = AC.build(specs, AC.header(), ref)
    dense = AC.crafted_dense(3, 40, (12, 23, 37, 30, 6), empty_covs=(2,), longest=40)
    got, rerr = apply_ref.apply(w.batch, w.header, AC.oracle_tables(dense, 40))
    assert rerr == err
    if err is None:
        if kernel == "v1":
            monkeypatch.setenv("ELPREP_B200_APPLY", "v1")
        g = _device(w, 40, dense)
        _, _, oq, rq, _ = _expect(w, 40, dense)
        assert np.array_equal(g["qual"], rq)
        return
    _fail(w, 40, dense, *CODES[err], kernel, monkeypatch)


def test_invalid_qual_without_duplicate_marking(ref):
    """QUAL 100 in a read that enters duplicate marking: an error of MarkDuplicates only; sorted without marking, the read is recalibrated
    with its read group's estimate (QUAL above 93 has no table entries)"""
    from elprep_b200 import device
    specs = [AC.spec(30, 0, qual=[100] + [12] * 29)] + [AC.spec(30, 0x10)] * 20
    w, _ = AC.build(specs, AC.header(), ref)
    dense = AC.crafted_dense(3, 30, (12, 23, 37), empty_covs=(2,), longest=30)
    ctx = device.Context(w.header, max_cycle=30)
    try:
        ctx.append(w.batch)
        with pytest.raises(device.ElprepError) as ei:
            ctx.sort_markdup(device.SO_COORDINATE, True)
        assert ei.value.code == -10 and "Invalid QUAL character" in str(ei.value)
    finally:
        ctx.close()
    g = _device(w, 30, dense)
    _, srt, oq, rq, _ = _expect(w, 30, dense)
    assert np.array_equal(g["qual"], rq) and np.array_equal(rq, oq)
    assert rq[int(np.nonzero(srt.qual == 100)[0][0])] != 100


def test_gather_refuses_counted_qual_above_93(ref):
    """a base with QUAL above 93 that the gather would count (a mapped, MAPQ > 0 read): refused, and no tables are produced"""
    from elprep_b200 import device
    w, _ = AC.build([AC.spec(30, 0, qual=[94] + [12] * 29)] + [AC.spec(30)] * 5, AC.header(), ref)
    ctx = device.Context(w.header, max_cycle=30)
    try:
        ctx.set_reference(0, w.contig_bases[0])
        ctx.set_known_sites(0, w.sites[0])
        ctx.append(w.batch)
        ctx.sort_markdup(device.SO_COORDINATE, False)
        with pytest.raises(device.ElprepError) as ei:
            ctx.bqsr_gather()
        assert ei.value.code == -15 and "QUAL > 93 in a recalibrated read" in str(ei.value)
        with pytest.raises(device.ElprepError) as ei:
            ctx.bqsr_finalize(None)
        assert ei.value.code == -16
    finally:
        ctx.close()


# ---- the no-table path, apply twice, apply across elp_reset
def test_no_table_path(ref):
    """fetch without BQSR: reads up to 1024 bases (bqsr_apply2_kernel without a table) and longer ones (qual_copy_kernel), with empty reads"""
    from elprep_b200 import device
    for longest in (1024, 3000):
        specs = [AC.spec(x, f) for x in (0, 1, 17, 0, 1024, longest, 0, 33) for f in (0, 0x10)] + [AC.spec(0)] * 50 + [AC.spec(int(x)) for x in range(0, 300, 13)]
        w, _ = AC.build(specs, AC.header(), ref)
        ctx = device.Context(w.header, profile=True)
        try:
            ctx.append(w.batch)
            ctx.sort_markdup(device.SO_COORDINATE, False)
            idx, _, qoff, qual = ctx.fetch()
            assert "qual_materialize" in ctx.kernel_stats()
        finally:
            ctx.close()
        assert np.array_equal(qual[:int(qoff[-1])], w.batch.take(idx.astype(np.int64)).qual)


@pytest.mark.parametrize("kernel", ["default", "v1"])
def test_apply_twice_and_across_reset(kernel, ref, monkeypatch):
    from elprep_b200 import device
    if kernel == "v1":
        monkeypatch.setenv("ELPREP_B200_APPLY", "v1")
    w1, L1 = _context("len100", ref)
    w2, _ = AC.build(AC.lengths_context(64, seed=8), AC.header(), ref)
    dense = AC.crafted_dense(3, 100, (12, 23, 37), empty_covs=(2,), longest=100)
    ctx = device.Context(w1.header, max_cycle=100, profile=True)
    try:
        ctx.tables_put(dense)
        ctx.bqsr_finalize(None)
        for k, w in enumerate((w1, w2)):
            if k:
                ctx.reset()
                ctx.tables_put(dense)
                ctx.bqsr_finalize(None)
            ctx.append(w.batch)
            ctx.sort_markdup(device.SO_COORDINATE, False)
            _, _, _, rq, _ = _expect(w, 100, dense)
            for _ in range(2):                                   # apply twice: the second reads the original QUAL again
                ctx.bqsr_apply()
                _, _, qoff, qual = ctx.fetch()
                assert np.array_equal(qual[:int(qoff[-1])], rq)
            assert _kernel(ctx.kernel_stats()) == ("gmem" if kernel == "v1" else "v2")
    finally:
        ctx.close()


# ---- a large mixed workload against the oracle
def _mixed(n, longest, seed, n_rg=1, chunk=1 << 16):
    """n reads of 0..longest bases (1 % empty), every flag combination of apply_cases.FLAGS, 2 % unmapped and 2 % secondary, QUAL 12 / 37
    with low-quality prefixes and suffixes of 0, 11, 22 or 33 bases, 1 % N bases"""
    rng = np.random.default_rng(seed)
    L = rng.integers(1, longest + 1, size=n).astype(np.int32)
    L[rng.random(n) < 0.01] = 0
    flags = np.array(list(AC.FLAGS.values()), np.uint16)[rng.integers(0, len(AC.FLAGS), size=n)]
    flags |= np.where(rng.random(n) < 0.02, 0x4, 0).astype(np.uint16) | np.where(rng.random(n) < 0.02, 0x100, 0).astype(np.uint16)
    qo, so = np.zeros(n + 1, np.int64), np.zeros(n + 1, np.int64)
    np.cumsum(L, out=qo[1:])
    np.cumsum((L + 1) // 2, out=so[1:])
    qual, seq = np.empty(int(qo[-1]), np.uint8), np.zeros(int(so[-1]), np.uint8)
    head, tail = 11 * rng.integers(0, 4, size=n), 11 * rng.integers(0, 4, size=n)
    for c0 in range(0, n, chunk):                                    # (chunks keep the int64 temporaries small)
        c1 = min(n, c0 + chunk)
        Lc = L[c0:c1].astype(np.int64)
        tot = int(Lc.sum())
        k = np.arange(tot) - np.repeat(qo[c0:c1] - qo[c0], Lc)       # base k of its read
        q = rng.choice(np.array([12, 12, 37], np.uint8), size=tot)
        q[(k < np.repeat(head[c0:c1], Lc)) | (k >= np.repeat(Lc - tail[c0:c1], Lc))] = 2
        qual[qo[c0]:qo[c1]] = q
        nib = rng.choice(np.array([1, 2, 4, 8], np.uint8), size=tot)
        nib[rng.random(tot) < 0.01] = 15
        byte = np.repeat(so[c0:c1], Lc) + (k >> 1)
        even = (k & 1) == 0
        seq[byte[even]] = nib[even] << 4
        seq[byte[~even]] |= nib[~even]
    mapped = (flags & 0x4) == 0
    pos = np.where(mapped, rng.integers(1, 300_000, size=n), 0).astype(np.int32)
    names = np.frombuffer(b"".join(b"m%08d" % i for i in range(n)), np.uint8)
    b = sam.AlignmentBatch(refid=np.where(mapped, 0, -1), pos=pos, flag=flags, mapq=np.full(n, 60), nref=np.full(n, -1), pnext=np.zeros(n),
                           tlen=np.zeros(n), rg=rng.integers(0, n_rg, size=n), qname_off=np.arange(n + 1, dtype=np.uint64) * 9, qname=names,
                           cigar_off=np.zeros(n + 1, np.uint64), cigar=np.zeros(0, np.uint32), lseq=L, seq=seq, qual=qual)
    return synth.Workload(AC.header(n_rg), b, [None], [np.zeros((0, 2), np.int32)], {})


@pytest.mark.parametrize("kernel,longest", [("default", 1024), ("v1", 512)])
def test_million_mixed_reads(kernel, longest, monkeypatch):
    import oracle
    if kernel == "v1":
        monkeypatch.setenv("ELPREP_B200_APPLY", "v1")
    w = _mixed(1_000_000, longest, seed=longest)
    dense = AC.crafted_dense(1, longest, (12, 37), longest=longest)
    g = _device(w, longest, dense)
    assert _kernel(g["stats"]) == ("gmem" if kernel == "v1" else "v2")
    perm = oracle.coordinate_sort(w.batch, n_threads=8)
    srt = synth.take(w.batch, perm)
    oracle.bqsr_apply(srt, w.header, AC.oracle_tables(dense, longest), n_threads=8)
    assert np.array_equal(g["perm"], perm)
    bad = np.nonzero(g["qual"] != srt.qual)[0]
    assert bad.size == 0, f"{bad.size} QUAL bytes differ, first at {bad[:8].tolist()}"
