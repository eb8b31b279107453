"""GPU parity: the CUDA path, called through the C ABI, against the oracle on the same seeded inputs.
Bit-exact for FLAG (0x400 bits), output order, table counters, EmpiricalQuality, report text and QUAL bytes."""
import numpy as np
import pytest

from elprep_b200 import sam, synth
from util import gpu_pipeline, oracle_pipeline, oracle_tables_dense

pytestmark = pytest.mark.gpu

SMALL = [("chr20", 600_000), ("chr21", 300_000), ("chrM", 16_569)]


def _ctx():
    from elprep_b200 import device
    return device.Context(sam.Header(sq=[{"SN": "c", "LN": 1000}]))


@pytest.mark.parametrize("n,bits", [(0, 8), (1, 8), (5, 3), (1000, 17), (6144, 34), (6145, 34), (100_000, 52), (1_000_003, 40), (300_000, 64), (200_000, 1)])
def test_radix_sort_u64(n, bits):
    rng = np.random.default_rng(n + bits)
    keys = rng.integers(0, 2 ** 63, size=n, dtype=np.uint64) * np.uint64(2) + rng.integers(0, 2, size=n, dtype=np.uint64)
    if bits < 64:
        keys &= np.uint64((1 << bits) - 1)
    if n > 100:
        keys[rng.integers(0, n, size=n // 3)] = keys[0]      # many duplicates: stability matters
    vals = np.arange(n, dtype=np.uint32)
    ctx = _ctx()
    k2, v2 = ctx.debug_sort_u64(keys, vals, bits)
    order = np.argsort(keys, kind="stable")
    assert np.array_equal(k2, keys[order]) and np.array_equal(v2, vals[order])
    ctx.close()


@pytest.mark.parametrize("n,bits", [(0, 70), (3, 70), (4096, 87), (4097, 87), (250_000, 128), (100_000, 65)])
def test_radix_sort_u128(n, bits):
    rng = np.random.default_rng(n + bits)
    lo = rng.integers(0, 2 ** 63, size=n, dtype=np.uint64) * np.uint64(2) + rng.integers(0, 2, size=n, dtype=np.uint64)
    hi = rng.integers(0, 2 ** 63, size=n, dtype=np.uint64)
    hb = bits - 64
    hi &= np.uint64((1 << hb) - 1) if hb < 64 else np.uint64(2 ** 64 - 1)
    if n > 100:
        dup = rng.integers(0, n, size=n // 3); hi[dup] = hi[0]; lo[dup] = lo[0]
    vals = np.arange(n, dtype=np.uint32)
    ctx = _ctx()
    h2, l2, v2 = ctx.debug_sort_u128(hi, lo, vals, bits)
    order = np.lexsort((lo, hi))      # stable, hi most significant
    assert np.array_equal(h2, hi[order]) and np.array_equal(l2, lo[order]) and np.array_equal(v2, vals[order])
    ctx.close()


def _compare(w, g, o, bqsr=True):
    assert np.array_equal(g["perm"], o["perm"]), "output order differs"
    assert np.array_equal(g["flag"], o["flag"]), "FLAG differs"
    assert np.array_equal(g["qual_off"], o["qual_off"])
    if bqsr:
        d, e = oracle_tables_dense(o["tables"], 500)
        assert np.array_equal(g["tables"], d), "BQSR table counters differ"
        assert np.array_equal(g["emp"], e), "EmpiricalQuality differs"
        assert g["report"] == o["report"], "recalibration report text differs"
    assert np.array_equal(g["qual"], o["qual"]), "QUAL bytes differ"


def test_adapt_matches_oracle(orc):
    w = synth.make_workload(20_000, SMALL, seed=11, want_reference=False)
    from elprep_b200 import device
    ctx = device.Context(w.header)
    ctx.append(w.batch)
    up, sc = ctx.debug_adapt()
    b = w.batch.copy()
    ou, os_ = orc.mark_duplicates(b, w.header, want_adapt=True)
    enter = (w.batch.flag & 0x904) == 0
    assert np.array_equal(up[enter], ou[enter]) and np.array_equal(sc[enter], os_[enter])
    ctx.close()


@pytest.mark.parametrize("seed,kw", [(1, {}), (2, dict(exome=True)), (3, dict(wide_quals=True)), (4, dict(dup_frac=0.5, optical_frac=0.5)),
                                      (5, dict(unmapped_frac=0.3)), (6, dict(n_rg=1)), (7, dict(n_rg=0))])
def test_full_path_small(seed, kw):
    w = synth.make_workload(15_000, SMALL, seed=seed, **kw)
    bqsr = kw.get("n_rg", 4) != 0     # without read groups BQSR panics in the reference; sort+markdup still run
    g = gpu_pipeline(w, bqsr=bqsr, n_batches=3)
    o = oracle_pipeline(w, bqsr=bqsr)
    _compare(w, g, o, bqsr)
    assert int(((g["flag"] & 0x400) != 0).sum()) > 0 or kw.get("unmapped_frac", 0) > 0.2


@pytest.mark.parametrize("L", [36, 75, 100, 151, 250, 300])
def test_read_lengths(L):
    """other read lengths: the BQSR chunk kernels give every read ceil(L/16) lanes, so 36 / 75 / 100 / 151 / 250 / 300 bases mean
    10 / 6 / 4 / 3 / 2 / 1 reads per warp step (and a partial last chunk of every size)"""
    w = synth.make_workload(4_000, SMALL, seed=100 + L, L=L)
    assert int(w.batch.lseq.max()) == L
    g = gpu_pipeline(w, n_batches=2)
    o = oracle_pipeline(w)
    _compare(w, g, o)


def test_mixed_read_lengths():
    """reads of 20 to 300 bases in one context (lanes per read follow the longest)"""
    a = synth.make_workload(2_000, SMALL, seed=201, L=150)
    parts = [a.batch] + [synth.make_workload(600, SMALL, seed=202 + k, L=L, genome_seed=201, pair_id_base=(k + 1) << 24, want_reference=False).batch
                         for k, L in enumerate((20, 32, 33, 49, 100, 151, 250, 300))]
    w = synth.Workload(a.header, sam.AlignmentBatch.concat(parts), a.contig_bases, a.sites, a.params)
    assert int(w.batch.lseq.min()) == 20 and int(w.batch.lseq.max()) == 300
    g = gpu_pipeline(w, n_batches=3)
    o = oracle_pipeline(w)
    _compare(w, g, o)


def test_full_path_c1_shape():
    """config[0] shape (single contig), 200k reads: sort + markdup + BQSR"""
    w = synth.make_workload(100_000, [("chr20", 6_444_416)], seed=20260924)
    g = gpu_pipeline(w, n_batches=4)
    o = oracle_pipeline(w, threads=8)
    _compare(w, g, o)


def test_no_sort_keep_order():
    w = synth.make_workload(5_000, SMALL, seed=9)
    g = gpu_pipeline(w, sort=False)
    o = oracle_pipeline(w, sort=False)
    _compare(w, g, o)
    assert np.array_equal(g["perm"], np.arange(w.batch.n, dtype=np.uint64))


def test_sqq_and_quantize():
    w = synth.make_workload(8_000, SMALL, seed=21)
    g = gpu_pipeline(w, quantize_levels=4, sqq=[10, 20, 30])
    o = oracle_pipeline(w, quantize_levels=4, sqq=[10, 20, 30])
    _compare(w, g, o)


def test_long_tie_runs_and_unmapped_block():
    """many reads at identical (refid,pos,strand) and a large unmapped block: exercises the long-run tie-break path"""
    w = synth.make_workload(6_000, [("chr20", 3_000)], seed=31, unmapped_frac=0.4, dup_frac=0.6)
    g = gpu_pipeline(w, bqsr=False)
    o = oracle_pipeline(w, bqsr=False)
    _compare(w, g, o, bqsr=False)


def test_empty_and_single():
    h = synth.make_header(SMALL)
    from elprep_b200 import device
    ctx = device.Context(h)
    ctx.sort_markdup()
    idx, flag, qoff, qual = ctx.fetch()
    assert idx.size == 0 and flag.size == 0
    ctx.close()
    w = synth.make_workload(1, SMALL, seed=3)
    _compare(w, gpu_pipeline(w), oracle_pipeline(w))


def _adversarial_records(quals=(2, 2, 5, 6, 12, 23, 37, 40)):
    """hand-built reads covering clip/indel/adaptor/N/low-qual-tail corner cases (SURVEY.md Appendix C); QUAL drawn from ``quals``"""
    rng = np.random.default_rng(77)
    recs, L = [], 60
    cigars = ["60M", "5S55M", "55M5S", "3H5S50M5S", "20M3I37M", "20M4D40M", "10S20M2I10M3D18M", "5S20M5D30M5S", "1M1I58M", "58M1I1M",
              "2S10M2D10M2I10M2D10M2I14M", "30M30S", "30S30M", "10M10N40M"]
    for t in range(400):
        c = cigars[t % len(cigars)]
        pos = 1000 + int(rng.integers(0, 400))
        rev = bool(rng.integers(0, 2))
        paired = rng.random() < 0.8
        flag = (0x1 | (0x40 if rng.random() < .5 else 0x80)) if paired else 0
        if rev:
            flag |= 0x10
        elif paired:
            flag |= 0x20
        ins = int(rng.integers(20, 160))
        pnext = pos - ins + 50 if rev else pos + ins - 50
        tlen = (-ins if rev else ins) if paired else 0
        q = rng.choice(list(quals), size=L).astype(int)
        if t % 7 == 0:
            q[:8] = 2
        if t % 11 == 0:
            q[-9:] = 1
        seq = "".join(rng.choice(list("ACGTN"), p=[.24, .24, .24, .24, .04], size=L))
        recs.append(dict(QNAME=f"adv{t:04d}" if paired else f"frag{t:04d}", FLAG=flag, RNAME="chr20", POS=pos, MAPQ=int(rng.choice([0, 30, 60, 255])),
                         CIGAR=c, RNEXT="=" if paired else "*", PNEXT=max(1, pnext) if paired else 0, TLEN=tlen, SEQ=seq, QUAL=[int(x) for x in q],
                         RG=["rg1", "rg2", "rg3", "rg4"][t % 4]))
    return recs


def _adversarial_run(quals):
    contigs = [("chr20", 4_000)]
    base = synth.make_workload(10, contigs, seed=5)       # header + reference + sites
    b = sam.AlignmentBatch.from_records(base.header, _adversarial_records(quals))
    assert set(np.unique(b.qual).tolist()) == set(quals) | {1}
    sites = [np.array([[1005, 1005], [1100, 1109], [1200, 1200], [1250, 1300]], dtype=np.int32)]
    w = synth.Workload(base.header, b, base.contig_bases, sites, {})
    g = gpu_pipeline(w, profile=True)
    _compare(w, g, oracle_pipeline(w))
    return g


def test_adversarial_clipping_cases():
    """five QUAL values >= 6: the general kernels gather every read"""
    from util import bqsr_paths
    g = _adversarial_run((2, 2, 5, 6, 12, 23, 37, 40))
    assert bqsr_paths(g["stats"])[0] == "general", sorted(g["stats"])


def test_adversarial_clipping_cases_fast_path():
    """the same reads with an alphabet the count kernel accepts ({1,2,3,12,23,37}: S = 3, six values): checks closed_form_clip on the
    device, <= 2 known-site ranges, the indel records and the hand-off of the remaining reads to the general kernels (cx_list), both
    adding into one table"""
    from util import bqsr_paths
    g = _adversarial_run((2, 3, 12, 23, 37))
    assert bqsr_paths(g["stats"])[0] == "fast", sorted(g["stats"])
    assert g["stats"]["bqsr_g_count"]["launches"] and g["stats"]["bqsr_g_count_indel"]["launches"]
    assert "bqsr_g_prep" in g["stats"], "no read was handed to the general kernels"


def test_invalid_qual_is_an_error():
    from elprep_b200 import device
    w = synth.make_workload(200, SMALL, seed=8, want_reference=False)
    w.batch.qual[5] = 100
    ctx = device.Context(w.header)
    ctx.append(w.batch)
    with pytest.raises(device.ElprepError) as ei:
        ctx.sort_markdup()
    assert ei.value.code == -10 and "Invalid QUAL character" in str(ei.value)
    ctx.close()


def test_reference_style_api():
    """the phase order of runBestPracticesPipelineIntermediateSam (cmd/filter.go:142-211) through the mirrored operator API"""
    import os
    import tempfile
    from elprep_b200 import filters
    w = synth.make_workload(6_000, SMALL, seed=41)
    n = w.batch.n
    batches = [w.batch.take(np.arange(a, b)) for a, b in ((0, n // 2), (n // 2, n))]
    reads = filters.DeviceSam()
    md, fragments, pairs = filters.MarkDuplicates(False)
    filters.InputBatches(w.header, batches).RunPipeline(reads, [filters.AddREFID, md], sam.Coordinate)      # phase 1
    assert w.header.HDSO() == sam.Coordinate
    recal = filters.NewBaseRecalibrator(w.sites, w.contig_bases)
    tables = recal.Recalibrate(reads, 500)                                                                  # phase 3
    with tempfile.TemporaryDirectory() as d:
        tables.FinalizeBQSRTables()
        tables.PrintBQSRTables(os.path.join(d, "x.recal"))                                                  # phase 4
        report = open(os.path.join(d, "x.recal")).read()
    reads.RunPipeline(reads, [tables.ApplyBQSR(0, [], 500)], sam.Keep)                                      # phase 5
    out = filters.HostResult()
    reads.RunPipeline(out, [], sam.Keep)                                                                    # phase 6
    o = oracle_pipeline(w)
    assert np.array_equal(out.record_index, o["perm"]) and np.array_equal(out.flag, o["flag"])
    assert np.array_equal(out.qual[:int(out.qual_off[-1])], o["qual"]) and report == o["report"]


# ---- duplication metrics / optical duplicates (filters.MarkOpticalDuplicates, SURVEY.md §8 a9) ----
def _optical_both(w, pixel=100, n_batches=1, tmp=None):
    import oracle
    from elprep_b200 import device, _lib
    b = w.batch.copy()
    oracle.mark_duplicates(b, w.header, n_threads=1)
    perm = oracle.coordinate_sort(b, n_threads=4)                       # the reference visits the sorted reads (:470-494)
    b2 = w.batch.copy()
    om = oracle.markdup_optical(b2, w.header, order=perm, pixel_distance=pixel,
                                metrics_path=(tmp + "/o.txt") if tmp else None, command_line="elprep filter a b", started_on="now")
    ctx = device.Context(w.header, optical_pixel_distance=pixel)
    n = w.batch.n
    bounds = [n * i // n_batches for i in range(n_batches + 1)]
    for a, e in zip(bounds[:-1], bounds[1:]):
        ctx.append(w.batch.take(np.arange(a, e)))
    ctx.sort_markdup(device.SO_COORDINATE, _lib.MARKDUP_OPTICAL)
    gm = ctx.optical_metrics()
    assert ctx.optical_libraries() == om.lib_names
    idx, flag, _, _ = ctx.fetch()
    assert np.array_equal(idx, perm.astype(np.uint64)) and np.array_equal(flag, b2.flag[perm])
    for slot, g in enumerate(gm):
        for k_g, k_o in zip(_lib.ElpDupMetrics.COUNTERS, oracle.COUNTERS):
            assert g[k_g] == om.counters[slot][k_o], (slot, k_g)
        assert g["hist"] == om.hist[slot], slot
        assert g["estimated_library_size"] == om.library_size[slot]
        assert g["percent_duplication"] == om.percent_duplication[slot] or (np.isnan(g["percent_duplication"]) and np.isnan(om.percent_duplication[slot]))
        assert g["roi"] == om.roi[slot]
    if tmp:
        ctx.print_duplicates_metrics(tmp + "/g.txt", "elprep filter a b", "now")
        assert open(tmp + "/g.txt").read() == open(tmp + "/o.txt").read()
    ctx.close()
    return om


@pytest.mark.parametrize("seed,kw", [(3, dict(dup_frac=0.3, optical_frac=0.4)), (4, dict(dup_frac=0.1, optical_frac=0.2, n_rg=1)),
                                     (5, dict(dup_frac=0.5, optical_frac=0.5, unmapped_frac=0.2, exome=True))])
def test_optical_metrics(seed, kw, tmp_path):
    w = synth.make_workload(20_000, SMALL, seed=seed, want_reference=False, **kw)
    om = _optical_both(w, n_batches=3, tmp=str(tmp_path))
    assert sum(c["read_pair_optical_duplicates"] for c in om.counters) > 100


def test_optical_long_runs_and_pixel_distance(tmp_path):
    # 97 % duplicates of ~100 roots: runs far longer than 32 pairs take the block kernel (lock-free union-find)
    w = synth.make_workload(4_000, [("chr20", 200_000)], seed=9, dup_frac=0.97, optical_frac=0.6, unmapped_frac=0.0, want_reference=False, n_rg=1)
    om = _optical_both(w, tmp=str(tmp_path))
    assert max(max(h[0]) for h in om.hist if h[0]) > 64
    _optical_both(w, pixel=10)
    _optical_both(w, pixel=3000)


def test_optical_hand_cases():
    from elprep_b200 import device, _lib
    import oracle
    h = sam.Header(sq=[{"SN": "chr1", "LN": 100000}], rg=[{"ID": "rg1", "LB": "libA"}, {"ID": "rg2", "LB": "libA"}, {"ID": "rg3"}])
    def R(q, flag, pos, score, rg="rg1", **kw):
        return dict(QNAME=q, FLAG=flag, RNAME="chr1", POS=pos, CIGAR="4M", SEQ="ACGT", QUAL=[score] * 4, RG=rg, **kw)
    def pair(q, p1, p2, score, flags=(99, 147), rg="rg1"):
        return [R(q, flags[0], p1, score, RNEXT="=", PNEXT=p2, rg=rg), R(q, flags[1], p2, score, RNEXT="=", PNEXT=p1, rg=rg)]
    cases = {
        "strand lists": pair("M:1:F:1:7:100:100", 100, 300, 40) + pair("M:2:F:1:7:101:101", 100, 300, 30) + pair("M:3:F:1:7:102:102", 100, 300, 20, flags=(163, 83)),
        "read groups": pair("M:1:F:1:7:100:100", 100, 300, 40) + pair("M:2:F:1:7:101:101", 100, 300, 30, rg="rg2"),
        "five columns": pair("F:1:7:100:200", 100, 300, 40) + pair("F:1:7:110:210", 100, 300, 30),
        "no tile info": pair("a:7:100:200", 100, 300, 40) + pair("b:7:100:200", 100, 300, 30),
        "signs": pair("F:1:+7:-5:+20", 100, 300, 40) + pair("F:1:7:5:20", 100, 300, 30),
        "unparsed singleton": pair("F:1:7:100:2x0", 100, 300, 40) + pair("F:1:7:110:210", 500, 700, 30),
        "preset flags": pair("M:1:F:1:1:10:10", 100, 300, 40, flags=(99 | 0x400, 147 | 0x400)) + pair("M:2:F:1:1:20:20", 100, 300, 30),
        "single pair": pair("M:1:F:1:1:10:10", 100, 300, 40),
        "no pairs": [R("f1", 0, 10, 30), R("f2", 0, 10, 20), R("u", 4, 0, 30), R("n", 0, 50, 30, rg="rg3")],
    }
    for name, recs in cases.items():
        b = sam.AlignmentBatch.from_records(h, recs)
        om = oracle.markdup_optical(b.copy(), h)
        ctx = device.Context(h)
        ctx.append(b)
        ctx.sort_markdup(device.SO_KEEP, _lib.MARKDUP_OPTICAL)
        gm = ctx.optical_metrics()
        for slot, g in enumerate(gm):
            assert [g[k] for k in _lib.ElpDupMetrics.COUNTERS] == [om.counters[slot][k] for k in oracle.COUNTERS], name
            assert g["hist"] == om.hist[slot], name
        ctx.close()
    # a tile field that does not parse, inside a list of two: the reference panics in strconv.ParseInt
    b = sam.AlignmentBatch.from_records(h, pair("F:1:7:100:2x0", 100, 300, 40) + pair("F:1:7:110:210", 100, 300, 30))
    ctx = device.Context(h)
    ctx.append(b)
    with pytest.raises(device.ElprepError) as ei:
        ctx.sort_markdup(device.SO_KEEP, _lib.MARKDUP_OPTICAL)
    assert ei.value.code == -17 and "ParseInt" in str(ei.value)
    ctx.close()
    # metrics asked for without the optical pass
    ctx = device.Context(h)
    ctx.append(b)
    ctx.sort_markdup(device.SO_KEEP, True)
    with pytest.raises(device.ElprepError):
        ctx.optical_metrics()
    ctx.close()


def test_two_workers_spread_pairs_on_device():
    """two contig-group workers in one process (threads stand in for ranks): cross-group pairs are exchanged
    (elprep_b200.multi), duplicate flags and the merged duplication metrics equal the whole-file run of the oracle"""
    import threading
    import oracle
    from elprep_b200 import device, multi, _lib
    contigs = [("c1", 300_000), ("c2", 250_000), ("c3", 120_000), ("c4", 80_000)]
    w = synth.make_workload(6000, contigs, seed=92, cross_contig_frac=0.3, dup_frac=0.4, optical_frac=0.3, want_reference=False)
    whole = w.batch.copy()
    wm = oracle.markdup_optical(whole, w.header)
    world = 2
    groups = multi.contig_groups(contigs, world)
    owner = multi.owner_table(w.header, groups)
    slots, bar, out, errs = [None] * world, threading.Barrier(world), [None] * world, []

    def gather_for(rank):
        def gather(obj):
            slots[rank] = obj
            bar.wait()
            res = list(slots)
            bar.wait()
            return res
        return gather

    def worker(rank):
        try:
            own = multi.partition(w.batch, owner, rank, world)
            sub = w.batch.take(own)
            sm = multi.exchange_spread_duplicates(sub, w.header, owner, rank, world, multi.device_markdup(0, optical=True), gather_for(rank))
            ctx = device.Context(w.header)
            ctx.append(sub)
            ctx.sort_markdup(device.SO_COORDINATE, _lib.MARKDUP_OPTICAL)
            multi.merge_spread_metrics(ctx, sm)
            idx, flag, _, _ = ctx.fetch(want_qual=False)
            fl = np.empty(sub.n, np.uint16); fl[idx.astype(np.int64)] = flag
            out[rank] = (own, fl, ctx.optical_metrics())
            ctx.close()
        except Exception as e:      # noqa: BLE001
            errs.append(e)
            bar.abort()

    th = [threading.Thread(target=worker, args=(r,)) for r in range(world)]
    for t in th: t.start()
    for t in th: t.join()
    assert not errs, errs
    for own, fl, _ in out:
        assert np.array_equal(fl, whole.flag[own])
    # sum of the workers' metrics (mergeDuplicatesCtrMaps) == whole-file metrics
    ctx = device.Context(w.header)
    for slot in range(len(wm.counters)):
        for _, _, m in out:
            c7 = [m[slot][k] for k in _lib.ElpDupMetrics.COUNTERS]
            c7[1] = m[slot]["paired_reads_examined"]
            ctx.optical_merge(slot, c7, m[slot]["hist"])
    tot = ctx.optical_metrics()
    for slot, g in enumerate(tot):
        assert [g[k] for k in _lib.ElpDupMetrics.COUNTERS] == [wm.counters[slot][k] for k in oracle.COUNTERS], slot
        assert g["hist"] == wm.hist[slot] and g["estimated_library_size"] == wm.library_size[slot]
    ctx.close()


# ---- BAM records parsed on the device (SURVEY.md §8f row 1: sam/bam-files.go:314-400) ----
def test_bam_ingest_equals_column_ingest():
    """elp_append_bam over encoded records gives the same sorted order, FLAGs, BQSR tables and QUAL bytes as elp_append_batch
    over the columns -- and both equal the oracle"""
    from elprep_b200 import device
    from util import encode_bam
    w = synth.make_workload(6_000, SMALL, seed=17, unmapped_frac=0.05)
    o = oracle_pipeline(w)
    raw, offs = encode_bam(w.batch, w.header)
    nrec = offs.size - 1
    cuts = [0, nrec // 3, nrec // 2, nrec]                      # three calls; the last one lets the library walk the block_size chain
    ctx = device.Context(w.header)
    for ci in range(len(w.header.SQ)):
        ctx.set_reference(ci, w.contig_bases[ci]); ctx.set_known_sites(ci, w.sites[ci], already_flat=True)
    for a, b in zip(cuts[:-1], cuts[1:]):
        part = raw[int(offs[a]):int(offs[b])]
        ctx.append_bam(part, (offs[a:b + 1] - offs[a]) if b != nrec else None)
    assert ctx.n == w.batch.n
    ctx.sort_markdup()
    ctx.bqsr_gather(); ctx.bqsr_finalize(None); ctx.bqsr_apply()
    idx, flag, qoff, qual = ctx.fetch()
    assert np.array_equal(idx, o["perm"]) and np.array_equal(flag, o["flag"])
    assert np.array_equal(qoff, o["qual_off"]) and np.array_equal(qual[:int(qoff[-1])], o["qual"])
    d, _ = oracle_tables_dense(o["tables"], 500)
    assert np.array_equal(ctx.tables_get(), d)
    # egress: the stored records in output order with FLAG and QUAL patched, everything else byte-identical
    from util import decode_bam
    out, ooff = ctx.fetch_bam()
    b2 = decode_bam(out, ooff, w.header)
    srt = w.batch.take(o["perm"].astype(np.int64))
    assert np.array_equal(b2.flag, o["flag"]) and np.array_equal(b2.qual, o["qual"])
    for f in ("refid", "pos", "mapq", "nref", "pnext", "tlen", "rg", "qname", "qname_off", "cigar", "cigar_off", "lseq", "seq"):
        assert np.array_equal(getattr(b2, f), getattr(srt, f)), f
    for k in (0, 1, 77, int(ooff.size) - 2):                              # optional fields untouched
        i = int(o["perm"][k]); L = int(w.batch.lseq[i])
        rin, rout = raw[int(offs[i]):int(offs[i + 1])], out[int(ooff[k]):int(ooff[k + 1])]
        tail = 36 + int(rin[12]) + 4 * int(rin[16] | (rin[17] << 8)) + (L + 1) // 2 + L
        assert rin.size == rout.size and np.array_equal(rin[tail:], rout[tail:]) and np.array_equal(rin[:18], rout[:18])
    part, poff = ctx.fetch_bam(100, 50)                                    # a sub-range
    assert np.array_equal(part, out[int(ooff[100]):int(ooff[150])]) and np.array_equal(poff, ooff[100:151] - ooff[100])
    ctx.close()


def test_bam_ingest_errors():
    from elprep_b200 import device
    from util import encode_bam
    w = synth.make_workload(300, SMALL, seed=18, want_reference=False)
    raw, offs = encode_bam(w.batch, w.header, with_aux=False)
    # an RG:Z value the header does not know (the reference would invent a table entry; here it is an error)
    h2 = sam.Header(sq=w.header.SQ, rg=[{"ID": "other"}])
    ctx = device.Context(h2)
    with pytest.raises(device.ElprepError) as ei:
        ctx.append_bam(raw, offs)
    assert ei.value.code == -18 and "RG:Z" in str(ei.value) and ctx.n == 0
    ctx.close()
    # a record whose lengths do not add up; nothing is appended
    bad = raw.copy(); bad[int(offs[5]) + 20] ^= 0x40                  # l_seq of record 5
    ctx = device.Context(w.header)
    with pytest.raises(device.ElprepError) as ei:
        ctx.append_bam(bad, offs)
    assert ei.value.code == -18 and ctx.n == 0
    ctx.append_bam(raw, offs)                                          # the context is still usable
    assert ctx.n == w.batch.n
    # block_size chain that does not end at n_bytes
    with pytest.raises(device.ElprepError):
        ctx.append_bam(raw[:-3], None)
    ctx.close()


def test_against_committed_golden_digests(tmp_path):
    """the CUDA path against tests/golden/oracle_regression.json (digests committed by tools/make_golden.py)"""
    import hashlib, json, os, sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    sys.path.insert(0, os.path.join(root, "tools"))
    import make_golden
    from elprep_b200 import device, _lib
    gold = json.load(open(os.path.join(root, "tests", "golden", "oracle_regression.json")))
    for name, case in make_golden.CASES.items():
        w = synth.make_workload(case["n_pairs"], case["contigs"], **case["kw"])
        g = gpu_pipeline(w, n_batches=2)
        exp = gold[name]
        assert make_golden.digest(g["perm"]) == exp["perm"] and make_golden.digest(g["flag"]) == exp["flag"], name
        assert make_golden.digest(g["qual"]) == exp["qual"] and hashlib.sha256(g["report"].encode()).hexdigest()[:24] == exp["report"], name
        ctx = device.Context(w.header)
        ctx.append(w.batch)
        ctx.sort_markdup(device.SO_KEEP, _lib.MARKDUP_OPTICAL)
        p = str(tmp_path / (name + ".txt"))
        ctx.print_duplicates_metrics(p, "elprep filter in out", "T")
        assert hashlib.sha256(open(p).read().encode()).hexdigest()[:24] == exp["metrics"], name
        ctx.close()


def test_whole_bam_file_in_memory():
    """BGZF file bytes -> inflate (host threads) -> header walk -> elp_append_bam -> path -> elp_fetch_bam -> deflate;
    the result, decoded with Python's gzip and the parseBamAlignment restatement, carries the oracle's FLAGs and QUALs"""
    import gzip, struct
    from elprep_b200 import device, bgzf
    from util import decode_bam, encode_bam
    w = synth.make_workload(3_000, SMALL, seed=23)
    o = oracle_pipeline(w)
    raw, offs = encode_bam(w.batch, w.header)
    text = b"@HD\tVN:1.6\tSO:unsorted\n"
    hdr = b"BAM\1" + struct.pack("<i", len(text)) + text + struct.pack("<i", len(w.header.SQ)) + b"".join(
        struct.pack("<i", len(sq["SN"]) + 1) + sq["SN"].encode() + b"\0" + struct.pack("<i", int(sq["LN"])) for sq in w.header.SQ)
    bam_file = bgzf.deflate(np.concatenate([np.frombuffer(hdr, np.uint8), raw]))
    # ---- the flow a caller with the file in memory runs
    plain = bgzf.inflate(bam_file)
    h0, nref = bgzf.bam_header_size(plain)
    assert nref == len(w.header.SQ) and h0 == len(hdr)
    ctx = device.Context(w.header)
    for ci in range(len(w.header.SQ)):
        ctx.set_reference(ci, w.contig_bases[ci]); ctx.set_known_sites(ci, w.sites[ci], already_flat=True)
    ctx.append_bam(plain[h0:], None)
    ctx.sort_markdup(); ctx.bqsr_gather(); ctx.bqsr_finalize(None); ctx.bqsr_apply()
    out, _ = ctx.fetch_bam()
    out_file = bgzf.deflate(np.concatenate([plain[:h0], out]))
    ctx.close()
    # ---- check
    dec = np.frombuffer(gzip.decompress(out_file.tobytes()), np.uint8)
    assert dec[:h0].tobytes() == hdr
    body = dec[h0:]
    offs2, x = [0], 0
    while x < body.size:
        x += 4 + int(body[x]) + (int(body[x + 1]) << 8) + (int(body[x + 2]) << 16) + (int(body[x + 3]) << 24); offs2.append(x)
    b2 = decode_bam(body, np.array(offs2, np.uint64), w.header)
    assert np.array_equal(b2.flag, o["flag"]) and np.array_equal(b2.qual, o["qual"])
    assert np.array_equal(b2.pos, w.batch.pos[o["perm"].astype(np.int64)])


def test_bam_ingest_filters():
    """per-record filters fused into elp_append_bam (filters/simple-filters.go:71-103,131-133,332-347): the reads that survive, and
    everything computed from them, equal the column path over the host-filtered batch"""
    from elprep_b200 import device, _lib
    from util import encode_bam
    w = synth.make_workload(5_000, SMALL, seed=29, unmapped_frac=0.1)
    b = w.batch
    b.flag[::17] |= 0x400                                     # duplicate flags on input, for RemoveDuplicateReads
    raw, offs = encode_bam(b, w.header)
    ncig = (b.cigar_off[1:] - b.cigar_off[:-1]).astype(np.int64)
    ops_ok = np.ones(b.n, bool)
    for i in np.nonzero(ncig > 0)[0]:
        ops = b.cigar[int(b.cigar_off[i]):int(b.cigar_off[i + 1])] & 15
        ops_ok[i] = bool(np.all((ops == 0) | (ops == 4)))
    preds = {
        _lib.FILTER_UNMAPPED: (b.flag & 4) == 0,
        _lib.FILTER_UNMAPPED_STRICT: ((b.flag & 4) == 0) & (b.pos != 0) & (b.refid >= 0),
        _lib.FILTER_NON_EXACT: ops_ok,
        _lib.FILTER_DUPLICATES: (b.flag & 0x400) == 0,
    }
    cases = [(m, 0) for m in preds] + [(0, 30), (_lib.FILTER_UNMAPPED | _lib.FILTER_NON_EXACT | _lib.FILTER_DUPLICATES, 20), (0, 300)]
    for mask, mq in cases:
        keep = b.mapq.astype(np.int64) >= mq
        for bit, p in preds.items():
            if mask & bit:
                keep &= p
        sub = b.take(np.nonzero(keep)[0])
        ctx = device.Context(w.header)
        ctx.set_ingest_filter(mask, mq)
        half = b.n // 2
        ctx.append_bam(raw[:int(offs[half])], offs[:half + 1])
        ctx.append_bam(raw[int(offs[half]):], None)
        assert ctx.n == sub.n and ctx.n_filtered() == b.n - sub.n, (mask, mq)
        ref = device.Context(w.header)
        ref.append(sub)
        for c_ in (ctx, ref):
            c_.sort_markdup()
        a1, a2 = ctx.fetch(), ref.fetch()
        assert all(np.array_equal(x, y) for x, y in zip(a1[:3], a2[:3])), (mask, mq)
        assert np.array_equal(a1[3][:int(a1[2][-1])], a2[3][:int(a2[2][-1])]), (mask, mq)
        if sub.n:
            out, ooff = ctx.fetch_bam()
            assert ooff.size == sub.n + 1 and int(ooff[-1]) == out.size
        ctx.close(); ref.close()


def test_queryname_order():
    """--sorting-order queryname: By(QNAMELess).ParallelStableSort (sam/sam-types.go:479-481) on the device; duplicate marking and
    BQSR are order independent"""
    import oracle
    from elprep_b200 import device, _lib
    w = synth.make_workload(8_000, SMALL, seed=31)
    b = w.batch.copy()
    oracle.mark_duplicates(b, w.header)
    perm = oracle.queryname_sort(b)
    srt = b.take(perm)
    ref = oracle.Reference(w.header, w.contig_bases, w.sites)
    t = oracle.bqsr_gather(srt, w.header, ref, n_threads=4)
    oracle.bqsr_finalize(t); oracle.bqsr_apply(srt, w.header, t, n_threads=4)
    ctx = device.Context(w.header)
    for ci in range(len(w.header.SQ)):
        ctx.set_reference(ci, w.contig_bases[ci]); ctx.set_known_sites(ci, w.sites[ci], already_flat=True)
    half = w.batch.n // 2
    ctx.append(w.batch.take(np.arange(0, half))); ctx.append(w.batch.take(np.arange(half, w.batch.n)))
    ctx.sort_markdup(_lib.SO_QUERYNAME, True)
    ctx.bqsr_gather(); ctx.bqsr_finalize(None); ctx.bqsr_apply()
    idx, flag, qoff, qual = ctx.fetch()
    assert np.array_equal(idx, perm.astype(np.uint64)) and np.array_equal(flag, srt.flag)
    assert np.array_equal(qual[:int(qoff[-1])], srt.qual)
    d, _ = oracle_tables_dense(t, 500)
    assert np.array_equal(ctx.tables_get(), d)
    ctx.close()
    # names of different lengths, prefixes, equal names (stability)
    h = sam.Header(sq=[{"SN": "chr1", "LN": 1000}])
    names = ["r10", "r2", "r1", "r1", "r", "R9", "r1:x", "a" * 40, "a" * 39 + "b", "a" * 40]
    bb = sam.AlignmentBatch.from_records(h, [dict(QNAME=q, FLAG=0, RNAME="chr1", POS=10 - i) for i, q in enumerate(names)])
    ctx = device.Context(h)
    ctx.append(bb); ctx.sort_markdup(_lib.SO_QUERYNAME, False)
    assert np.array_equal(ctx.fetch(want_qual=False)[0], oracle.queryname_sort(bb).astype(np.uint64))
    ctx.close()
