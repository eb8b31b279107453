"""The smaller sorts of duplicate marking against the exact ones.

When true fragments are few, only they are sorted: their group bits go into a set that the entering true-pair reads probe for the
has-pair bit.  Pair groups are sorted by a 32-bit hash of the signature and told apart on the signatures inside equal-hash runs.
ELPREP_B200_MARKDUP=exact forces the full fragment sort and the exact signature sort; =hashed takes the smaller sorts at every size;
ELPREP_B200_MARKDUP_HASH_BITS=k keeps k hash bits, so that many signatures share a run.  Every case runs both settings in one
process and compares FLAG bit for bit between them and with the oracle, and checks from kernel_stats() which path ran."""
import numpy as np
import pytest

from elprep_b200 import _lib, device, sam, synth

pytestmark = pytest.mark.gpu

SPARSE = ("frag_set_insert", "frag_set_probe", "frag_sparse_mark")


def _header(n_libs=1, n_contigs=2):
    return sam.Header(sq=[{"SN": f"c{i}", "LN": 1_000_000} for i in range(n_contigs)],
                      rg=[{"ID": f"rg{i}", "LB": f"lib{i}"} for i in range(n_libs)])


def R(q, flag, pos, score=30, rg="rg0", rname="c0", **kw):
    return dict(QNAME=q, FLAG=flag, RNAME=rname, POS=pos, MAPQ=60, CIGAR="4M", SEQ="ACGT", QUAL=[score] * 4, RG=rg, **kw)


def pair(q, p1, p2, s1=30, s2=None, rg="rg0", rname="c0", flags=(99, 147)):
    return [R(q, flags[0], p1, s1, rg=rg, rname=rname, RNEXT="=", PNEXT=p2),
            R(q, flags[1], p2, s1 if s2 is None else s2, rg=rg, rname=rname, RNEXT="=", PNEXT=p1)]


def frag(q, pos, score=30, rev=False, rg="rg0", rname="c0", mate_unmapped=True):
    """a true fragment: the mapped read of a mate-unmapped pair, or an unpaired read"""
    f = (0x1 | 0x8 | 0x40) if mate_unmapped else 0
    return R(q, f | (0x10 if rev else 0), pos, score, rg=rg, rname=rname)


def filler(k, base=500_000):
    """k distinct pairs far from every case, so that fragments stay a small share of the entering reads"""
    return [r for j in range(k) for r in pair(f"fill{j:05d}", base + 20 * j, base + 20 * j + 300)]


def _run(b, h, monkeypatch, mode, hash_bits=None, optical=False):
    monkeypatch.setenv("ELPREP_B200_MARKDUP", mode)
    if hash_bits is None:
        monkeypatch.delenv("ELPREP_B200_MARKDUP_HASH_BITS", raising=False)
    else:
        monkeypatch.setenv("ELPREP_B200_MARKDUP_HASH_BITS", str(hash_bits))
    ctx = device.Context(h, profile=True)
    try:
        ctx.append(b)
        ctx.sort_markdup(device.SO_COORDINATE, _lib.MARKDUP_OPTICAL if optical else _lib.MARKDUP)
        idx, flag, _, _ = ctx.fetch(want_qual=False)
        stats = ctx.kernel_stats()
    finally:
        ctx.close()
    out = np.empty(b.n, np.uint16)
    out[idx.astype(np.int64)] = flag
    return out, stats


def compare(b, h, monkeypatch, sparse=True, hashed=True, hash_bits=None, mode="hashed"):
    """FLAG in arrival order of the `mode` run, which must equal the exact run and the oracle; checks which paths each run took"""
    import oracle
    want = b.copy()
    oracle.mark_duplicates(want, h, n_threads=1)
    exact, se = _run(b, h, monkeypatch, "exact")
    got, sn = _run(b, h, monkeypatch, mode, hash_bits)
    monkeypatch.delenv("ELPREP_B200_MARKDUP")
    assert np.array_equal(exact, want.flag), "exact sorts: FLAG differs from the oracle"
    assert np.array_equal(got, exact), "smaller sorts: FLAG differs from the exact sorts"
    assert not any(k in se for k in SPARSE + ("pair_hash_mark",))
    assert all(k in sn for k in SPARSE) == sparse and ("frag_keys" in sn) == (not sparse)
    assert ("pair_hash_mark" in sn) == hashed and not (hashed and "pair_mark" in sn)
    return got, sn, se


def _dup(flag, recs, name):
    return [bool(flag[i] & 0x400) for i, r in enumerate(recs) if r["QNAME"] == name]


def _batch(h, recs):
    return sam.AlignmentBatch.from_records(h, recs)


# ---------------------------------------------------------------- fragment groups
def test_fragment_groups_with_and_without_pair_reads(monkeypatch):
    h = _header()
    recs = [frag("a1", 1000, 20), frag("a2", 1000, 35), frag("a3", 1000, 25)]             # no pair read: 35 survives
    recs += [frag("b1", 2000, 40), frag("b2", 2000, 41)] + pair("bp", 2000, 2400, 10)      # a pair read: every fragment is a duplicate
    recs += pair("cp", 3000, 3300, 10) + [frag("c1", 3000, 50)]                             # a lone fragment after the pair read
    recs += [frag("d1", 4000, 30)]                                                          # alone: never a duplicate
    recs += [frag("e1", 5000, 30, mate_unmapped=False), frag("e2", 5000, 31)]               # an unpaired read and a mate-unmapped one
    recs += pair("fp", 6000, 6300, 20) + pair("fq", 6000, 6300, 22)                         # pair reads alone: not touched by fragments
    recs += filler(40)
    flag, _, _ = compare(_batch(h, recs), h, monkeypatch)
    assert _dup(flag, recs, "a1") == [True] and _dup(flag, recs, "a2") == [False] and _dup(flag, recs, "a3") == [True]
    assert _dup(flag, recs, "b1") == [True] and _dup(flag, recs, "b2") == [True] and _dup(flag, recs, "bp") == [False, False]
    assert _dup(flag, recs, "c1") == [True] and _dup(flag, recs, "d1") == [False]
    assert _dup(flag, recs, "e1") == [True] and _dup(flag, recs, "e2") == [False]
    assert _dup(flag, recs, "fp") == [True, True] and _dup(flag, recs, "fq") == [False, False]


@pytest.mark.parametrize("field", ["strand", "library", "contig", "none"])
def test_fragment_and_pair_read_differ_in_one_field(field, monkeypatch):
    """the pair read has the fragment's unclipped 5' position; only `field` differs (none: same group)"""
    h = _header(n_libs=2)
    fr = frag("f", 1003, 30, rev=False)
    if field == "strand":      # reverse 4M at 1000: unclipped 5' end 1003, reverse strand
        p = pair("p", 900, 1000, 30)
    else:
        p = pair("p", 1003, 1400, 30, rg="rg1" if field == "library" else "rg0", rname="c1" if field == "contig" else "c0")
        if field == "contig":
            for r in p:
                r["RNEXT"] = "="
    recs = [fr] + p + filler(10)
    flag, _, _ = compare(_batch(h, recs), h, monkeypatch)
    assert _dup(flag, recs, "f") == [field == "none"]


@pytest.mark.parametrize("order", ["forward", "reverse"])
def test_fragment_tie_rules(order, monkeypatch):
    """score first, then the smallest QNAME, then the later arrival; 40 groups so that a group's fragments leave the set pass in
    several warps"""
    h = _header()
    recs = []
    for g in range(40):
        p = 10_000 + 100 * g
        grp = [frag(f"g{g}s", p, 20 + g % 3), frag(f"g{g}z", p, 40), frag(f"g{g}y", p, 40),         # score ties: QNAME y < z
               frag(f"g{g}t", p, 39), frag(f"g{g}w", p, 37)]
        tie = [frag(f"t{g}", p + 50, 33) for _ in range(3 + g % 4)]                                  # full ties: the last one survives
        grp = grp if order == "forward" else grp[::-1]
        recs += grp + tie
    recs += filler(1200)
    flag, _, _ = compare(_batch(h, recs), h, monkeypatch)
    for g in range(40):
        assert _dup(flag, recs, f"g{g}y") == [False] and _dup(flag, recs, f"g{g}z") == [True] and _dup(flag, recs, f"g{g}s") == [True]
        k = 3 + g % 4
        assert _dup(flag, recs, f"t{g}") == [True] * (k - 1) + [False]


def test_single_end_input_takes_the_full_sort(monkeypatch):
    h = _header()
    recs = [R(f"s{k}", 16 if k % 3 == 0 else 0, 1000 + 7 * (k % 50), 20 + k % 13) for k in range(600)]
    compare(_batch(h, recs), h, monkeypatch, sparse=False, hashed=False)


@pytest.mark.parametrize("n_frag,sparse", [(20, True), (21, False)])
def test_fragment_share_cut_off(n_frag, sparse, monkeypatch):
    """30 pairs and n_frag fragments: the set path while 4 x fragments <= entering reads (80 <= 80; 84 > 81)"""
    h = _header()
    recs = []
    for k in range(30):
        recs += pair(f"p{k}", 1000 + 40 * (k % 10), 1300 + 40 * (k % 10), 20 + k % 7)
    recs += [frag(f"f{k}", 1000 + 40 * (k % 12), 25 + k % 5, rev=k % 2 == 1) for k in range(n_frag)]
    recs.append(dict(QNAME="u", FLAG=4, RNAME="*", POS=0, MAPQ=0, CIGAR="*", SEQ="ACGT", QUAL=[30] * 4, RG="rg0"))   # enters neither count
    compare(_batch(h, recs), h, monkeypatch, sparse=sparse)


# ---------------------------------------------------------------- pair groups
def _pair_groups(n_sig, rng, h_libs=1, illumina=False):
    """pairs in n_sig signatures, 1..6 pairs each, shuffled in arrival order; ties in score and in QNAME inside groups (illumina:
    distinct names with tile and coordinates, as optical marking parses them)"""
    pairs = []
    for s in range(n_sig):
        k = 1 + s % 6
        for j in range(k):
            sc = 30 + (j * 7 + s) % 4
            name = f"s{s:03d}{'ab'[(j + s) % 2]}"                                                  # repeated names: full ties
            if illumina:
                name = f"M1:7:FC:1:{1101 + s % 3}:{1000 + 500 * j}:{2000 + 97 * s}"
            pairs.append((name, 1000 + 37 * s, 1300 + 37 * s + (s % 3), sc, f"rg{s % h_libs}"))
    order = rng.permutation(len(pairs))
    recs = []
    for i in order:
        name, p1, p2, sc, rg = pairs[i]
        recs += pair(name, p1, p2, sc, rg=rg)
    return recs


@pytest.mark.parametrize("hash_bits", [1, 2, 3, 32])
def test_pair_signatures_in_colliding_runs(hash_bits, monkeypatch):
    """with k hash bits every run holds many signatures, interleaved in arrival order; one bit puts more than eight distinct
    signatures in a run, past the leaders the walk remembers"""
    h = _header(n_libs=2)
    recs = _pair_groups(60, np.random.default_rng(hash_bits), h_libs=2) + [frag("f", 99_000)]
    compare(_batch(h, recs), h, monkeypatch, hash_bits=hash_bits)


@pytest.mark.parametrize("hash_bits", [1, 4])
def test_colliding_signatures_in_separate_stretches(hash_bits, monkeypatch):
    """each signature's pairs arrive together, one signature after another"""
    h = _header()
    recs = []
    for s in range(30):
        for j in range(1 + s % 5):
            recs += pair(f"q{s}_{j}", 2000 + 11 * s, 2500 + 11 * s, 30 + (j * 5) % 3)
    recs.append(frag("f", 99_000))
    compare(_batch(h, recs), h, monkeypatch, hash_bits=hash_bits)


def test_optical_marking_keeps_the_exact_pair_sort(monkeypatch):
    import oracle
    h = _header()
    recs = _pair_groups(20, np.random.default_rng(3), illumina=True) + [frag("M1:7:FC:1:1101:5:5", 99_000)]
    b = _batch(h, recs)
    exact, _ = _run(b, h, monkeypatch, "exact", optical=True)
    got, stats = _run(b, h, monkeypatch, "hashed", optical=True)
    want = b.copy()
    oracle.mark_duplicates(want, h, n_threads=1)
    assert np.array_equal(got, exact) and np.array_equal(exact & 0x400, want.flag & 0x400)
    assert "pair_mark" in stats and "pair_hash_mark" not in stats


@pytest.mark.parametrize("hash_bits", [2, 32])
def test_u64_and_u128_pair_layouts(hash_bits, monkeypatch):
    """62-bit signatures (u64) and, with 4000 contigs, signatures over 64 bits (u128)"""
    w = synth.make_workload(20_000, [("chr20", 600_000), ("chr21", 300_000)], seed=5, want_reference=False, dup_frac=0.3, mate_unmapped_frac=0.05)
    compare(w.batch, w.header, monkeypatch, hash_bits=hash_bits)
    contigs = [("chr1", 3_000_000)] + [(f"c{i}", 1_500) for i in range(4000)]
    w = synth.make_workload(20_000, contigs, seed=7, want_reference=False, dup_frac=0.3, cross_contig_frac=0.2, mate_unmapped_frac=0.05)
    _, _, exact_stats = compare(w.batch, w.header, monkeypatch, hash_bits=hash_bits)
    assert exact_stats["radix_onesweep_u128"]["launches"] > 0


# ---------------------------------------------------------------- a generated workload
@pytest.mark.parametrize("permuted", [False, True])
def test_generated_workload(permuted, monkeypatch):
    """2 M reads: the default setting takes the set path at this size; the hashed setting also takes the pair hash"""
    w = synth.make_workload(1_000_000, synth.scaled_hg38(400.0), seed=11, want_reference=False)
    b = w.batch
    if permuted:
        b = synth.take(b, np.random.default_rng(5).permutation(b.n))
    assert b.n >= 2_000_000
    compare(b, w.header, monkeypatch)
    flag, _, _ = compare(b, w.header, monkeypatch, hashed=False, mode="auto")
    assert 0 < int(((flag & 0x400) != 0).sum())
