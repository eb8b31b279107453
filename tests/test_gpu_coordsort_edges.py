"""The coordinate and queryname sorts at their edges: tie runs of 1 to 5000 reads placed across the tie_short (128-thread) and
tie_long_flag (256-thread) block edges, QNAMEs whose common prefix ends at every chunk edge and nq from 1 to 32, every comparator
clause as the only differing field of a short and of a long run, primary keys with POS up to 2^31 - 1 and up to 4000 contigs, names
that differ only by trailing NUL bytes, names of 4 and 40 kB, and one large case.

Every run compares the device order with the restatement in coordsort_ref.py (and the oracle, which agrees with it on every input
here), and checks from kernel_stats() how many long-tie rounds ran and how many radix passes the sort took in all, so a case that
lands on another path fails even when its order happens to be right."""
import numpy as np
import pytest

import coordsort_ref as R
from coordsort_cases import CASES, NUL_NAMES, columns, header
from elprep_b200 import _lib, sam

pytestmark = pytest.mark.gpu


def _launches(stats, name):
    return stats.get(name, {}).get("launches", 0)


def _sort(b, n_contigs, order=_lib.SO_COORDINATE, mark=0, sam_text=None):
    from elprep_b200 import device
    ctx = device.Context(header(n_contigs), profile=True)
    try:
        if sam_text is None:
            ctx.append(b)
        else:
            ctx.append_sam(sam_text)
        ctx.sort_markdup(order, mark)
        idx, flag, _, _ = ctx.fetch(want_qual=False)
        stats = ctx.kernel_stats()
    finally:
        ctx.close()
    return idx.astype(np.int64), flag, stats


def check_coordinate(b, n_contigs, sam_text=None):
    import oracle
    idx, _, stats = _sort(b, n_contigs, sam_text=sam_text)
    want = R.coordinate_order(b, n_contigs)
    assert np.array_equal(idx, want), f"order differs at {np.flatnonzero(idx != want)[:8]}"
    assert np.array_equal(want, oracle.coordinate_sort(b, n_threads=4))
    rounds, passes = R.coordinate_sort_launches(b, n_contigs)
    assert _launches(stats, "tie_chunk_keys") == rounds
    assert _launches(stats, "radix_onesweep_u64") == passes
    return stats


def check_queryname(b, n_contigs, sam_text=None):
    import oracle
    idx, _, stats = _sort(b, n_contigs, _lib.SO_QUERYNAME, sam_text=sam_text)
    want = R.queryname_order(b)
    assert np.array_equal(idx, want), f"order differs at {np.flatnonzero(idx != want)[:8]}"
    assert np.array_equal(want, oracle.queryname_sort(b))
    assert _launches(stats, "qname_chunk_keys") == (R.n_qname_chunks(b) + 1 if b.n > 1 else 0)
    assert _launches(stats, "radix_onesweep_u64") == R.queryname_passes(b)


@pytest.mark.parametrize("name", list(CASES))
def test_coordinate_order(name):
    b, n_contigs = CASES[name]()
    check_coordinate(b, n_contigs)


QUERYNAME_CASES = ["n1", "n2", "runs_33", "same_coordinate", "qname_short", "qname_long", "c583c7f", "nuls_8", "nuls_200", "names_4k",
                   "nq_1", "nq_2", "nq_8", "nq_9", "nq_16", "nq_17", "nq_31", "nq_32"]


@pytest.mark.parametrize("name", QUERYNAME_CASES)
def test_queryname_order(name):
    b, n_contigs = CASES[name]()
    check_queryname(b, n_contigs)


def test_queryname_equal_names_and_extreme_lengths():
    """equal names keep arrival order; names of 1 and 254 bytes in one context"""
    rng = np.random.default_rng(3)
    pool = [b"x", b"x" * 254, b"y", b"x" * 253 + b"y", b"\xff", b"\x80" * 254]
    names = [pool[k] for k in rng.integers(0, len(pool), 400)]
    check_queryname(columns(names, 0, rng.integers(1, 50, 400)), 1)


@pytest.mark.parametrize("name", ["c583c7f", "qname_long", "nq_32", "nuls_200", "widths_4000", "clause_modflag_rev_100", "names_4k"])
def test_chunk_keys(name):
    """elp_debug_coord_chunk_keys against coordsort_ref.chunk_keys, chunk by chunk, for every read.  c583c7f: a run of 2400 reads with
    names shorter than 8 bytes (every QNAME chunk but the last is zero in whole warps) next to one 200-byte name"""
    from elprep_b200 import device
    b, n_contigs = CASES[name]()
    nq = R.n_qname_chunks(b)
    ctx = device.Context(header(n_contigs))
    try:
        ctx.append(b)
        for ch in range(R.QC0 + nq + 1):
            got = ctx.debug_coord_chunk_keys(ch)
            want = R.chunk_keys(b, ch, nq, n_contigs)
            assert np.array_equal(got, want), (ch, np.flatnonzero(got != want)[:8])
        for ch in (-1, R.QC0 + nq + 1):
            with pytest.raises(device.ElprepError) as ei:
                ctx.debug_coord_chunk_keys(ch)
            assert ei.value.code == _lib.EINVAL
    finally:
        ctx.close()


# ---------------------------------------------------------------- REFID / NextREFID outside [-1, n_contigs)
@pytest.mark.parametrize("n_contigs", [0, 3])
@pytest.mark.parametrize("field", ["refid", "nref"])
@pytest.mark.parametrize("delta", [0, 5, "-2"])
def test_refid_out_of_range_is_refused(n_contigs, field, delta):
    """a columnar batch with such a value is refused whole at append, before duplicate marking could pack it into the library bits;
    the reads appended before it are sorted and marked as if it had never come"""
    from elprep_b200 import device
    import oracle
    h = sam.Header(sq=[{"SN": f"c{i}", "LN": 10_000} for i in range(n_contigs)], rg=[{"ID": "rg0", "LB": "lib0"}])
    r = 0 if n_contigs else -1
    good = sam.AlignmentBatch.from_records(h, [dict(QNAME=f"d{k}", FLAG=0, RNAME=f"c{r}" if n_contigs else "*", POS=100, MAPQ=60, CIGAR="4M",
                                                    SEQ="ACGT", QUAL=[30 + k] * 4, RG="rg0") for k in range(3)])
    bad = good.copy()
    value = -2 if delta == "-2" else n_contigs + delta
    getattr(bad, field)[1] = value
    bad.flag[:] = 0
    ctx = device.Context(h)
    try:
        ctx.append(good)
        with pytest.raises(device.ElprepError) as ei:
            ctx.append(bad)
        assert ei.value.code == _lib.EINVAL and "REFID" in str(ei.value)
        assert ctx.n == good.n
        ctx.sort_markdup(device.SO_COORDINATE, _lib.MARKDUP)
        idx, flag, _, _ = ctx.fetch(want_qual=False)
    finally:
        ctx.close()
    b1 = good.copy()
    oracle.mark_duplicates(b1, h, n_threads=1)
    perm = oracle.coordinate_sort(b1, n_threads=1)
    assert np.array_equal(idx, perm.astype(np.uint64)) and np.array_equal(flag, b1.flag[perm])
    if n_contigs:
        assert int(((flag & 0x400) != 0).sum()) == 2                   # three fragments at one place: the two lower scores


# ---------------------------------------------------------------- names that differ only by trailing NUL bytes, through SAM text
def _sam_lines(b):
    out = bytearray()
    for i, nm in enumerate(R.qnames(b)):
        out += nm + b"\t%d\tc0\t%d\t%d\t4M\t*\t0\t0\tACGT\tIIII\n" % (b.flag[i], b.pos[i], b.mapq[i])
    return bytes(out)


@pytest.mark.parametrize("run_len", [8, 200])
def test_trailing_nuls_through_sam(run_len):
    rng = np.random.default_rng(run_len)
    names = [NUL_NAMES[k] for k in rng.integers(0, len(NUL_NAMES), run_len)] + [b"z"] * 3
    b = columns(names, 0, [300] * run_len + [1, 2, 3], flag=0, mapq=60, nref=-1, pnext=0, tlen=0)
    text = _sam_lines(b)
    check_coordinate(b, 1, sam_text=text)
    check_queryname(b, 1, sam_text=text)


# ---------------------------------------------------------------- with duplicate marking
def _dup_runs(n_pairs, n_frags, seed):
    rng = np.random.default_rng(seed)
    recs = []
    for k in range(n_pairs):                                             # one signature: long runs at both mate positions
        nm = f"M:1:FC:1:1101:{1000 + int(rng.integers(0, 300))}:{2000 + k}"
        s = 30 + k % 7
        recs += [dict(QNAME=nm, FLAG=99, RNAME="c0", POS=10_000, MAPQ=60, CIGAR="4M", SEQ="ACGT", QUAL=[s] * 4, RG="rg0", RNEXT="=", PNEXT=10_400, TLEN=404),
                 dict(QNAME=nm, FLAG=147, RNAME="c0", POS=10_400, MAPQ=60, CIGAR="4M", SEQ="ACGT", QUAL=[s] * 4, RG="rg0", RNEXT="=", PNEXT=10_000, TLEN=-404)]
    for k in range(n_frags):                                             # fragments at one place, some with the input duplicate bit
        recs.append(dict(QNAME=f"f{k % 9}", FLAG=16 | (0x400 if k % 5 == 0 else 0), RNAME="c1", POS=20_000, MAPQ=int(rng.integers(0, 3)) * 127,
                         CIGAR="4M", SEQ="ACGT", QUAL=[20 + k % 11] * 4, RG="rg0"))
    recs += [dict(QNAME=f"u{k % 4}", FLAG=4, RNAME="*", POS=0, MAPQ=0, CIGAR="*", SEQ="ACGT", QUAL=[30] * 4, RG="rg0") for k in range(40)]
    order = rng.permutation(len(recs))
    return [recs[i] for i in order]


@pytest.mark.parametrize("n_pairs,n_frags", [(40, 60), (300, 35)])
def test_long_runs_with_marking(n_pairs, n_frags):
    """the modFlag chunk must see the 0x400 that marking set: order, FLAG and metrics against the oracle, pass counts restated"""
    from markdup_check import check
    h = sam.Header(sq=[{"SN": "c0", "LN": 1_000_000}, {"SN": "c1", "LN": 1_000_000}], rg=[{"ID": "rg0", "LB": "lib0"}])
    b = sam.AlignmentBatch.from_records(h, _dup_runs(n_pairs, n_frags, n_pairs))
    flag, stats = check(b, h)
    assert (flag & 0x400).sum() >= n_pairs and _launches(stats, "tie_chunk_keys") > 0


# ---------------------------------------------------------------- one large case
def test_large():
    """a million reads, about 30 % of them in runs of 33..400: tie_long_flag spans thousands of blocks and the tie rounds many tiles"""
    from coordsort_cases import large
    b, n_contigs = large()
    long = R.long_run_elements(b, n_contigs).size
    assert 0.25 * b.n < long < 0.4 * b.n
    stats = check_coordinate(b, n_contigs)
    assert _launches(stats, "tie_chunk_keys") >= 5
