"""Duplicate marking at the edges of its data-dependent layouts: packed keys of exactly 63 to 69 bits with a field across bit 64,
the fragment key at 64 bits and one bit past it, the radix sort over a bit range, the mate join on colliding (library, QNAME)
hashes, and optical clustering at its run-length, histogram, list-length and tile-value limits.

Every run compares output order, FLAG, counters, histograms and the metrics file text with the oracle (markdup_check.check), which
pairs mates by a different hash, and checks from kernel_stats() which sort widths ran and how many digit passes each took.  Where
the answer can be derived by hand, it is asserted as well."""
import numpy as np
import pytest

from elprep_b200 import _lib, sam
from markdup_check import check
from markdup_edges import COLLIDING_LENGTHS, COLLIDING_PAIRS, COLLIDING_TRIPLE, join_hash, join_key

pytestmark = pytest.mark.gpu

I32_MAX = 2 ** 31 - 1
ETILE = -17                                                         # ELP_ETILE: a tile/x/y field strconv.ParseInt rejects


def _header(n_contigs=1, n_libs=1, ln=I32_MAX):
    return sam.Header(sq=[{"SN": f"c{i}", "LN": ln} for i in range(n_contigs)],
                      rg=[{"ID": f"rg{i}", "LB": f"lib{i}"} for i in range(n_libs)])


def R(q, flag, pos, score=30, rg="rg0", rname="c0", cigar="4M", n=4, **kw):
    return dict(QNAME=q, FLAG=flag, RNAME=rname, POS=pos, MAPQ=60, CIGAR=cigar, SEQ="A" * n, QUAL=[score] * n, RG=rg, **kw)


def pair(q, p1, p2, s1=30, s2=None, flags=(99, 147), rg="rg0", r1="c0", r2="c0"):
    return [R(q, flags[0], p1, s1, rg=rg, rname=r1, RNEXT=r2, PNEXT=p2), R(q, flags[1], p2, s1 if s2 is None else s2, rg=rg, rname=r2, RNEXT=r1, PNEXT=p1)]


def _dup(flag, recs, name):
    return [bool(flag[i] & 0x400) for i, r in enumerate(recs) if r["QNAME"] == name]


def _ctx(h, **kw):
    from elprep_b200 import device
    return device.Context(h, **kw)


# ---------------------------------------------------------------- A. key widths
def _bits(x):
    return int(x).bit_length()


def _layout_reads(bU, neg=False):
    """fragment reads that set the unclipped-position range to exactly bU bits; neg: the low end is a soft clip at POS 1"""
    if neg:
        lo = R("ext_lo", 0, 1, cigar="100S4M", n=104)                 # upos -99
        return [lo, R("ext_hi", 0, -99 + (1 << (bU - 1)))], -99
    if bU == 31:
        return [R("ext_lo", 0, 1, cigar="1S4M", n=5), R("ext_hi", 0, I32_MAX)], 0   # upos 0 .. 2^31 - 1
    return [R("ext_lo", 0, 1), R("ext_hi", 0, 1 << bU)], 1


def _filler():
    """reads that never enter duplicate marking: with a 64-bit fragment key they take the all-ones key"""
    return [dict(QNAME=f"un{k}", FLAG=4, RNAME="*", POS=0, MAPQ=0, CIGAR="*", SEQ="ACGT", QUAL=[30] * 4, RG="rg0") for k in range(3)] + \
           [R("sec", 0x100, 500), R("sup", 0x800, 500)]


# (bU, n_contigs, n_libs, field, two values of it whose key fields differ in the top bits only, pair key bits); key layout from
# bit 0: upos2 (bU), upos1 (bU), rev2, rev1, refid2 + 1 (bR), refid1 + 1 (bR), library + 1 (bL); no LB (n_libs 0) gives bL = 1
LAYOUTS = {
    "u64_63": (28, 1, 3, "lib", (0, 2), 63),             # lib at bits 60..62
    "u64_64": (28, 1, 7, "lib", (0, 4), 64),             # lib ends on bit 63
    "u128_65_lib": (28, 2, 5, "lib", (0, 4), 65),        # lib at bits 62..64: 1 vs 5 differ in bit 64 only
    "u128_66_lib": (28, 2, 9, "lib", (0, 8), 66),        # lib at bits 62..65: 1 vs 9 differ in bit 65 only
    "u128_refid1": (29, 4, 0, "r1", (0, 2), 67),         # refid1 at bits 63..65: 1 vs 3 differ in bit 64 only (4 contigs)
    "u128_refid2": (30, 5, 0, "r2", (0, 4), 69),         # refid2 at bits 62..64: 1 vs 5 differ in bit 64 only
    "u128_refid2_at_64": (31, 2, 0, "r2", (0, 1), 69),   # refid2 starts at bit 64
    "u128_after_upos1": (32, 1, 0, "v2", (0, 1), 69),    # rev2 is bit 64 (upos range just over 2^31, from a negative upos_min)
}


@pytest.mark.parametrize("name", list(LAYOUTS))
def test_pair_key_layouts(name):
    bU, n_contigs, n_libs, field, (va, vb), key_bits = LAYOUTS[name]
    h = _header(n_contigs, max(n_libs, 1) if n_libs else 1)
    if n_libs == 0:
        h = sam.Header(sq=[{"SN": f"c{i}", "LN": I32_MAX} for i in range(n_contigs)], rg=[{"ID": "rg0"}])   # no LB: one bit of library
    ext, lo = _layout_reads(bU, neg=bU == 32)
    recs = ext + _filler()
    base = lo + 1000
    groups = []
    for gi, v in enumerate((va, vb)):
        kw = dict(rg=f"rg{v if field == 'lib' else 0}", r1="c0", r2=f"c{n_contigs - 1}")
        flags, p2 = (99, 147), base + 400
        if field == "r1":
            kw["r1"], kw["r2"] = f"c{v}", "c3"
        elif field == "r2":
            kw["r2"] = f"c{v}"
        elif field == "v2":
            flags = (97, 145) if v else (65, 129)          # mate 2 reverse (v2 = 1) or forward (v2 = 0); mate 1 forward
            p2 = base + 397 if v else base + 400           # the same unclipped 5' position either way
        for k, s in enumerate((20, 35, 25)):               # three pairs with the same signature: the 35 survives
            nm = f"g{gi}p{k}"
            groups.append(nm)
            recs += pair(nm, base, p2, s, flags=flags, **kw)
    b = sam.AlignmentBatch.from_records(h, recs)
    flag, stats = check(b, h)
    import oracle
    upos, _ = oracle.mark_duplicates(b.copy(), h, want_adapt=True)
    entering = (b.flag & 0x904) == 0
    assert _bits(int(upos[entering].max()) - int(upos[entering].min())) == bU
    assert 2 * bU + 2 + 2 * _bits(n_contigs) + _bits(n_libs + 1) == key_bits
    assert ("radix_onesweep_u128" in stats) == (key_bits > 64)
    for gi in range(2):
        assert _dup(flag, recs, f"g{gi}p0") == [True, True] and _dup(flag, recs, f"g{gi}p1") == [False, False] and _dup(flag, recs, f"g{gi}p2") == [True, True]


@pytest.mark.parametrize("n_libs,bits", [(30, 63), (62, 64)])
def test_fragment_key_63_and_64_bits(n_libs, bits):
    """bS = 17 (1 kb reads at Q93), bU = 32, bR = 7 (100 contigs), bL = 5 or 6: the group sort covers bits [18, 63) or [18, 64); the
    reads that do not enter take the all-ones key and must sort after every group"""
    h = _header(100, n_libs)
    ext, lo = _layout_reads(32, neg=True)
    recs = ext + _filler()
    recs += [R("big1", 0, 5000, 93, n=1000, cigar="1000M"), R("big2", 0, 5000, 92, n=1000, cigar="1000M")]   # a 1 kb fragment group
    recs += [R("f1", 16, 7000, 30, rg=f"rg{n_libs - 1}", rname="c99"), R("f2", 16, 7000, 31, rg=f"rg{n_libs - 1}", rname="c99")]
    recs += [R("f3", 16, 7000, 40, rg="rg0", rname="c99")]       # same place, other library: its own group
    b = sam.AlignmentBatch.from_records(h, recs)
    flag, _ = check(b, h)
    assert _bits(93 * 1000) + 2 + 32 + 7 + _bits(n_libs + 1) == bits
    assert _dup(flag, recs, "big1") == [False] and _dup(flag, recs, "big2") == [True]
    assert _dup(flag, recs, "f1") == [True] and _dup(flag, recs, "f2") == [False] and _dup(flag, recs, "f3") == [False]


def test_fragment_key_65_bits_is_refused_and_flag_untouched():
    from elprep_b200 import device
    h = _header(100, 63)                                              # bL = 7: 17 + 2 + 32 + 7 + 7 = 65
    ext, _ = _layout_reads(32, neg=True)
    recs = ext + _filler() + [R("big1", 0, 5000, 93, n=1000, cigar="1000M"), R("big2", 0, 5000, 92, n=1000, cigar="1000M")]
    recs += [R("d", 1024, 6000), R("d", 0, 6000)]                     # one read already flagged: it must stay so, the other must not gain it
    b = sam.AlignmentBatch.from_records(h, recs)
    ctx = _ctx(h)
    try:
        ctx.append(b)
        with pytest.raises(device.ElprepError) as ei:
            ctx.sort_markdup(device.SO_COORDINATE, _lib.MARKDUP)
        assert ei.value.code == _lib.ELIMIT and "65 bits" in str(ei.value)
        ctx.sort_markdup(device.SO_KEEP, 0)                           # the refused call left the context unsorted: read FLAG back
        idx, flag, _, _ = ctx.fetch()
    finally:
        ctx.close()
    assert np.array_equal(idx, np.arange(b.n, dtype=np.uint64)) and np.array_equal(flag, b.flag)


# ---------------------------------------------------------------- B. radix sort over a bit range
@pytest.mark.parametrize("n", [1, 6143, 6144, 6145, 50_001])
@pytest.mark.parametrize("lo,bits", [(1, 20), (7, 9), (8, 16), (33, 31), (56, 8), (63, 1), (1, 63)])
def test_sort_u64_bit_range(n, lo, bits):
    rng = np.random.default_rng(n * 131 + lo)
    keys = rng.integers(0, 2 ** 63, size=n, dtype=np.uint64) * np.uint64(2) + rng.integers(0, 2, size=n, dtype=np.uint64)
    field = (keys >> np.uint64(lo)) & np.uint64((1 << bits) - 1)
    if lo + bits < 64:
        keys &= np.uint64((1 << (lo + bits)) - 1)                     # nothing above the range (the caller's contract)
    if n > 100:
        few = rng.integers(0, min(5, 1 << bits), size=n, dtype=np.uint64)             # many equal ranges with different low bits: order must hold
        keys = (keys & np.uint64((1 << lo) - 1)) | (few << np.uint64(lo))
        field = few
    vals = np.arange(n, dtype=np.uint32)
    ctx = _ctx(_header(), profile=True)
    try:
        k2, v2 = ctx.debug_sort_u64(keys, vals, bits, lo_bit=lo)
        stats = ctx.kernel_stats()
    finally:
        ctx.close()
    order = np.argsort(field, kind="stable")
    assert np.array_equal(v2, vals[order]) and np.array_equal(k2, keys[order])
    assert stats["radix_onesweep_u64"]["launches"] == (bits + 7) // 8


@pytest.mark.parametrize("n", [3, 4095, 4096, 4097, 30_001])
@pytest.mark.parametrize("lo,bits", [(60, 9), (64, 20), (64, 64), (100, 28), (1, 127), (57, 30)])
def test_sort_u128_bit_range(n, lo, bits):
    rng = np.random.default_rng(n * 17 + lo)
    klo = rng.integers(0, 2 ** 63, size=n, dtype=np.uint64) * np.uint64(2) + rng.integers(0, 2, size=n, dtype=np.uint64)
    khi = rng.integers(0, 2 ** 63, size=n, dtype=np.uint64) * np.uint64(2) + rng.integers(0, 2, size=n, dtype=np.uint64)
    if n > 100:                                                       # few distinct values in the range, random bits below it
        few = rng.integers(0, 4, size=n)
        tmpl = [(int(a) << 64 | int(c)) for a, c in zip(khi[:4], klo[:4])]
        for t in range(4):
            sel = few == t
            v = tmpl[t] >> lo << lo
            below_mask = (1 << lo) - 1
            full = [(v | ((int(a) << 64 | int(c)) & below_mask)) for a, c in zip(khi[sel], klo[sel])]
            khi[sel] = np.array([x >> 64 for x in full], dtype=np.uint64)
            klo[sel] = np.array([x & (2 ** 64 - 1) for x in full], dtype=np.uint64)
    top = lo + bits
    full = [(int(a) << 64 | int(c)) & ((1 << top) - 1) for a, c in zip(khi, klo)]
    khi = np.array([x >> 64 for x in full], dtype=np.uint64)
    klo = np.array([x & (2 ** 64 - 1) for x in full], dtype=np.uint64)
    field = [x >> lo for x in full]
    vals = np.arange(n, dtype=np.uint32)
    ctx = _ctx(_header(), profile=True)
    try:
        h2, l2, v2 = ctx.debug_sort_u128(khi, klo, vals, bits, lo_bit=lo)
        stats = ctx.kernel_stats()
    finally:
        ctx.close()
    order = sorted(range(n), key=lambda i: field[i])                  # Python's sort is stable
    assert np.array_equal(v2, vals[order]) and np.array_equal(h2, khi[order]) and np.array_equal(l2, klo[order])
    assert stats["radix_onesweep_u128"]["launches"] == (bits + 7) // 8


def test_sort_bit_range_outside_the_key_is_refused():
    from elprep_b200 import device
    ctx = _ctx(_header())
    try:
        with pytest.raises(device.ElprepError) as ei:
            ctx.debug_sort_u64(np.zeros(4, np.uint64), np.arange(4, dtype=np.uint32), 8, lo_bit=57)
        assert ei.value.code == _lib.EINVAL
        with pytest.raises(device.ElprepError):
            ctx.debug_sort_u128(np.zeros(4, np.uint64), np.zeros(4, np.uint64), np.arange(4, dtype=np.uint32), 2, lo_bit=127)
    finally:
        ctx.close()


# ---------------------------------------------------------------- C. mate join
def _hash_batch(names_flags, h, long_cluster=0):
    """one read per (name, flag); the arena offset of every name is whatever the names before it add up to"""
    recs = []
    for nm, f in names_flags:
        recs.append(R(nm, f, 100, rname="c0"))
    if long_cluster:
        mid = len(recs) // 2
        recs[mid:mid] = [R(f"long{k:012d}", 99, 200, n=3000, cigar="3000M") for k in range(long_cluster)]   # 16-byte names
    return recs


@pytest.mark.parametrize("long_cluster", [0, 600])
def test_join_hash_matches_restatement(long_cluster):
    """names of 1 .. 254 bytes at every arena offset mod 16 (a filler name in front of each sets the offset); with a cluster of
    3 kb reads in the middle the adapt tiles there do not fit a ring slot and read the arenas with global loads"""
    h = _header()
    chars = b"ABCDEFGHIJKLMNOPQRSTUVWXYZabcdefghijklmnopqrstuvwxyz0123456789_."
    items, off = [], 0
    for L in range(1, 255):
        for r in range(16):
            pad = (r - off) % 16 or 16                                 # filler so that the test name starts at offset = r (mod 16)
            items.append(("z" * pad, 4))                               # unmapped: not a true pair, hash 0
            nm = bytes(chars[(L * 7 + r * 3 + j) % len(chars)] for j in range(L)).decode()
            items.append((nm, 65 if (L + r) % 3 else 129))             # true-pair reads (their mates absent)
            off += pad + L
            assert (off - L) % 16 == r
    recs = _hash_batch(items, h, long_cluster)
    b = sam.AlignmentBatch.from_records(h, recs)
    ctx = _ctx(h)
    try:
        ctx.append(b)
        got = ctx.debug_join_hash()
    finally:
        ctx.close()
    names = [r["QNAME"].encode() for r in recs]
    tp = np.array([(r["FLAG"] & 0x90d) == 0x1 for r in recs])
    want = join_hash(names, 0)
    assert np.array_equal(got[tp], want[tp])
    assert not got[~tp].any()
    staged = _adapt_tiles_staged(b)
    assert staged.any() and (not long_cluster or not staged.all())


def _adapt_tiles_staged(b):
    """phase_adapt's tile plan restated: reads per tile from the average strip lengths, and whether each tile's 16-byte aligned
    QUAL / QNAME / CIGAR windows fit a ring slot (39, 9 and 3 kB) or the tile reads the arenas with global loads"""
    n = b.n
    qo = b.qual_off.astype(np.int64) + 64                              # the QUAL arena starts at a 64-byte pad
    no, co = b.qname_off.astype(np.int64), b.cigar_off.astype(np.int64) * 4
    rpt = min(256, 0.94 * 39 * 1024 / ((qo[-1] - 64) / n + 1), 0.94 * 9 * 1024 / (no[-1] / n + 1), 0.94 * 3 * 1024 / (co[-1] / n + 1))
    rpt = max(32, int(rpt) & ~31)
    out = []
    for i0 in range(0, n, rpt):
        i1 = min(n, i0 + rpt)
        span = [((o[i1] + 15) & ~15) - (o[i0] & ~15) for o in (qo, no, co)]
        out.append(span[0] <= 39 * 1024 and span[1] <= 9 * 1024 and span[2] <= 3 * 1024)
    return np.array(out)


def _join_case(recs, h, optical=True):
    b = sam.AlignmentBatch.from_records(h, recs)
    flag, _ = check(b, h, optical=optical)
    return flag


def test_colliding_non_mates_without_their_mates():
    """a run of exactly two equal join keys that are not mates: the fast path must not pair them (their mates are absent, so
    nothing pairs and nothing is a pair duplicate)"""
    h = _header()
    recs = []
    for a, b_ in COLLIDING_PAIRS[:2]:
        recs += [R(a.decode(), 99, 1000, RNEXT="=", PNEXT=1300), R(b_.decode(), 147, 1300, RNEXT="=", PNEXT=1000)]
    flag = _join_case(recs, h)
    assert not (flag & 0x400).any()        # joined by key alone, the two runs would be two pairs of one signature and one would lose


def test_colliding_non_mates_with_mates_elsewhere():
    h = _header()
    out = []
    for (a, b_) in COLLIDING_PAIRS:
        a, b_ = a.decode(), b_.decode()
        out += [R(a, 99, 1000, RNEXT="=", PNEXT=1300), R(b_, 99, 1000, RNEXT="=", PNEXT=1300)]
        out += [R(a, 147, 1300, 20, RNEXT="=", PNEXT=1000), R(b_, 147, 1300, 40, RNEXT="=", PNEXT=1000)]
    flag = _join_case(out, h)
    # six pairs of one signature: the three second names score 30 + 40 per base, the first names 30 + 20; the smallest of the
    # three second names wins the tie
    best = min(b_.decode() for _, b_ in COLLIDING_PAIRS)
    assert [nm for nm in dict.fromkeys(r["QNAME"] for r in out) if not any(_dup(flag, out, nm))] == [best]


@pytest.mark.parametrize("order", ["A1 C1 A2", "A1 B1 A2 B2", "A1 B1 B2 A2", "A1 A2 B1 B2", "A1 B1 C1 A2 B2", "A1 B1 C1 A2 C2 B2", "C1 A1 B1 B2 A2 C2"])
def test_colliding_runs_in_arrival_orders(order):
    h = _header()
    names = dict(zip("ABC", (x.decode() for x in COLLIDING_TRIPLE)))
    pos = {"A": (1000, 1400), "B": (1000, 1400), "C": (2000, 2400)}
    score = {"A": 30, "B": 35, "C": 30}
    recs = []
    for tok in order.split():
        who, mate = tok[0], tok[1]
        p1, p2 = pos[who]
        recs.append(R(names[who], 99 if mate == "1" else 147, p1 if mate == "1" else p2, score[who], RNEXT="=", PNEXT=p2 if mate == "1" else p1))
    flag = _join_case(recs, h)
    assert _dup(flag, recs, names["A"]) == ([True, True] if "B" in order else [False, False])
    assert not any(_dup(flag, recs, names["B"])) and not any(_dup(flag, recs, names["C"]))


def test_colliding_names_of_different_lengths():
    h = _header()
    a, b_ = (x.decode() for x in COLLIDING_LENGTHS)
    recs = pair(a, 1000, 1300, 30) + pair(b_, 1000, 1300, 31)
    recs = [recs[0], recs[2], recs[1], recs[3]]
    flag = _join_case(recs, h)
    assert _dup(flag, recs, a) == [True, True] and _dup(flag, recs, b_) == [False, False]


@pytest.mark.parametrize("k", [3, 4, 5])
def test_qname_used_k_times(k):
    """one QNAME as k true-pair primaries (concatenated inputs): DeleteOrStore pairs the 1st with the 2nd, the 3rd with the 4th;
    an odd last read stays unpaired.  Also inside a run of colliding keys."""
    h = _header()
    a, b_ = (x.decode() for x in COLLIDING_PAIRS[1])
    recs = []
    for j in range(k):
        recs.append(R("same", 99 if j % 2 == 0 else 147, 1000 + 500 * (j // 2) if j % 2 == 0 else 1300 + 500 * (j // 2), 30 + j))
        recs.append(R(a, 99 if j % 2 == 0 else 147, 5000 if j % 2 == 0 else 5300, 30 + j))
        if j == 1:
            recs += [R(b_, 99, 5000, 50), R(b_, 147, 5300, 50)]
    flag = _join_case(recs, h, optical=False)
    assert not any(_dup(flag, recs, "same"))                          # every pair of "same" has its own signature
    # (a 1st, a 2nd) and (a 3rd, a 4th) and b_ share the signature at 5000/5300: b_ (score 100) wins
    assert _dup(flag, recs, b_) == [False, False]
    assert _dup(flag, recs, a) == [True] * (k - k % 2) + [False] * (k % 2)   # an odd last read is unpaired: never a pair duplicate


def test_same_qname_in_two_libraries():
    h = _header(1, 2)
    recs = [R("q", 99, 1000, 30, rg="rg0"), R("q", 99, 1000, 40, rg="rg1"), R("q", 147, 1300, 30, rg="rg1"), R("q", 147, 1300, 30, rg="rg0")]
    recs += pair("r", 1000, 1300, 20, rg="rg0") + pair("r", 1000, 1300, 25, rg="rg0")   # same signature as q of rg0, lower scores
    flag = _join_case(recs, h, optical=False)
    assert join_hash([b"q"], 0)[0] != join_hash([b"q"], 1)[0]
    assert [bool(f & 0x400) for f in flag[:4]] == [False, False, False, False]
    assert _dup(flag, recs, "r") == [True, True, True, True]


# ---------------------------------------------------------------- D. optical limits
D = 100


def _optical_run(coords, strands=None, p1=10_000, p2=10_400, rg="rg0", tile=1101):
    """one duplicate set: pair k at (x, y) = coords[k]; strands[k] = 1 puts its first-of-pair read on the reverse strand"""
    recs = []
    for k, (x, y) in enumerate(coords):
        t = tile(k) if callable(tile) else tile
        nm = f"M:1:FC:1:{t}:{x}:{y}"
        rev_first = strands is not None and strands[k]
        flags = (163, 83) if rev_first else (99, 147)
        recs += pair(nm, p1, p2, 30 + (k % 5), flags=flags, rg=rg)
    return recs


def _opt_metrics(recs, h, expect_optical):
    b = sam.AlignmentBatch.from_records(h, recs)
    check(b, h, pixel=D)
    if expect_optical is not None:
        import oracle
        om = oracle.markdup_optical(b.copy(), h, pixel_distance=D)
        assert om.counters[1]["read_pair_optical_duplicates"] == expect_optical


# name: (x, y of pair k; strand of its first-of-pair read; optical duplicates = members - clusters, over both strand lists)
TOPOLOGIES = {
    "one_cluster": (lambda n: [(1000 + k, 2000) for k in range(n)], None, lambda n: n - 1),
    "none": (lambda n: [(1000 + k * (D + 1), 2000) for k in range(n)], None, lambda n: 0),
    "chain": (lambda n: [(1000 + k * D, 2000 + (k % 2) * D) for k in range(n)], None, lambda n: n - 1),
    "two_chains": (lambda n: [(1000 + (k // 2) * D, 2000 + (k % 2) * 10 * D) for k in range(n)], None, lambda n: n - 2),
    # one chain per strand list: neighbours in a list are D apart
    "both_strands": (lambda n: [(1000 + (k // 2) * D, 2000 + k % 2) for k in range(n)], lambda n: [k % 2 for k in range(n)], lambda n: n - 2),
}


@pytest.mark.parametrize("n", [32, 33])
@pytest.mark.parametrize("topo", list(TOPOLOGIES))
def test_optical_run_lengths(n, topo):
    """32 pairs: one thread and a byte union-find; 33: one block and the CAS union-find"""
    coords, strands, expect = TOPOLOGIES[topo]
    recs = _optical_run(coords(n), strands(n) if strands else None)
    _opt_metrics(recs, _header(), expect(n))


@pytest.mark.parametrize("dx,clustered", [(D, True), (D + 1, False)])
def test_optical_distance_edge(dx, clustered):
    h = _header()
    recs = _optical_run([(1000, 1000), (1000 + dx, 1000 - dx)])
    recs += _optical_run([(1000, 1000), (1000 - dx, 1000), (5000, 5000 + dx)], p1=20_000, p2=20_300)
    _opt_metrics(recs, h, 2 if clustered else 0)


def test_optical_set_over_histogram_bins():
    """a duplicate set of 1100 pairs: the histogram keys 1100 (all) and 1100 - optical go through the overflow list"""
    h = _header()
    n = 1100
    coords = [(1000 + (k // 2) * (D + 1), 2000 + (k % 2)) for k in range(n)]     # clusters of two
    recs = _optical_run(coords) + _optical_run([(1, 1), (1, 2)], p1=50_000, p2=50_300)
    _opt_metrics(recs, h, n // 2 + 1)


def _optical_columns(n_fwd, n_rev, p1=10_000, p2=10_400):
    """a batch of n_fwd + n_rev pairs of one signature built column-wise (first-of-pair on the reverse strand for the last n_rev)"""
    n = n_fwd + n_rev
    names = [f"M:1:FC:1:7:{k}:{k % 997}".encode() for k in range(n)]
    qn = np.frombuffer(b"".join(nm for nm in names for _ in (0, 1)), np.uint8)
    lens = np.repeat(np.array([len(x) for x in names], np.uint64), 2)
    qoff = np.zeros(2 * n + 1, np.uint64)
    np.cumsum(lens, out=qoff[1:])
    rev = np.r_[np.zeros(n_fwd, bool), np.ones(n_rev, bool)]
    flag = np.empty(2 * n, np.uint16)
    flag[0::2] = np.where(rev, 163, 99)
    flag[1::2] = np.where(rev, 83, 147)
    pos = np.tile(np.array([p1, p2], np.int32), n)
    score = (30 + np.arange(2 * n) % 5).astype(np.uint8)
    return sam.AlignmentBatch(refid=np.zeros(2 * n, np.int32), pos=pos, flag=flag, mapq=np.full(2 * n, 60, np.uint8),
                              nref=np.zeros(2 * n, np.int32), pnext=np.tile(np.array([p2, p1], np.int32), n), tlen=np.zeros(2 * n, np.int32),
                              rg=np.zeros(2 * n, np.int32), qname_off=qoff, qname=qn, cigar_off=np.arange(2 * n + 1, dtype=np.uint64),
                              cigar=np.full(2 * n, 4 << 4, np.uint32), lseq=np.full(2 * n, 4, np.int32),
                              seq=np.full(4 * n, 0x11, np.uint8), qual=np.repeat(score, 4))


def test_optical_list_cap():
    """300 001 first-of-pair reads on the forward strand (past the 300 000 cap: not clustered) and 5 on the reverse strand
    (clustered).  Exactly 300 000 is left out: the clustering is quadratic in the list length on both sides."""
    h = _header()
    b = _optical_columns(300_001, 5)
    check(b, h, pixel=D)
    import oracle
    om = oracle.markdup_optical(b.copy(), h, pixel_distance=D)
    assert om.counters[1]["read_pair_optical_duplicates"] == 4        # the 5 reverse ones: x = k and k+1 apart: one cluster
    assert om.hist[1][0] == {300_006: 1}


@pytest.mark.parametrize("value,code", [("2147483647", 0), ("-2147483648", 0), ("2147483648", _lib.ELIMIT), ("-2147483649", _lib.ELIMIT),
                                        ("9223372036854775808", ETILE), ("x12", ETILE)])
@pytest.mark.parametrize("field", [0, 1, 2])
@pytest.mark.parametrize("in_list", [True, False])
def test_tile_values_at_int32_limits(value, code, field, in_list):
    """a tile/x/y value is parsed only for a strand list of two or more reads"""
    from elprep_b200 import device
    h = _header()
    tx = ["1101", "1000", "1000"]
    tx[field] = value
    odd = f"M:1:FC:1:{tx[0]}:{tx[1]}:{tx[2]}"
    recs = pair(odd, 10_000, 10_400, 30) + pair("M:1:FC:1:1101:1000:1050", 10_000, 10_400, 35)
    if not in_list:
        recs[0]["FLAG"], recs[1]["FLAG"] = 163, 83                   # the odd pair's first-of-pair read is on the other strand
    recs += pair("M:1:FC:1:1101:1:1", 30_000, 30_300)
    b = sam.AlignmentBatch.from_records(h, recs)
    if code == 0 or not in_list:
        check(b, h, pixel=D)
        return
    ctx = _ctx(h, optical_pixel_distance=D)
    try:
        ctx.append(b)
        with pytest.raises(device.ElprepError) as ei:
            ctx.sort_markdup(device.SO_COORDINATE, _lib.MARKDUP_OPTICAL)
        assert ei.value.code == code
    finally:
        ctx.close()
