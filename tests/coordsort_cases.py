"""Inputs for the coordinate and queryname sort at their edges (tests/test_gpu_coordsort_edges.py), built column-wise so that a QNAME can
hold any byte.  Each builder returns (batch, n_contigs); CASES maps a name to a builder, and test_coordsort_ref_cpu.py pins the
restatement in coordsort_ref.py to the oracle on every case without an empty QNAME."""
import numpy as np

from elprep_b200 import sam

I32_MAX, I32_MIN = 2 ** 31 - 1, -2 ** 31
ALPHA = b"ABCDEFGHIJKLMNOPQRSTUVWXYZabcdefghijklmnopqrstuvwxyz0123456789:_"


def header(n_contigs, ln=I32_MAX):
    return sam.Header(sq=[{"SN": f"c{i}", "LN": ln} for i in range(n_contigs)])


def columns(names, refid, pos, flag=0, mapq=60, nref=-1, pnext=0, tlen=0):
    """one read per name; the other fields are scalars or per-read sequences.  Every read has CIGAR 4M and four bases."""
    n = len(names)
    col = lambda v, dt: np.ascontiguousarray(np.broadcast_to(np.asarray(v, dtype=np.int64), (n,)).astype(dt))
    qoff = np.zeros(n + 1, np.uint64)
    np.cumsum([len(x) for x in names], out=qoff[1:])
    return sam.AlignmentBatch(refid=col(refid, np.int32), pos=col(pos, np.int32), flag=col(flag, np.uint16), mapq=col(mapq, np.uint8),
                              nref=col(nref, np.int32), pnext=col(pnext, np.int32), tlen=col(tlen, np.int32), rg=np.full(n, -1, np.int32),
                              qname_off=qoff, qname=np.frombuffer(b"".join(names), np.uint8).copy(),
                              cigar_off=np.arange(n + 1, dtype=np.uint64), cigar=np.full(n, 4 << 4, np.uint32), lseq=np.full(n, 4, np.int32),
                              seq=np.full(2 * n, 0x12, np.uint8), qual=np.full(4 * n, 30, np.uint8))


def shuffled(b, seed):
    return b.take(np.random.default_rng(seed).permutation(b.n))


def rand_name(rng, lo, hi, alphabet=ALPHA):
    return bytes(rng.choice(np.frombuffer(alphabet, np.uint8), size=int(rng.integers(lo, hi + 1))))


# secondary fields drawn per read inside a run: every value a clause treats specially, few enough that full ties happen
FLAGS_FWD = [0x0, 0x1, 0x3, 0x9, 0x21, 0x29, 0x8, 0x20, 0x28, 0x41, 0x81, 0x100, 0x200, 0x800, 0x4, 0x5, 0xd, 0x400]
MAPQS, NREFS, PNEXTS, TLENS = [0, 1, 60, 254, 255], [-1, 0, "last"], [0, 1, I32_MAX], [I32_MIN, -1, 0, 1, I32_MAX]


def run_reads(rng, L, refid, pos, rev, n_contigs, names):
    """L reads with one primary key and random secondary fields; names: a pool to draw QNAMEs from"""
    fl = np.array([FLAGS_FWD[k] for k in rng.integers(0, len(FLAGS_FWD), L)], np.uint16) | np.uint16(0x10 if rev else 0)
    nr = [n_contigs - 1 if v == "last" else v for v in (NREFS[k] for k in rng.integers(0, len(NREFS), L))]
    if n_contigs == 0:
        nr = [-1] * L
    return dict(names=[names[k] for k in rng.integers(0, len(names), L)], refid=[refid] * L, pos=[pos] * L, flag=fl,
                mapq=[MAPQS[k] for k in rng.integers(0, len(MAPQS), L)], nref=nr, pnext=[PNEXTS[k] for k in rng.integers(0, len(PNEXTS), L)],
                tlen=[TLENS[k] for k in rng.integers(0, len(TLENS), L)])


def from_runs(runs):
    cols = {k: [] for k in ("names", "refid", "pos", "flag", "mapq", "nref", "pnext", "tlen")}
    for r in runs:
        for k in cols:
            cols[k] += list(r[k])
    return columns(cols.pop("names"), **cols)


def primary_keys(n_contigs, count):
    """`count` distinct (refid, pos, strand) in coordinate order, spread over every contig and then the unmapped block"""
    refs = list(range(n_contigs)) + [-1]
    per = -(-count // len(refs))
    out = [(r, 100 + 7 * (k // 2), k % 2) if r >= 0 else (r, k, 0) for r in refs for k in range(per)]
    return out[:count]


def layout(run_starts, total, n_contigs, seed, name_pool):
    """runs of the given lengths starting at the given sorted positions, single reads in between, arrival order shuffled"""
    rng = np.random.default_rng(seed)
    segs, at = [], 0
    for start, L in run_starts:
        assert start >= at
        segs += [1] * (start - at) + [L]
        at = start + L
    segs += [1] * max(0, total - at)
    keys = primary_keys(n_contigs, len(segs))
    runs = [run_reads(rng, L, r, p, s, n_contigs, name_pool) for L, (r, p, s) in zip(segs, keys)]
    return shuffled(from_runs(runs), seed)


def name_pool(rng, k, lo=1, hi=12):
    return [rand_name(rng, lo, hi, b"ab") for _ in range(k)] + [rand_name(rng, lo, hi) for _ in range(k)]


RUN_LENGTHS = [1, 2, 31, 32, 33, 34, 64, 255, 256, 257, 5000]


def runs_at_block_edges(L, n_contigs=3):
    """four runs of length L: starting one before the 256 edge, one after the next 128 edge, ending on a 256 edge and starting on one"""
    s0 = 255
    s1 = ((s0 + L) // 128 + 1) * 128 + 1
    e2 = ((s1 + L) // 256 + 1) * 256 + L            # ends at e2 - 1, the read before a 256 edge
    s2 = e2 - L
    s3 = ((e2 + 1) // 256 + 1) * 256
    rng = np.random.default_rng(L)
    return layout([(s0, L), (s1, L), (s2, L), (s3, L)], s3 + L + 40, n_contigs, L, name_pool(rng, 6))


def same_coordinate(n=5000):
    rng = np.random.default_rng(5)
    return shuffled(from_runs([run_reads(rng, n, 0, 1000, 1, 1, name_pool(rng, 20))]), 5), 1


def tiny(n):
    rng = np.random.default_rng(n)
    return from_runs([run_reads(rng, n, 0, 10, 0, 1, [b"r1", b"r2"])]), 1


def no_sq():
    """no @SQ lines: every read is unmapped with REFID -1; one long run and short ones"""
    rng = np.random.default_rng(7)
    runs = [run_reads(rng, 300, -1, 0, 0, 0, name_pool(rng, 8))] + [run_reads(rng, int(rng.integers(1, 6)), -1, p, 0, 0, name_pool(rng, 4)) for p in range(1, 40)]
    return shuffled(from_runs(runs), 7), 0


# ---------------------------------------------------------------- QNAME chunk boundaries
PREFIXES = [7, 8, 9, 15, 16, 17, 63, 64, 65] + list(range(248, 254))


def qname_boundaries(run_len, seed=11):
    """names whose common prefix ends at chunk edges, names that are prefixes of each other at chunk ends, bytes 0x80-0xFF; a run of
    run_len reads per prefix length, so the same names go through tie_short (<= 32) or the long rounds"""
    rng = np.random.default_rng(seed)
    runs = []
    for k, p in enumerate(PREFIXES):
        stem = rand_name(rng, p, p)
        pool = [stem, stem[:-1], stem + b"\x00", stem[:max(1, p // 8 * 8)]]
        for tail in (b"A", b"a", b"\x7f", b"\x80", b"\xff", b"\x00A", b"\xfe\xff"):
            pool.append((stem + tail)[:254])
        pool += [(stem + rand_name(rng, 1, 254 - p, bytes(range(1, 256))))[:254] for _ in range(4)]
        runs.append(run_reads(rng, run_len, 0, 1000 + k, k % 2, 1, pool))
    # names of 1..254 bytes at every arena offset mod 16 (a random-length name in front of each sets the offset)
    runs.append(run_reads(rng, 3 * 254, 0, 5000, 0, 1, [bytes([0x30 + (L % 70)]) * L for L in range(1, 255)]))
    return shuffled(from_runs(runs), seed), 1


def qname_nq(nq, seed=None):
    """longest name exactly 8 * nq bytes (nq 1..32): a long run and short runs of names that share prefixes across chunk ends"""
    rng = np.random.default_rng(100 + nq if seed is None else seed)
    top = 8 * nq
    stems = [rand_name(rng, top, top, b"xy\x80\xff") for _ in range(3)]
    pool = [s[:L] for s in stems for L in {1, max(1, top - 8), max(1, top - 1), top, max(1, top - 9), (top // 2 // 8) * 8 or 1}]
    runs = [run_reads(rng, 90, 0, 500, 1, 2, pool)] + [run_reads(rng, int(rng.integers(2, 20)), 1, 600 + k, 0, 2, pool) for k in range(12)]
    return shuffled(from_runs(runs), nq), 2


def c583c7f_shape(seed=13):
    """the shape on which the per-byte QNAME chunk once came out wrong: a run of 2400 reads whose names are all shorter than 8 bytes (whole
    warps with a zero last chunk), and one 200-byte name elsewhere, so that nq = 25"""
    rng = np.random.default_rng(seed)
    pool = [rand_name(rng, 1, 7) for _ in range(60)]
    runs = [run_reads(rng, 2400, 0, 777, 0, 1, pool), run_reads(rng, 1, 0, 900, 0, 1, [rand_name(rng, 200, 200)])]
    runs += [run_reads(rng, 3, 0, 1000 + k, 1, 1, pool) for k in range(50)]
    return shuffled(from_runs(runs), seed), 1


# ---------------------------------------------------------------- one comparator clause at a time
CLAUSES = {
    # field: values; the other fields of the run are equal
    "modflag_fwd": ("flag", [0x0, 0x8, 0x20, 0x28, 0x1, 0x9, 0x21, 0x29, 0x100, 0x200, 0x800, 0x4, 0x5, 0xd, 0x2d, 0x3]),
    "modflag_rev": ("flag", [0x10, 0x14, 0x18, 0x30, 0x38, 0x11, 0x15, 0x19, 0x31, 0x39, 0x110, 0x114, 0x210, 0x810, 0x1d, 0x3d]),
    "mapq": ("mapq", [0, 254, 255, 60, 1]),
    "nref_paired": ("nref", [-1, 0, "last"]),
    "pnext_paired": ("pnext", [0, 1, I32_MAX]),
    "nref_pnext_unpaired": ("nref_pnext_unpaired", None),
    "tlen": ("tlen", [I32_MIN, -1, 0, 1, I32_MAX]),
    "equal": ("equal", None),
    # single differing bit: bit 0 of TLEN, bit 31 of the TLEN chunk (its sign), bits 32..63 of chunk 1 (NextREFID -1 against 0), bit 31
    # of chunk 1 (PNEXT 0 against INT32_MIN), bit 0 of MAPQ, bit 0 of the primary key (strand, two runs)
    "bit0_tlen": ("tlen", [0, 1]),
    "bit31_tlen": ("tlen", [0, I32_MIN]),
    "bits32_63_nref": ("nref", [-1, 0]),
    "bit31_pnext": ("pnext", [0, I32_MIN]),
    "bit0_mapq": ("mapq", [60, 61]),
}


def clause_case(clause, run_len, n_contigs=3, seed=17):
    field, values = CLAUSES[clause]
    rng = np.random.default_rng(seed + run_len)
    L = run_len
    base = dict(names=[b"same"] * L, refid=[1] * L, pos=[4242] * L, flag=[0x1] * L, mapq=[60] * L, nref=[0] * L, pnext=[77] * L, tlen=[5] * L)
    if field == "flag":
        base["flag"] = [values[k] for k in rng.integers(0, len(values), L)]
    elif field == "nref_pnext_unpaired":
        base["flag"] = [0] * L
        base["nref"] = [[-1, 0, n_contigs - 1][k] for k in rng.integers(0, 3, L)]
        base["pnext"] = [[0, 1, I32_MAX][k] for k in rng.integers(0, 3, L)]
    elif field != "equal":
        base[field] = [n_contigs - 1 if values[k] == "last" else values[k] for k in rng.integers(0, len(values), L)]
    runs = [base]
    if clause == "equal":                               # a second run that differs from the first in the strand bit only
        runs.append(dict(base, flag=[0x11] * L))
    runs.append(run_reads(rng, 5, 0, 10, 0, n_contigs, [b"x"]))
    return shuffled(from_runs(runs), seed), n_contigs


# ---------------------------------------------------------------- primary key widths
def key_widths(n_contigs, seed=19):
    """POS up to 2^31 - 1 on the first and last contig, a long run at the very end of the last contig next to the unmapped block, and
    unmapped reads placed with their mate (REFID and POS set, 0x4) next to mapped reads and to fully unmapped ones"""
    rng = np.random.default_rng(seed + n_contigs)
    last = n_contigs - 1
    pool = name_pool(rng, 5)
    runs = []
    for r in sorted({0, last}):
        for p in (0, 1, 2, 2 ** 30, I32_MAX - 1):
            runs.append(run_reads(rng, int(rng.integers(1, 4)), r, p, int(rng.integers(0, 2)), n_contigs, pool))
    runs.append(run_reads(rng, 70, last, I32_MAX, 0, n_contigs, pool))
    placed = run_reads(rng, 40, last, I32_MAX, 0, n_contigs, pool)
    placed["flag"] = np.asarray(placed["flag"]) | np.uint16(0x4)       # unmapped, with the mate's RNAME and POS: same primary key
    runs.append(placed)
    runs.append(run_reads(rng, 60, -1, 0, 0, n_contigs, pool))
    unm = runs[-1]
    unm["flag"] = np.asarray(unm["flag"]) | np.uint16(0x4)
    if n_contigs > 3:
        runs += [run_reads(rng, 2, int(r), int(rng.integers(1, I32_MAX)), 0, n_contigs, pool) for r in rng.integers(0, n_contigs, 300)]
    return shuffled(from_runs(runs), seed), n_contigs


# ---------------------------------------------------------------- QNAMEs that differ only by trailing NUL bytes
NUL_NAMES = [b"a", b"a\x00", b"a\x00\x00", b"ab\x00c", b"ab", b"ab\x00", b"a\x00b", b"b"]


def trailing_nuls(run_len, seed=23):
    rng = np.random.default_rng(seed + run_len)
    runs = [run_reads(rng, run_len, 0, 300, 0, 1, NUL_NAMES)]
    for r in runs:                                      # equal secondary fields: only the name orders the run
        for k in ("flag", "mapq", "nref", "pnext", "tlen"):
            r[k] = [r[k][0]] * run_len
    runs.append(run_reads(rng, 3, 0, 1, 0, 1, [b"z"]))
    return shuffled(from_runs(runs), seed), 1


def long_names(size, run_len=40, seed=29):
    """names of `size` bytes that differ in a few places (first, middle and last chunk) and by length, in one long run"""
    rng = np.random.default_rng(seed)
    stem = bytearray(rand_name(rng, size, size))
    pool = []
    for at in (3, size // 2, size - 2):
        for v in (b"A", b"z"):
            s = bytearray(stem)
            s[at:at + 1] = v
            pool.append(bytes(s))
    pool += [bytes(stem), bytes(stem[:-1]), bytes(stem) + b"\x00"]
    runs = [run_reads(rng, run_len, 0, 55, 0, 1, pool), run_reads(rng, 5, 0, 56, 0, 1, [b"q"])]
    return shuffled(from_runs(runs), seed), 1


def large(n=1_000_000, seed=31):
    """about 30 % of the reads in runs of 33..400, the rest in short runs and singles; names of 1..40 bytes over a small alphabet"""
    rng = np.random.default_rng(seed)
    names_alpha = np.frombuffer(b"ACGT:_0123456789", np.uint8)
    n_contigs = 5
    runs, total, key = [], 0, 0
    while total < n:
        L = int(rng.integers(33, 401)) if rng.random() < 0.008 else int(rng.integers(1, 8))
        total += L
        runs.append((L, key))
        key += 1
    refid = np.empty(total, np.int64)
    pos = np.empty(total, np.int64)
    flag = np.empty(total, np.uint16)
    at = 0
    per = -(-key // (n_contigs + 1))
    for L, k in runs:
        c, p = divmod(k, per)
        refid[at:at + L] = c if c < n_contigs else -1
        pos[at:at + L] = 1 + p // 2 * 3
        flag[at:at + L] = 0x10 * (p % 2) if c < n_contigs else 0x4
        at += L
    fl = np.array(FLAGS_FWD, np.uint16)[rng.integers(0, len(FLAGS_FWD), total)] & ~np.uint16(0x10)
    flag = flag | fl
    lens = rng.integers(1, 41, total)
    qn = names_alpha[rng.integers(0, 4, int(lens.sum()))]          # ACGT only: many equal prefixes
    qoff = np.zeros(total + 1, np.uint64)
    np.cumsum(lens, out=qoff[1:])
    names = [bytes(qn[int(qoff[i]):int(qoff[i + 1])]) for i in range(total)]
    nr = np.array([-1, 0, n_contigs - 1], np.int64)[rng.integers(0, 3, total)]
    b = columns(names, refid, pos, flag, np.array(MAPQS)[rng.integers(0, len(MAPQS), total)], nr,
                np.array(PNEXTS[:2] + [I32_MAX])[rng.integers(0, 3, total)], np.array(TLENS, np.int64)[rng.integers(0, len(TLENS), total)])
    return shuffled(b, seed), n_contigs


CASES = {f"runs_{L}": (lambda L=L: (runs_at_block_edges(L), 3)) for L in RUN_LENGTHS}
CASES.update({"same_coordinate": same_coordinate, "n1": lambda: tiny(1), "n2": lambda: tiny(2), "no_sq": no_sq,
              "qname_short": lambda: qname_boundaries(20), "qname_long": lambda: qname_boundaries(120),
              "c583c7f": c583c7f_shape})
CASES.update({f"nq_{nq}": (lambda nq=nq: qname_nq(nq)) for nq in range(1, 33)})
CASES.update({f"clause_{c}_{L}": (lambda c=c, L=L: clause_case(c, L)) for c in CLAUSES for L in (20, 100)})
CASES.update({f"widths_{nc}": (lambda nc=nc: key_widths(nc)) for nc in (1, 2, 3, 4000)})
CASES.update({f"nuls_{L}": (lambda L=L: trailing_nuls(L)) for L in (8, 200)})
CASES.update({"names_4k": lambda: long_names(4096), "names_40k": lambda: long_names(40960)})
