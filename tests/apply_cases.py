"""Hand-built reads for the edges of BQSR apply (bqsr_apply2_kernel and bqsr_apply_kernel, csrc/bqsr_apply.cu).

A "context" is a list of read specs in OUTPUT order (coordinate order: mapped reads at increasing POS, then the unmapped ones).  The
batch is built in the reverse order, so that QUAL and SEQ arena offsets mod 16 differ from the output phases.  The longest read of a
context fixes lanes per read / reads per warp pass of both kernels, so every short read is processed the way that one read dictates.

Spec fields: L, flag, qual (list of ints), seq (str or None: the reference with a few mismatches), rg (index or None), mapq, kind
("mapped" | "secondary" | "unmapped").  SEQ and QUAL are written exactly; a spec's seq may carry N, IUPAC codes and '='."""
from __future__ import annotations

import numpy as np

from elprep_b200 import sam, synth

CONTIG = "chr20"
IUPAC = "=MRSVWYHKDB"                   # every nibble that is neither A, C, G, T nor N
FLAGS = {"fwd": 0x0, "rev": 0x10, "first": 0x1 | 0x40, "first_rev": 0x1 | 0x40 | 0x10, "second": 0x1 | 0x80,
         "second_rev": 0x1 | 0x80 | 0x10, "last_unpaired": 0x80, "last_unpaired_rev": 0x80 | 0x10}


def header(n_rg=4):
    """rg1 and rg2 share PU FC1.1 (one covariate); rg3 has no PU (its ID is the covariate); rg4's covariate gets no table entries"""
    rg = [{"ID": "rg1", "PU": "FC1.1", "LB": "lib"}, {"ID": "rg2", "PU": "FC1.1", "LB": "lib"}, {"ID": "rg3", "LB": "lib"},
          {"ID": "rg4", "PU": "FC9.9", "LB": "lib"}][:n_rg]
    return sam.Header(sq=[{"SN": CONTIG, "LN": 400_000}], rg=rg, so=sam.Unsorted)


def genome(seed=7):
    return synth.make_workload(1, [(CONTIG, 400_000)], seed=seed, n_rg=1).contig_bases[0]


def spec(L, flag=0, qual=None, seq=None, rg=0, mapq=60, kind="mapped"):
    return dict(L=L, flag=flag, qual=qual, seq=seq, rg=rg, mapq=mapq, kind=kind)


def build(specs, hdr, ref, quals=(12, 23, 37), seed=0, mismatch=0.03):
    """-> (Workload, output-order index of every spec in the batch) -- arrival order is the reverse of output order"""
    rng = np.random.default_rng(seed)
    recs, pos = [], 1000
    for k, s in enumerate(specs):
        L = s["L"]
        q = list(s["qual"]) if s["qual"] is not None else [int(x) for x in rng.choice(quals, size=L)]
        assert len(q) == L
        p = pos
        pos += max(L, 1) + 7
        if s["seq"] is not None:
            bases = s["seq"]
        else:
            b = [chr(x) for x in ref[p - 1:p - 1 + L]]
            for i in np.nonzero(rng.random(L) < mismatch)[0]:
                b[i] = "ACGT"[("ACGT".index(b[i]) + 1 + int(rng.integers(0, 3))) % 4] if b[i] in "ACGT" else "A"
            bases = "".join(b)
        assert len(bases) == L
        flag = s["flag"] | (0x100 if s["kind"] == "secondary" else 0) | (0x4 if s["kind"] == "unmapped" else 0)
        mapped = s["kind"] != "unmapped"
        paired = bool(flag & 1)
        recs.append(dict(QNAME=f"r{k:06d}", FLAG=flag, RNAME=CONTIG if mapped else "*", POS=p if mapped else 0, MAPQ=s["mapq"] if mapped else 0,
                         CIGAR=f"{L}M" if (mapped and L) else "*", RNEXT="=" if (paired and mapped) else "*", PNEXT=p if (paired and mapped) else 0,
                         TLEN=0, SEQ=bases, QUAL=q, RG=(hdr.RG[s["rg"]]["ID"] if s["rg"] is not None else None)))
    batch = sam.AlignmentBatch.from_records(hdr, recs[::-1])
    return synth.Workload(hdr, batch, [ref], [np.zeros((0, 2), np.int32)], {}), np.arange(len(specs))[::-1]


# ---------------------------------------------------------------- contexts
def _flag_cycle():
    while True:
        for f in FLAGS.values():
            yield f


def lengths_context(longest, seed=0):
    """the listed read lengths up to ``longest`` (and ``longest`` itself) on every flag, many 0-40 base reads in between, passes made of
    empty reads only, and slices of 0, 1, 15, 16 and 17 bytes"""
    rng = np.random.default_rng(seed)
    fl = _flag_cycle()
    lens = [x for x in (1, 2, 15, 16, 17, 31, 32, 33, 63, 64, 65, 100, 151, 255, 256, 257, 511, 512, 1023, 1024) if x <= longest] + [longest]
    rpw = 32 // min(32, max(1, (longest + 31) // 32))
    out = []
    for L in lens:
        for _ in range(len(FLAGS) * max(1, rpw // 2)):      # enough passes that every 16-byte phase starts one
            out.append(spec(L, next(fl)))
            for _ in range(int(rng.integers(0, 4))):
                out.append(spec(int(rng.integers(0, 41)) if longest >= 40 else int(rng.integers(0, longest + 1)), next(fl)))
    # whole passes of 0, 1, 15, 16, 17 bytes, one made only of empty reads, between non-empty ones
    for total in (0, 1, 15, 16, 17, 0):
        part = [0] * rpw
        left, i = total, 0
        while left:
            take = min(left, longest, 1 + int(rng.integers(0, 16)))
            part[i % rpw] += take
            left -= take
            i += 1
        part = [min(x, longest) for x in part]
        out += [spec(x, next(fl)) for x in part]
    # a slice that ends exactly on a 16-byte boundary: pad until the output offset is a multiple of 16 at a pass end
    n_before = len(out)
    off = sum(s["L"] for s in out)
    pad = (-off) % 16
    fill = [0] * ((-n_before) % rpw or rpw)
    fill[0] = pad
    out += [spec(x, next(fl)) for x in fill]
    out += [spec(int(rng.integers(1, longest + 1)), next(fl)) for _ in range(int(rng.integers(3 * rpw, 5 * rpw)) | 1)]   # n not a multiple of rpw
    return out


def many_short_in_long(longest=1024, n=4000, seed=1):
    """one longest read, then many 1-40-base reads (one per warp pass each, with 1024)"""
    rng = np.random.default_rng(seed)
    fl = _flag_cycle()
    return [spec(longest, 0x10)] + [spec(int(rng.integers(1, 41)), next(fl)) for _ in range(n)] + [spec(longest - 1, 0x1 | 0x80)]


def tail_context(L=100, seed=2):
    """QUAL <= 2 prefixes and suffixes of 0, 1, 31, 32, 33, L-1 and L bases, alone and together; reads whose only QUAL > 2 base sits at
    31 or 32; on both strands and both mates"""
    rng = np.random.default_rng(seed)
    out = []
    cuts = sorted({0, 1, 31, 32, 33, L - 1, L})
    for f in (0, 0x10, 0x1 | 0x80, 0x1 | 0x80 | 0x10):
        for a in cuts:
            for b in cuts:
                if a + b > L and not (a == L and b == 0):
                    continue
                q = [int(x) for x in rng.choice((12, 23, 37, 6, 5), size=L)]
                for i in range(a):
                    q[i] = int(rng.integers(0, 3))
                for i in range(L - b, L):
                    q[i] = int(rng.integers(0, 3))
                out.append(spec(L, f, q))
        for only in (31, 32):
            q = [int(rng.integers(0, 3)) for _ in range(L)]
            q[only] = 30
            out.append(spec(L, f, q))
    return out


def base_context(ref, L=100, seed=3):
    """N and every IUPAC code at the first and last base, at 31/32 and 63/64, and in runs, on both strands.  A code among the first two
    bases of the stranded sequence makes contextWith panic unless the second one is N, so there the code is paired with an N."""
    rng = np.random.default_rng(seed)
    out, p = [], 0
    for f in (0, 0x10, 0x1 | 0x40, 0x1 | 0x80 | 0x10):
        rev = bool(f & 0x10)
        for x in "N" + IUPAC:
            for where in ("first", "last", "31", "32", "63", "64", "run"):
                b = ["ACGT"[int(v)] for v in rng.integers(0, 4, size=L)]
                if where == "first":
                    b[0] = x
                    if not rev:
                        b[1] = "N"
                elif where == "last":
                    b[L - 1] = x
                    if rev:
                        b[L - 2] = "N"
                elif where == "run":
                    for i in range(40, 40 + 1 + int(rng.integers(1, 6))):
                        b[i] = x if i % 3 else "N"
                else:
                    b[int(where)] = x
                out.append(spec(L, f, seq="".join(b)))
                p += 1
    return out


def qual_context(L=100, seed=4, every_value=True):
    """QUAL 5/6, 93 and every value 0-93 in mapped reads (every_value); 94, 127, 128 and 255 in reads that apply recalibrates but the
    gather does not count (unmapped, secondary, MAPQ 0), next to and inside low-quality tails"""
    rng = np.random.default_rng(seed)
    out = []
    for f in (0, 0x10, 0x1 | 0x80):
        if every_value:
            out.append(spec(94, f, list(range(94))))
            out.append(spec(94, f | 0x10, list(range(93, -1, -1))))
            out.append(spec(L, f, [int(x) for x in rng.choice((5, 6, 93), size=L)]))
        else:
            out.append(spec(L, f))
    high = (94, 127, 128, 255)
    for kind, mapq in (("unmapped", 0), ("secondary", 60), ("mapped", 0)):
        for f in (0, 0x10, 0x1 | 0x80, 0x1 | 0x40 | 0x10):
            for h in high:
                q = [int(x) for x in rng.choice((2, 12, 37, h, h), size=L)]
                out.append(spec(L, f, q, mapq=mapq, kind=kind))
            q = [255] + [int(x) for x in rng.choice((12, 37), size=L - 2)] + [255]   # 0xFF at both ends: not a tail (byte comparison)
            out.append(spec(L, f, q, mapq=mapq, kind=kind))
            q = [1, 2, 255] + [int(x) for x in rng.choice((12, 128), size=L - 6)] + [94, 0, 2]
            out.append(spec(L, f, q, mapq=mapq, kind=kind))
    return out


def read_group_context(L=60, seed=5):
    """reads in every read group, rg4 with no table entries (all its reads unmapped, QUAL above 93 included), empty reads"""
    rng = np.random.default_rng(seed)
    out = []
    for rg in (0, 1, 2):
        out += [spec(L, f, rg=rg) for f in (0, 0x10, 0x1 | 0x80)]
        out.append(spec(0, 0, qual=[], seq="", rg=rg))
    out += [spec(L, f, [int(x) for x in rng.choice((12, 37, 200), size=L)], rg=3, mapq=0, kind="unmapped") for f in (0, 0x10)]
    out.append(spec(0, 0, qual=[], seq="", rg=3, kind="unmapped"))
    return out


def quirk_reads():
    """(seq, qual, flag) whose contextWith keys differ from the plain 2-mer rule at the read start (the device does not restate this)"""
    q = [30] * 8
    return [("RACGTACG", q, 0), ("ARCGTACG", q, 0), ("NRACGTAC", q, 0), ("N=ACGTAC", q, 0), ("CGTACGYA", q, 0x10), ("CGTACGMN", q, 0x10),
            ("=ACGTACG", q, 0), ("CGTACGAR", q, 0x10), ("ARCGTACG", [2] + [30] * 7, 0)]


# ---------------------------------------------------------------- crafted tables
def crafted_dense(n_cov, max_cycle, quals, seed=9, empty_covs=(), longest=1024):
    """dense tables [n_cov][94][1 + (2 max_cycle + 1) + 16][2] in which every cycle and every context column of every QUAL row has its own
    mismatch rate (Phred 8..45 drawn per column), with 10^6 observations per column"""
    rng = np.random.default_rng(seed)
    ncol = 1 + (2 * max_cycle + 1) + 16
    d = np.zeros((n_cov, 94, ncol, 2), np.int64)
    lim = min(max_cycle, longest)
    cols = [1 + c + max_cycle for c in range(-lim, lim + 1) if c != 0] + [1 + 2 * max_cycle + 1 + x for x in range(16)]
    for cv in range(n_cov):
        if cv in empty_covs:
            continue
        for q in quals:
            if not 6 <= q <= 93:
                continue
            obs = 10 ** 7
            d[cv, q, 0] = (obs, int(obs * 10 ** (-q / 10) * rng.uniform(0.3, 3)))
            ph = rng.uniform(8, 45, size=len(cols))
            d[cv, q, cols, 0] = 10 ** 6
            d[cv, q, cols, 1] = (10 ** 6 * 10 ** (-ph / 10)).astype(np.int64)
    return d


def oracle_tables(dense, max_cycle):
    """the C ABI's dense layout -> finalized oracle tables (QUAL rows 94..255 empty)"""
    import oracle
    n_cov = dense.shape[0]
    t = oracle.OracleTables(n_cov, max_cycle)
    nc = 2 * max_cycle + 1
    t.q_obs[:, :94], t.q_mis[:, :94] = dense[:, :, 0, 0], dense[:, :, 0, 1]
    t.c_obs[:, :94], t.c_mis[:, :94] = dense[:, :, 1:1 + nc, 0], dense[:, :, 1:1 + nc, 1]
    t.x_obs[:, :94], t.x_mis[:, :94] = dense[:, :, 1 + nc:, 0], dense[:, :, 1 + nc:, 1]
    oracle.bqsr_finalize(t)
    return t
