"""The device sort's two orders restated on the CPU in plain Python, and the chunk keys of its long-tie rounds.

coordinate_order is CoordinateLess (sam/sam-types.go:425-473) as a stable sort on one tuple per read; queryname_order is QNAMELess
(:479-481).  chunk_keys gives what coordsort.cu's chunk_key returns for every read, and tie_rounds which of those chunks the
long-tie rounds sort and over which bits, so a test can check the path a case took as well as its order."""
import numpy as np

F_PAIRED, F_UNMAPPED, F_NEXTUNMAPPED, F_REVERSED, F_NEXTREVERSED = 0x1, 0x4, 0x8, 0x10, 0x20
SHORT_RUN = 32      # runs of more than this many equal primary keys take the long-tie rounds
QC0 = 4             # chunk id of the last QNAME chunk; 3 counts the trailing NUL bytes of the QNAME


def passes(bits):
    """digit passes of one radix sort over `bits` bits"""
    return (max(bits, 1) + 7) // 8


def mod_flag(f):
    """sam-types.go:408-420"""
    f = np.asarray(f, np.uint16).copy()
    f[(f & F_PAIRED) == 0] &= ~np.uint16(F_NEXTUNMAPPED | F_NEXTREVERSED)
    f[(f & F_UNMAPPED) != 0] &= ~np.uint16(F_REVERSED)
    f[(f & F_NEXTUNMAPPED) != 0] &= ~np.uint16(F_NEXTREVERSED)
    return f.astype(np.uint64)


def qnames(b):
    return [bytes(b.qname[int(b.qname_off[i]):int(b.qname_off[i + 1])]) for i in range(b.n)]


def pos_bits(b):
    """bP: the POS field of the primary key, sized by the largest POS"""
    return int(max(0, int(b.pos.max()) if b.n else 0)).bit_length()


def primary_key(b, n_contigs, bP=None):
    """(refid with -1 last | POS | strand), the key of the first radix sort and the last tie chunk"""
    bP = pos_bits(b) if bP is None else bP
    refid = b.refid.astype(np.int64)
    rr = np.where((refid < 0) | (refid >= n_contigs), n_contigs, refid).astype(np.uint64)
    return ((b.flag & F_REVERSED) != 0).astype(np.uint64) | (b.pos.astype(np.uint64) << np.uint64(1)) | (rr << np.uint64(1 + bP))


def coordinate_order(b, n_contigs):
    """perm[k] = arrival index of the k-th read.  One tuple per read, arrival index last (a stable sort):
    refid (-1 as n_contigs), POS, strand, QNAME bytes (Python bytes compare unsigned, a prefix first; the empty name is the smallest,
    the device's documented deviation), modFlag, MAPQ, NextREFID and PNEXT, TLEN.
    NextREFID and PNEXT count only if both reads are paired; zeroing them for unpaired reads is the same thing, because modFlag keeps
    0x1 and so a paired and an unpaired read are ordered by modFlag before they get there."""
    names = qnames(b)
    refid = b.refid.astype(np.int64)
    rr = np.where(refid < 0, n_contigs, refid).tolist()
    rev = ((b.flag & F_REVERSED) != 0).tolist()
    mf = mod_flag(b.flag).tolist()
    paired = (b.flag & F_PAIRED) != 0
    nref = np.where(paired, b.nref, 0).tolist()
    pnext = np.where(paired, b.pnext, 0).tolist()
    pos, mapq, tlen = b.pos.tolist(), b.mapq.tolist(), b.tlen.tolist()
    keys = [(rr[i], pos[i], rev[i], names[i], mf[i], mapq[i], nref[i], pnext[i], tlen[i], i) for i in range(b.n)]
    return np.array(sorted(range(b.n), key=keys.__getitem__), dtype=np.int64)


def queryname_order(b):
    names = qnames(b)
    return np.array(sorted(range(b.n), key=names.__getitem__), dtype=np.int64)


def n_qname_chunks(b):
    qlen = np.diff(b.qname_off.astype(np.int64))
    return max(1, (int(qlen.max()) + 7) // 8 if b.n else 1)


def trailing_nuls(b):
    return np.array([len(s) - len(s.rstrip(b"\0")) for s in qnames(b)], dtype=np.uint64)


def chunk_keys(b, chunk, nq, n_contigs, bP=None):
    """what chunk_key(chunk) returns for every read, in arrival order: 0 TLEN, 1 NextREFID|PNEXT (0 unless paired), 2 modFlag|MAPQ,
    3 trailing NUL bytes of the QNAME, QC0 + k QNAME bytes [8 * (nq - 1 - k), +8) big-endian and zero padded, QC0 + nq the primary key"""
    u32 = lambda v: (v.astype(np.int64) & 0xffffffff).astype(np.uint64) ^ np.uint64(0x80000000)
    if chunk == 0:
        return u32(b.tlen)
    if chunk == 1:
        return np.where((b.flag & F_PAIRED) != 0, (u32(b.nref) << np.uint64(32)) | u32(b.pnext), np.uint64(0)).astype(np.uint64)
    if chunk == 2:
        return (mod_flag(b.flag) << np.uint64(8)) | b.mapq.astype(np.uint64)
    if chunk == 3:
        return trailing_nuls(b)
    if chunk < QC0 + nq:
        qc = nq - 1 - (chunk - QC0)
        off = b.qname_off.astype(np.int64)
        start = off[:-1] + 8 * qc
        avail = np.clip(off[1:] - start, 0, 8)
        j = np.arange(8)
        idx = np.minimum(start[:, None] + j, max(int(off[-1]) - 1, 0))
        byte = b.qname[idx].astype(np.uint64) if b.qname.size else np.zeros((b.n, 8), np.uint64)
        byte = np.where(j < avail[:, None], byte, np.uint64(0))
        return (byte << (np.uint64(56) - np.uint64(8) * j.astype(np.uint64))).sum(axis=1, dtype=np.uint64)
    assert chunk == QC0 + nq
    return primary_key(b, n_contigs, bP)


def long_run_elements(b, n_contigs, bP=None):
    """arrival indices of the reads in runs of more than SHORT_RUN equal primary keys"""
    key = primary_key(b, n_contigs, bP)
    order = np.argsort(key, kind="stable")
    ks = key[order]
    starts = np.flatnonzero(np.r_[True, ks[1:] != ks[:-1]])
    lens = np.diff(np.r_[starts, ks.size])
    return np.concatenate([order[s:s + n] for s, n in zip(starts, lens) if n > SHORT_RUN] or [np.zeros(0, np.int64)])


def tie_rounds(b, n_contigs, bP=None):
    """[(chunk, lo_bit, bits)] of the long-tie rounds: every chunk whose keys differ among the long-run reads, sorted over the bits from
    its lowest to its highest differing one"""
    elems = long_run_elements(b, n_contigs, bP)
    if elems.size == 0:
        return []
    nq = n_qname_chunks(b)
    sub = b.take(elems)
    out = []
    for ch in range(QC0 + nq + 1):
        col = chunk_keys(sub, ch, nq, n_contigs, pos_bits(b) if bP is None else bP)
        diff = int(np.bitwise_or.reduce(col)) ^ int(np.bitwise_and.reduce(col))
        if diff:
            lo = (diff & -diff).bit_length() - 1
            out.append((ch, lo, diff.bit_length() - lo))
    return out


def coordinate_sort_launches(b, n_contigs):
    """(tie_chunk_keys launches, u64 radix passes) of one coordinate sort without duplicate marking"""
    if b.n < 2:
        return 0, 0
    bP = pos_bits(b)
    rounds = tie_rounds(b, n_contigs, bP)
    return len(rounds), passes(1 + bP + n_contigs.bit_length()) + sum(passes(r[2]) for r in rounds)


def queryname_passes(b):
    """u64 radix passes of one queryname sort: the trailing-NUL pass, then eight per QNAME chunk"""
    if b.n < 2:
        return 0
    qmax = int(np.diff(b.qname_off.astype(np.int64)).max())
    return passes(qmax.bit_length()) + 8 * n_qname_chunks(b)
