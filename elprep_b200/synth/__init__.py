"""Synthetic paired-read workloads (SURVEY.md section 8d): bench / test input only, host side.

``make_workload`` returns the SAM header, one columnar ``AlignmentBatch`` in aligner-like order
(mates adjacent, pairs in random genome order), the reference genome (1 byte/base per contig) and
flattened known-sites intervals -- everything the hot path needs, with no file I/O.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

from .. import sam

_HERE = os.path.dirname(os.path.abspath(__file__))
_SO = os.path.join(_HERE, "libelprep_synth.so")

# hg38 primary assembly contig lengths chr1..chr22, X, Y, M (25 @SQ lines)
HG38 = [("chr1", 248956422), ("chr2", 242193529), ("chr3", 198295559), ("chr4", 190214555), ("chr5", 181538259),
        ("chr6", 170805979), ("chr7", 159345973), ("chr8", 145138636), ("chr9", 138394717), ("chr10", 133797422),
        ("chr11", 135086622), ("chr12", 133275309), ("chr13", 114364328), ("chr14", 107043718), ("chr15", 101991189),
        ("chr16", 90338345), ("chr17", 83257441), ("chr18", 80373285), ("chr19", 58617616), ("chr20", 64444167),
        ("chr21", 46709983), ("chr22", 50818468), ("chrX", 156040895), ("chrY", 57227415), ("chrM", 16569)]


def build(force=False):
    src = os.path.join(_HERE, "synth.cpp")
    if force or not os.path.exists(_SO) or os.path.getmtime(src) > os.path.getmtime(_SO):
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-pthread", "-o", _SO, src])
    return _SO


class _Params(C.Structure):
    _fields_ = [("seed", C.c_uint64), ("n_pairs", C.c_int64), ("n_contigs", C.c_int32), ("contig_len", C.c_void_p), ("L", C.c_int32),
                ("dup_frac", C.c_double), ("optical_frac", C.c_double), ("unmapped_frac", C.c_double), ("mate_unmapped_frac", C.c_double),
                ("secondary_frac", C.c_double), ("supplementary_frac", C.c_double), ("cross_contig_frac", C.c_double),
                ("n_rg", C.c_int32), ("wide_quals", C.c_int32), ("exome", C.c_int32), ("threads", C.c_int32),
                ("home", C.c_void_p), ("pair_id_base", C.c_uint64), ("genome_seed", C.c_uint64)]


_lib = None


def _L():
    global _lib
    if _lib is None:
        build()
        _lib = C.CDLL(_SO)
        _lib.synth_known_sites.restype = C.c_int64
    return _lib


def scaled_hg38(scale):
    """hg38-shaped contig table with every length divided by ``scale`` (chrM kept >= 16569/scale, min 4000)."""
    return [(n, max(4000, int(ln / scale))) for n, ln in HG38]


class Workload:
    def __init__(self, header, batch, contig_bases, sites, params):
        self.header, self.batch, self.contig_bases, self.sites, self.params = header, batch, contig_bases, sites, params


def make_header(contigs, n_rg=4):
    rg = []
    for i in range(n_rg):
        rg.append({"ID": f"rg{i + 1}", "PU": f"FC1.{i + 1}", "SM": "SYN", "PL": "ILLUMINA", "LB": "libA" if i < (n_rg + 1) // 2 else "libB"})
    return sam.Header(sq=[{"SN": n, "LN": int(ln)} for n, ln in contigs], rg=rg, so=sam.Unsorted)


def exome_regions(contigs, seed=20260924, pad=0):
    """The exons make_workload(..., exome=True) places its fragments around (synth.cpp: 300 bases every 15 kbp at a seeded offset), as
    per-contig (k, 2) int32 (start, end) arrays widened by ``pad`` on both sides -- a target-regions BED for that workload."""
    def mix(z):
        M = (1 << 64) - 1
        z = (z + 0x9E3779B97F4A7C15) & M
        z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) & M
        z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) & M
        return z ^ (z >> 31)
    out = []
    for c, (_, ln) in enumerate(contigs):
        starts = [1000 + ex * 15000 + mix(int(seed) ^ (c << 32) ^ ex) % 5000 for ex in range(max(1, int(ln) // 15000))]
        out.append(np.array([(s - pad, s + 300 + pad) for s in starts], dtype=np.int32).reshape(-1, 2))
    return out


def make_workload(n_pairs, contigs, seed=20260924, L=150, dup_frac=0.10, optical_frac=0.20, unmapped_frac=0.01,
                  mate_unmapped_frac=0.005, secondary_frac=0.005, supplementary_frac=0.005, cross_contig_frac=0.01,
                  n_rg=4, wide_quals=False, exome=False, threads=None, want_reference=True, home=None, pair_id_base=0, genome_seed=None, reference_for=None):
    """home: bool per contig -- fragments start only on those contigs (one generator per contig group of ONE genome: the mates of its
    cross-contig pairs land on any contig, so pairs span the groups as in a real `elprep sfm` split); pair_id_base keeps QNAMEs unique across
    the generators; genome_seed: the shared reference genome; reference_for: contig indices whose reference / known sites are returned."""
    if not 20 <= L <= 8000:
        raise ValueError("read length outside the generator's range (20..8000)")
    lib = _L()
    threads = threads or min(32, os.cpu_count() or 1)
    clen = np.array([ln for _, ln in contigs], dtype=np.int32)
    home_a = np.ascontiguousarray(home, dtype=np.uint8) if home is not None else None
    gseed = int(genome_seed) if genome_seed is not None else int(seed)
    p = _Params(seed, n_pairs, len(contigs), clen.ctypes.data_as(C.c_void_p), L, dup_frac, optical_frac, unmapped_frac,
                mate_unmapped_frac, secondary_frac, supplementary_frac, cross_contig_frac, n_rg, int(wide_quals), int(exome), threads,
                home_a.ctypes.data_as(C.c_void_p) if home_a is not None else None, int(pair_id_base), gseed)
    rec0 = np.zeros(n_pairs + 1, dtype=np.int64)
    cig0 = np.zeros(n_pairs + 1, dtype=np.uint64)
    qn0 = np.zeros(n_pairs + 1, dtype=np.uint64)
    vp = lambda a: a.ctypes.data_as(C.c_void_p)
    lib.synth_sizes(C.byref(p), vp(rec0), vp(cig0), vp(qn0))
    n = int(rec0[-1])
    a = dict(refid=np.empty(n, np.int32), pos=np.empty(n, np.int32), flag=np.empty(n, np.uint16), mapq=np.empty(n, np.uint8),
             nref=np.empty(n, np.int32), pnext=np.empty(n, np.int32), tlen=np.empty(n, np.int32), rg=np.empty(n, np.int32),
             qname_off=np.empty(n + 1, np.uint64), qname=np.empty(int(qn0[-1]), np.uint8), cigar_off=np.empty(n + 1, np.uint64),
             cigar=np.empty(max(1, int(cig0[-1])), np.uint32), lseq=np.empty(n, np.int32), seq=np.empty(n * ((L + 1) // 2), np.uint8),
             qual=np.empty(n * L, np.uint8))
    lib.synth_fill(C.byref(p), vp(rec0), vp(cig0), vp(qn0), *[vp(a[k]) for k in
                   ("refid", "pos", "flag", "mapq", "nref", "pnext", "tlen", "rg", "qname_off", "qname", "cigar_off", "cigar", "lseq", "seq", "qual")])
    a["cigar"] = a["cigar"][:int(cig0[-1])]
    batch = sam.AlignmentBatch(**a)
    header = make_header(contigs, n_rg)
    bases, sites = None, None
    if want_reference:
        bases, sites = [], []
        want = set(range(len(contigs))) if reference_for is None else set(reference_for)
        for ci, (_, ln) in enumerate(contigs):
            if ci not in want:
                bases.append(None); sites.append(np.zeros((0, 2), np.int32)); continue
            b = np.empty(ln, dtype=np.uint8)
            lib.synth_genome(C.c_uint64(gseed), C.c_int32(ci), C.c_int64(0), C.c_int64(ln), vp(b), C.c_int32(threads))
            bases.append(b)
            cap = ln // 1000 + 2
            se = np.zeros(2 * cap, dtype=np.int32)
            k = lib.synth_known_sites(C.c_uint64(gseed), C.c_int32(ci), C.c_int32(ln), vp(se), C.c_int64(cap))
            sites.append(se[:2 * k].reshape(-1, 2).copy())
    return Workload(header, batch, bases, sites, dict(n_pairs=n_pairs, seed=seed, L=L, contigs=contigs))


def encode_bam(batch, header, threads=8):
    """columns -> (uint8 BAM alignment records, uint64 record offsets [n+1]); test / bench infrastructure for elp_append_bam"""
    L = _L()
    ids = [r["ID"].encode() for r in header.RG]
    rg_ids = np.frombuffer(b"".join(ids) or b"\0", dtype=np.uint8).copy()
    rg_off = np.zeros(len(ids) + 1, dtype=np.uint32)
    if ids:
        rg_off[1:] = np.cumsum([len(x) for x in ids])
    n = batch.n
    rec_off = np.zeros(n + 1, dtype=np.uint64)
    cols = [batch.refid, batch.pos, batch.flag, batch.mapq, batch.nref, batch.pnext, batch.tlen, batch.rg, batch.qname_off, batch.qname, batch.cigar_off,
            batch.cigar, batch.lseq, batch.seq_off, batch.seq, batch.qual_off, batch.qual, rg_ids, rg_off]
    ptr = [a.ctypes.data_as(C.c_void_p) for a in cols]
    L.synth_encode_bam(C.c_int64(n), *ptr, rec_off.ctypes.data_as(C.c_void_p), None, C.c_int32(threads))
    out = np.empty(int(rec_off[-1]), dtype=np.uint8)
    L.synth_encode_bam(C.c_int64(n), *ptr, rec_off.ctypes.data_as(C.c_void_p), out.ctypes.data_as(C.c_void_p), C.c_int32(threads))
    return out, rec_off


def take(batch, idx, threads=None):
    """``batch.take(idx)`` with the ragged gathers done by host threads (no element-wise index arrays): what the bench's
    verification and the C1/C2-sized parity tests use to materialise the oracle's output order."""
    lib = _L()
    threads = threads or min(32, os.cpu_count() or 1)
    idx = np.ascontiguousarray(idx, dtype=np.int64)
    n = idx.shape[0]
    vp = lambda a: a.ctypes.data_as(C.c_void_p)

    def ragged(off, data):
        off = np.ascontiguousarray(off, dtype=np.uint64)
        lens = (off[1:] - off[:-1])[idx]
        no = np.zeros(n + 1, dtype=np.uint64)
        np.cumsum(lens, out=no[1:])
        out = np.empty(int(no[-1]), dtype=data.dtype)
        if n:
            lib.synth_take_ragged(vp(idx), C.c_int64(n), vp(off), vp(data), C.c_int32(data.dtype.itemsize), vp(no), vp(out), C.c_int32(threads))
        return no, out
    qo, qn = ragged(batch.qname_off, batch.qname)
    co, cg = ragged(batch.cigar_off, batch.cigar)
    _, sq = ragged(batch.seq_off, batch.seq)
    _, ql = ragged(batch.qual_off, batch.qual)
    return sam.AlignmentBatch(refid=batch.refid[idx], pos=batch.pos[idx], flag=batch.flag[idx], mapq=batch.mapq[idx], nref=batch.nref[idx],
                              pnext=batch.pnext[idx], tlen=batch.tlen[idx], rg=batch.rg[idx], qname_off=qo, qname=qn, cigar_off=co, cigar=cg,
                              lseq=batch.lseq[idx], seq=sq, qual=ql, opt_flags=batch.opt_flags[idx])
