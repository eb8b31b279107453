"""Restatement of ApplyBQSR's per-base rule (filters/bqsr.go:35-51, 64-146, 312-387, 901-1006), written from the Go source.

For every read: readGroupCovariate (panics on a read without RG, whatever its length), the combined-table existence test, the stranded
clipped sequence (QUAL <= 2 tails read as N; a byte comparison, so 0xFF is not a tail), contextWith with context size 2 (the N penalty, and
-1 for every IUPAC code and '='), prepareCycleCovariates / checkCycleCovariate (the 0x80 bit decides "last" whether or not 0x1 is set; the
check runs only for QUAL >= 6) and estimateHierarchicalBayesianQuality in the reference's order of operations, then math.Round, the clamp
to [1, 93], the quantization map and the static quantization map.

EmpiricalQuality, math.Round and the Go math functions come from the oracle library (orc_empirical_quality is pinned by
test_oracle_kat.py); the quantization maps too (orc_quantized, orc_static_quantized).  The new part is the key of every base and the
decision which bases change.

The result is the QUAL bytes the reference leaves and the error it stops with: None, "ENORG" (no read group), "ECYCLE" (cycle beyond
--max-cycle) or "ECONTEXT" (contextWith indexes bases[-1]: a non-N IUPAC code or '=' among the first two bases of the stranded clipped
sequence, unless the second one is N)."""
from __future__ import annotations

import ctypes as C

import numpy as np

from elprep_b200 import sam

MIN_INTERESTING_QUAL = 6       # bqsr.go minInterestingQual
LOW_QUALITY_TAIL = 2           # :301
MAX_RECAL_QUAL = 93            # maxRecalibratedQualScore

_BASE_INDEX = {"A": 0, "a": 0, "*": 0, "C": 1, "c": 1, "G": 2, "g": 2, "T": 3, "t": 3}     # :55
_COMPLEMENT = {"A": "T", "a": "T", "C": "G", "c": "G", "G": "C", "g": "C", "T": "A", "t": "A"}   # :303


class ContextPanic(Exception):
    """contextWith reads bases[-1] (index out of range)"""


def _lib():
    import oracle
    L = oracle.lib()
    L.orc_quantized.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]
    L.orc_static_quantized.argtypes = [C.c_void_p, C.c_int, C.c_void_p]
    return L


def _i32(x):
    x &= 0xFFFFFFFF
    return x - (1 << 32) if x & 0x80000000 else x


def read_group_covariate(header, rg):
    """:35-51: the PU of the first @RG whose ID matches, else the ID; None where the reference panics (no RG)"""
    if rg < 0:
        return None
    rid = header.RG[rg]["ID"]
    for rec in header.RG:
        if rec.get("ID") == rid:
            if "PU" in rec:
                return rec["PU"]
            break
    return rid


def stranded_clipped_seq(bases, qual, reversed_):
    """computeStrandedClippedSeq (:312-362); None for a read that is all tail"""
    L = len(bases)
    left = L
    for i in range(L):
        if qual[i] > LOW_QUALITY_TAIL:
            left = i
            break
    right = left - 1
    for i in range(L - 1, left - 1, -1):
        if qual[i] > LOW_QUALITY_TAIL:
            right = i
            break
    if left > right:
        return None
    if reversed_:
        return ["N"] * (L - 1 - right) + [_COMPLEMENT.get(bases[i], bases[i]) for i in range(right, left - 1, -1)] + ["N"] * left
    return ["N"] * left + list(bases[left:right + 1]) + ["N"] * (L - 1 - right)


def _key_from_context(dna, start, end):   # :64-76
    key, off = end - start, 4
    for i in range(start, end):
        b = _BASE_INDEX.get(dna[i], -1)
        if b == -1:
            return -1
        key |= b << off
        off += 2
    return key


def context_with(bases, context_size=2):
    """contextWith (:87-131), int32 arithmetic as in Go"""
    mask = 0
    for _ in range(context_size):
        mask = (mask << 2) | 3
    mask <<= 4
    n = len(bases)
    keys = [-1 for i in range(1, context_size) if i <= n]
    if n < context_size:
        return keys
    nbo = 2 * (context_size - 1) + 4
    cur = _key_from_context(bases, 0, context_size)
    keys.append(cur)
    pen = 0
    if cur == -1:
        cur, pen, off = 0, context_size - 1, nbo
        while True:
            if pen < 0:
                raise ContextPanic()
            if bases[pen] == "N":
                break
            cur = _i32(cur | (_BASE_INDEX.get(bases[pen], -1) << off))
            off -= 2
            pen -= 1
    for i in range(context_size, n):
        b = _BASE_INDEX.get(bases[i], -1)
        if b == -1:
            pen, cur = context_size, 0
        else:
            cur = _i32(((cur >> 2) & mask) | (b << nbo) | context_size)
        if pen == 0:
            keys.append(cur)
        else:
            pen -= 1
            keys.append(-1)
    return keys


def context_covariates(bases, qual, flag):
    """computeBaseContextCovariate (:140-146): one key per stored base (-1: none); raises ContextPanic"""
    s = stranded_clipped_seq(bases, qual, bool(flag & sam.Reversed))
    keys = context_with(s if s is not None else [])
    return keys[::-1] if flag & sam.Reversed else keys


def cycle_covariates(flag, L):
    """prepareCycleCovariates (:376-383): (cycleFactor, increment)"""
    rev, last = (flag & sam.Reversed) >> 4, (flag & sam.Last) >> 7
    rof = 1 - 2 * last
    return rof + rev * (L - 1) * rof, (1 - 2 * rev) * rof


class Tables:
    """the finalized tables of oracle.bqsr_gather / OracleTables plus what ApplyBQSR derives from them once (:938-943)"""

    def __init__(self, t, quantize_levels=0, sqq=None):
        L = _lib()
        self.t, self.L = t, L
        self.emp = L.orc_empirical_quality
        qmap, self.quant = np.zeros(94, np.int64), np.zeros(94, np.uint8)
        L.orc_quantized(C.cast(C.byref(t.s), C.c_void_p), int(quantize_levels), qmap.ctypes.data, self.quant.ctypes.data)
        self.stat = None
        if sqq is not None and len(sqq):
            s = np.ascontiguousarray(sqq, np.uint8)
            self.stat = np.zeros(254, np.uint8)
            L.orc_static_quantized(s.ctypes.data, int(s.size), self.stat.ctypes.data)
        self.comb = [self._combined(cv) for cv in range(t.n_cov)]
        self.memo = {}

    def _combined(self, cov):
        """initializeCombinedBQSRTable (:655-674), accumulated in ascending QUAL order"""
        L, t = self.L, self.t
        have, rep, o, m = False, 0.0, 0, 0
        for q in range(t.q_obs.shape[1]):
            eo, em = int(t.q_obs[cov, q]), int(t.q_mis[cov, q])
            if eo <= 0:
                continue
            if have:
                sum_err = float(o) * L.gm_pow(10.0, rep / -10) + float(eo) * L.gm_pow(10.0, float(q) / -10)
                o += eo
                m += em
                rep = -10 * L.gm_log10(sum_err / float(o))
            else:
                have, rep, o, m = True, float(q), eo, em
        return (rep, o, m) if have else None

    def estimate(self, cov, q, cyc, ctx):
        """estimateHierarchicalBayesianQuality (:901-919), epsilon = the read group's reported quality (globalQualityScorePrior < 0)"""
        t, emp = self.t, self.emp
        eps, go, gm = self.comb[cov]
        dG = float(emp(go, gm, eps)) - eps
        dQ = 0.0
        if q < t.q_obs.shape[1] and t.q_obs[cov, q] > 0:
            dQ = float(emp(int(t.q_obs[cov, q]), int(t.q_mis[cov, q]), dG + eps)) - dG - eps
        dC = 0.0
        cp = dQ + dG + eps
        ci = cyc + t.max_cycle
        if q < t.c_obs.shape[1] and t.c_obs[cov, q, ci] > 0:
            dC = float(emp(int(t.c_obs[cov, q, ci]), int(t.c_mis[cov, q, ci]), cp)) - cp
        if ctx >= 0 and q < t.x_obs.shape[1] and t.x_obs[cov, q, ctx >> 4] > 0:
            dC += float(emp(int(t.x_obs[cov, q, ctx >> 4]), int(t.x_mis[cov, q, ctx >> 4]), cp)) - cp
        return cp + dC

    def recalibrated(self, cov, q, cyc, ctx):
        k = (cov, q, cyc, ctx)
        v = self.memo.get(k)
        if v is None:
            r = max(1, min(int(self.L.gm_round(self.estimate(cov, q, cyc, ctx))), MAX_RECAL_QUAL))
            v = int(self.quant[r])
            if self.stat is not None:
                v = int(self.stat[v])
            self.memo[k] = v
        return v


def apply_read(T, cov_of, header, bases, qual, flag, rg, max_cycle):
    """one read through the closure of ApplyBQSR (:947-1003): (new QUAL list, error or None)"""
    name = read_group_covariate(header, rg)
    if name is None:
        return list(qual), "ENORG"
    cov = cov_of[name]
    if T.comb[cov] is None:
        return list(qual), None                       # no recalibration, bqsr table empty
    L = len(bases)
    cf, inc = cycle_covariates(flag, L)
    try:
        keys = context_covariates(bases, qual, flag)
    except ContextPanic:
        return list(qual), "ECONTEXT"
    out = list(qual)
    for i in range(L):
        q = qual[i]
        if q >= MIN_INTERESTING_QUAL:
            cyc = cf + i * inc
            if cyc > max_cycle or cyc < -max_cycle:
                return out, "ECYCLE"
            out[i] = T.recalibrated(cov, q, cyc, keys[i])
    return out, None


def bases_of(batch, i):
    so, L = int(batch.seq_off[i]), int(batch.lseq[i])
    return sam.decode_seq(batch.seq[so:so + (L + 1) // 2], L)


def apply(batch, header, t, quantize_levels=0, sqq=None, T=None):
    """-> (QUAL arena of ``batch`` after ApplyBQSR, first error in read order or None).  ``t``: finalized oracle tables (their max_cycle
    is --max-cycle)."""
    T = T or Tables(t, quantize_levels, sqq)
    _, cov_names = header.rg_cov_ids()
    cov_of = {n: k for k, n in enumerate(cov_names)}
    out = batch.qual.copy()
    qo = batch.qual_off.astype(np.int64)
    err = None
    for i in range(batch.n):
        q = [int(x) for x in batch.qual[qo[i]:qo[i + 1]]]
        new, e = apply_read(T, cov_of, header, bases_of(batch, i), q, int(batch.flag[i]), int(batch.rg[i]), t.max_cycle)
        out[qo[i]:qo[i + 1]] = new
        if e and err is None:
            err = e
    return out, err


def context_quirk(bases, qual, flag):
    """True where contextWith's start-of-read handling gives keys other than the plain 2-mer rule: it panics (a non-N IUPAC code or '='
    among the first two stranded bases, the second not N), or it leaves TT / T? keys (N, then such a code, then a base)."""
    s = stranded_clipped_seq(bases, qual, bool(flag & sam.Reversed))
    if s is None or len(s) < 2:
        return False
    try:
        keys = context_with(s)
    except ContextPanic:
        return True
    plain = [-1] + [(2 | (_BASE_INDEX[s[i - 1]] << 4) | (_BASE_INDEX[s[i]] << 6)) if s[i - 1] in _BASE_INDEX and s[i] in _BASE_INDEX else -1
                    for i in range(1, len(s))]
    return keys != plain
