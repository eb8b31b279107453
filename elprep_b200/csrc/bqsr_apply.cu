// bqsr_apply.cu -- recalibrated QUAL bytes (replaces the per-read closure of ApplyBQSR, filters/bqsr.go:947-1003).
//
// Every base with QUAL >= 6 is replaced by LUT[read-group covariate][QUAL][cycle][context] -- the byte table
// bqsr_finalize.cu builds from the hierarchical Bayesian estimate (the reference memoises the same function per worker,
// :973-1000).  The result is written as a contiguous QUAL stream in output order (what elp_fetch copies back); the
// original QUAL arena stays untouched.
//
// Kernel shape (same decomposition as the gather's chunk kernel, bqsr_gather.cu): a lane owns 16 consecutive bases of a
// read, a warp takes 32 / lanes_per_read reads.
//   1. 16 QUAL bytes and 16 SEQ nibbles come out of aligned 128-bit loads (funnel-shifted to the read's byte offset);
//      base codes, the 2-mer context of every base and the low-quality tails (computeStrandedClippedSeq, bqsr.go:312-331)
//      are computed word-parallel; the tails are reduced across the lanes of the read with member-mask reductions;
//   2. per base: one byte load from the LUT (L1/L2 resident) and a byte insert; cycle advances by +-1, LUT address by +-17;
//   3. the lanes park their 16 result bytes in shared memory and the read's strip is written as 16-byte stores aligned
//      on the OUTPUT stream (funnel-shifted out of shared memory); only the partial chunks at the ends use byte stores.
// With lut == nullptr the kernel only materialises the output-order QUAL stream (no BQSR requested).
#include "ctx.h"
#include "bqsr_simd.cuh"
#include "bqsr_lane.cuh"
#include <algorithm>
#include <cstdlib>
#include <string>

namespace {

constexpr int WARPS = 8;

// nibble flags for chunk index >= k and <= k - 1 (filled by run_apply_kernel)
__constant__ unsigned long long c_ge[CHUNK + 1], c_le[CHUNK + 1];
__device__ __forceinline__ unsigned long long range16(int lo, int hi) { return c_ge[min(max(lo, 0), CHUNK)] & c_le[min(max(hi + 1, 0), CHUNK)]; }

struct ApplyArgs {
    uint64_t n;
    const uint16_t* flag; const int32_t *rg, *lseq; const uint64_t *qual_off, *seq_off, *out_off;
    const uint8_t *seq, *qual; uint8_t* out;
    const int32_t* rg_cov; int n_rg; const uint8_t* cov_exists;
    const uint8_t* lut; int lut_maxcyc, max_cycle;
    int lanes_per_read;
    uint32_t* err;
};

#ifndef APPLY_MINB
#define APPLY_MINB 8
#endif
__global__ void __launch_bounds__(WARPS * 32, APPLY_MINB) bqsr_apply_kernel(ApplyArgs A) {
    // image of the block's slice of the output stream, placed with the slice's 16-byte phase: the reads of a block are
    // consecutive in output order, so the whole slice leaves as aligned 128-bit stores (two partial chunks per BLOCK)
    __shared__ __align__(16) uint8_t sm_img[WARPS * 32 * CHUNK + 32];
    const unsigned lane = lane_id(), w = threadIdx.x >> 5;
    const int lpr = A.lanes_per_read, rpw = 32 / lpr;
    const int r = (int)lane / lpr, c = (int)lane - r * lpr;
    const bool lane_used = r < rpw;
    const uint64_t k = ((uint64_t)blockIdx.x * WARPS + w) * (uint64_t)rpw + (uint64_t)r;
    const bool valid = lane_used && k < A.n;
    int L = valid ? A.lseq[k] : 0;
    uint32_t errbits = 0;
    if (L > CHUNK * lpr) { errbits |= DERR_READLEN_LIMIT; L = 0; }
    const uint64_t qoff = valid ? A.qual_off[k] : 0, ooff = valid ? A.out_off[k] : 0;
    const uint64_t kb0 = (uint64_t)blockIdx.x * WARPS * (uint64_t)rpw, kb1 = min(A.n, kb0 + (uint64_t)(WARPS * rpw));
    const uint64_t o0 = A.out_off[kb0], o1 = A.out_off[kb1];               // the block's slice [o0, o1) of the output stream
    const uint32_t phase = (uint32_t)(o0 & 15);
    bool recal = valid && A.lut != nullptr && L > 0;
    int cov = 0;
    if (recal) {
        const int g = A.rg[k];
        if (g < 0 || g >= A.n_rg) { errbits |= DERR_NORG; recal = false; }                 // readGroupCovariate panics, bqsr.go:38
        else { cov = A.rg_cov[g]; if (!A.cov_exists[cov]) recal = false; }                  // no recalibration, bqsr table empty (:950-953)
    }
    const int i0 = c * CHUNK, nb = min(max(L - i0, 0), CHUNK);
    // ---- 1. loads and word-parallel covariates ----
    uint32_t Q[4] = {0, 0, 0, 0};
    unsigned long long C = 0;
    if (nb > 0) {
        load16_unaligned(A.qual + qoff + (uint64_t)i0, Q);
        if (A.lut != nullptr) {   // (not `recal`: the read-group look-ups above overlap with these loads)
            const unsigned long long nibs = load16_nibbles_bam(A.seq, A.seq_off[k] * 2 + (uint64_t)i0);
            C = (unsigned long long)codes_of((uint32_t)nibs) | ((unsigned long long)codes_of((uint32_t)(nibs >> 32)) << 32);
        }
    }
    if (nb < CHUNK) { const unsigned long long inlen = range16(0, nb - 1); C = (C & (inlen * 15ull)) | ((ONES & ~inlen) << 3); }   // codes past the read end: 8
    int first, last;
    qual_gt2_span(Q, nb, i0, first, last);
    const unsigned gmask = lane_used ? ((lpr == 32 ? 0xffffffffu : ((1u << lpr) - 1u)) << (r * lpr)) : (1u << lane);
    const int leftPos = __reduce_min_sync(gmask, first), rightPos = __reduce_max_sync(gmask, last);
    const uint32_t c_hi = (uint32_t)(C >> 32), c_lo = (uint32_t)C;
    uint32_t edge_prev = __shfl_up_sync(FULL_MASK, c_hi, 1) >> 28, edge_next = __shfl_down_sync(FULL_MASK, c_lo, 1) & 15u;
    if (c == 0) edge_prev = 8;
    if (c == lpr - 1 || lane == 31) edge_next = 8;
    // ---- 2. LUT lookups ----
    if (recal && nb > 0) {
        const uint16_t f = A.flag[k];
        const bool rev = f & F_REVERSED;
        const int lastf = (f & F_LAST) ? 1 : 0;
        const int rof = 1 - 2 * lastf, inc = rev ? -rof : rof, cf = rof + (rev ? (L - 1) * rof : 0);   // prepareCycleCovariates, bqsr.go:376-383 (full read length)
        const unsigned long long Pn = rev ? ((C >> 4) | ((unsigned long long)edge_next << 60)) : ((C << 4) | edge_prev);
        const unsigned long long M3 = 0x3333333333333333ull, xr = rev ? M3 : 0ull;
        const unsigned long long ctxw = ((Pn ^ xr) & M3) | (((C ^ xr) & M3) << 2);          // key>>4 = prev | cur<<2, complemented for reverse reads
        const int wlo = rev ? leftPos : leftPos + 1, whi = rev ? rightPos - 1 : rightPos;      // low-quality tails read as N
        const unsigned long long okc = ~((Pn | C) >> 3) & ONES & range16(wlo - i0, whi - i0);
        const uint32_t ncyc17 = (2u * (uint32_t)A.lut_maxcyc + 1u) * 17u;
        const uint8_t* lut_cov = A.lut + (size_t)cov * 94u * ncyc17;
        const uint32_t okc_w[2] = {(uint32_t)okc, (uint32_t)(okc >> 32)}, ctx_w[2] = {(uint32_t)ctxw, (uint32_t)(ctxw >> 32)};
        const int cyc_a = cf + i0 * inc, cyc_b = cyc_a + (nb - 1) * inc;                    // cycles of the chunk's first / last base
        // bytes past the read end must not look like bases (they belong to the next read of the arena and are never written back)
#pragma unroll
        for (int wq = 0; wq < 4; wq++) { const int keep = nb - 4 * wq; if (keep < 4) Q[wq] = keep <= 0 ? 0u : (Q[wq] & (0xffffffffu >> (8 * (4 - keep)))); }
        if (max(cyc_a, cyc_b) > A.max_cycle || min(cyc_a, cyc_b) < -A.max_cycle) {
            // checkCycleCovariate (:364-369) fails somewhere in this chunk: an error if one of those bases is recalibrated
            int cyc = cyc_a;
#pragma unroll
            for (int j = 0; j < CHUNK; j++) {
                const uint32_t q = (Q[j >> 2] >> (8 * (j & 3))) & 0xffu;
                if (q >= 6) errbits |= q > 93 ? DERR_QUAL_RANGE : ((cyc > A.max_cycle || cyc < -A.max_cycle) ? DERR_CYCLE : 0u);
                cyc += inc;
            }
        } else {
            uint32_t idx = (uint32_t)(cyc_a + A.lut_maxcyc) * 17u;
            const uint32_t step = (uint32_t)(inc * 17);
            uint32_t over = 0;
#pragma unroll
            for (int j = 0; j < CHUNK; j++) {
                const uint32_t q = (Q[j >> 2] >> (8 * (j & 3))) & 0xffu;
                const uint32_t nib = (ctx_w[j >> 3] >> (4 * (j & 7))) & 15u;
                const uint32_t ctx = ((okc_w[j >> 3] >> (4 * (j & 7))) & 1u) ? nib : 16u;   // 16 = no context (key -1)
                over |= q;
                if (q - 6u <= 87u) {                                                        // minInterestingQual <= q <= 93
                    const uint32_t v = __ldg(lut_cov + q * ncyc17 + idx + ctx);
                    Q[j >> 2] = __byte_perm(Q[j >> 2], v, (j & 3) == 0 ? 0x3214 : ((j & 3) == 1 ? 0x3240 : ((j & 3) == 2 ? 0x3410 : 0x4210)));
                }
                idx += step;
            }
            // a QUAL above 93 (any byte with bit 7, or 94..127) is an error for a recalibrated base
            if (over & 0x80u) errbits |= DERR_QUAL_RANGE;
            else if (over >= 94u) {
#pragma unroll
                for (int wq = 0; wq < 4; wq++) { const uint32_t v = Q[wq]; if ((((v & 0x7f7f7f7fu) + 0x22222222u) | v) & 0x80808080u) errbits |= DERR_QUAL_RANGE; }
            }
        }
    }
    // ---- 3. park the chunk in the block image, then write the image in 16-byte chunks aligned on the output stream ----
    if (nb > 0) {
        uint8_t* dst = sm_img + phase + (uint32_t)(ooff - o0) + (uint32_t)i0;
#pragma unroll
        for (int j = 0; j < CHUNK; j++) if (j < nb) dst[j] = (uint8_t)(Q[j >> 2] >> (8 * (j & 3)));
    }
    __syncthreads();
    {
        const uint32_t total = (uint32_t)(o1 - o0), end = phase + total;           // image bytes [phase, end)
        uint8_t* gbase = A.out + (o0 - phase);                                      // 16-byte aligned
        for (uint32_t m = threadIdx.x; m * 16u < end; m += blockDim.x) {
            const uint32_t b0 = m * 16u;
            if (b0 >= phase && b0 + 16u <= end) *reinterpret_cast<uint4*>(gbase + b0) = *reinterpret_cast<const uint4*>(sm_img + b0);
            else { const uint32_t lo = max(b0, phase), hi = min(b0 + 16u, end); for (uint32_t t = lo; t < hi; t++) gbase[t] = sm_img[t]; }   // shared with a neighbouring block
        }
    }
    for (int o = 16; o; o >>= 1) errbits |= __shfl_xor_sync(FULL_MASK, errbits, o);
    if (errbits && lane == 0) atomicOr(A.err, errbits);
}


// ---------------------------------------------------------------- apply, second generation
// Same per-base rule as bqsr_apply_kernel above, organised like the count kernel (bqsr_count.inl): a lane owns 32 consecutive bases of a
// read (stored order), QUAL / SEQ arrive as aligned 16-byte loads and are re-aligned in registers (bqsr_lane.cuh), the 2-mer contexts of all
// 32 bases are computed word-parallel, and the look-up table -- compacted to the QUAL values that occur (bqsr_finalize.cu) -- lives in
// SHARED memory, laid out [cycle][covariate][slot][17] with an odd block stride so that the lanes of a read (32 cycles apart) start in
// different banks.  Per base: one byte extract, one table-row look-up, one context extract, one table byte, one byte insert.
// Bases without a context (first base of the read, neighbours of N, low-quality tails) are rare and patched afterwards.
constexpr int AP2_WARPS = 16;
struct Apply2Args {
    uint64_t n;
    const uint16_t* flag; const int32_t *rg, *lseq; const uint64_t *qual_off, *seq_off, *out_off;
    const uint8_t *seq, *qual; uint8_t* out;
    const int32_t* rg_cov; int n_rg; const uint8_t* cov_exists;
    const uint8_t* clut; uint32_t clut_bytes, blk, Lc;     // compact table [2 Lc + 1 + 64 margin cycles][blk]; blk = n_cov * S * 17 rounded up to odd
    const uint16_t* rowtab;                                // [256] byte offset of the slot of a QUAL value inside a covariate's part of a block (0xffff: none)
    uint32_t S17;                                          // S * 17: bytes of one covariate inside a block
    int lpr, rpw;
    uint32_t* err;
};

__global__ void __launch_bounds__(AP2_WARPS * 32, 2) bqsr_apply2_kernel(Apply2Args A) {
    extern __shared__ __align__(16) unsigned char ap_smem[];
    __shared__ uint16_t s_rowtab[256];
    const unsigned lane = lane_id(), warp = threadIdx.x >> 5;
    // shared memory: [table | per-warp output image]
    const uint32_t lut_s = (uint32_t)__cvta_generic_to_shared(ap_smem);
    const uint32_t img_bytes = (uint32_t)(A.rpw * A.lpr * 32 + 32);
    unsigned char* img = ap_smem + ((A.clut_bytes + 15u) & ~15u) + warp * img_bytes;
    const uint32_t img_s = (uint32_t)__cvta_generic_to_shared(img);
    for (uint32_t i = threadIdx.x * 16; i < A.clut_bytes; i += blockDim.x * 16) *reinterpret_cast<uint4*>(ap_smem + i) = __ldg(reinterpret_cast<const uint4*>(A.clut + i));
    for (int i = threadIdx.x; i < 256; i += blockDim.x) s_rowtab[i] = A.rowtab[i];
    __syncthreads();
    const uint32_t rowtab_s = (uint32_t)__cvta_generic_to_shared(s_rowtab);
    const int lpr = A.lpr, rpw = A.rpw;
    const int r = (int)lane / lpr, c = (int)lane - r * lpr;
    const bool lane_used = r < rpw;
    const unsigned gmask = lane_used ? ((lpr == 32 ? 0xffffffffu : ((1u << lpr) - 1u)) << (r * lpr)) : (1u << lane);
    const uint64_t n_pass = (A.n + rpw - 1) / rpw;
    const uint64_t gw = (uint64_t)blockIdx.x * AP2_WARPS + warp, nw = (uint64_t)gridDim.x * AP2_WARPS;
    uint32_t errbits = 0;
    // metadata of the next pass is fetched one pass ahead
    auto meta = [&](uint64_t p, int& L, uint64_t& qoff, uint64_t& soff, uint64_t& ooff, uint32_t& fg) {
        const uint64_t k = p * rpw + (uint64_t)r;
        L = 0; qoff = 0; soff = 0; ooff = 0; fg = 0;
        if (lane_used && p < n_pass && k < A.n) { L = A.lseq[k]; qoff = A.qual_off[k]; soff = A.seq_off[k]; ooff = A.out_off[k]; fg = (uint32_t)A.flag[k] | ((uint32_t)(A.rg[k] + 1) << 16); }
    };
    int Ln; uint64_t qn, sn, on; uint32_t fn;
    meta(gw, Ln, qn, sn, on, fn);
    for (uint64_t p = gw; p < n_pass; p += nw) {
        const int L = Ln; const uint64_t qoff = qn, soff = sn, ooff = on; const uint32_t fg = fn;
        meta(p + nw, Ln, qn, sn, on, fn);
        const uint64_t k0 = p * rpw, k1 = min(A.n, k0 + (uint64_t)rpw);
        const uint64_t o0 = A.out_off[k0], o1 = A.out_off[k1];
        const uint32_t phase = (uint32_t)(o0 & 15);
        if (L > 32 * lpr) { errbits |= DERR_READLEN_LIMIT; }
        const int nb = L > 32 * lpr ? 0 : min(max(L - 32 * c, 0), 32);
        const int i0 = 32 * c;
        // ---- windows ----
        uint32_t Q[8], N[4];
        {
            uint32_t W[12];
            const uint8_t* qp = A.qual + qoff + i0;
            const uint4* q16 = reinterpret_cast<const uint4*>(reinterpret_cast<uintptr_t>(qp) & ~(uintptr_t)15);
            uint4 a0 = make_uint4(0, 0, 0, 0), a1 = a0, a2 = a0;
            if (nb > 0) { a0 = ld_stream_u4(q16); a1 = ld_stream_u4(q16 + 1); a2 = ld_stream_u4(q16 + 2); }
            W[0] = a0.x; W[1] = a0.y; W[2] = a0.z; W[3] = a0.w; W[4] = a1.x; W[5] = a1.y; W[6] = a1.z; W[7] = a1.w; W[8] = a2.x; W[9] = a2.y; W[10] = a2.z; W[11] = a2.w;
            lanes::align_bytes32(W, (uint32_t)(reinterpret_cast<uintptr_t>(qp) & 15), Q);
            uint32_t V[8];
            const uint64_t ni = soff * 2 + (uint64_t)i0;
            const uint8_t* sp = A.seq + (ni >> 1);
            const uint4* s16 = reinterpret_cast<const uint4*>(reinterpret_cast<uintptr_t>(sp) & ~(uintptr_t)15);
            uint4 b0 = make_uint4(0, 0, 0, 0), b1 = b0;
            if (nb > 0 && A.clut) { b0 = ld_stream_u4(s16); b1 = ld_stream_u4(s16 + 1); }
            V[0] = b0.x; V[1] = b0.y; V[2] = b0.z; V[3] = b0.w; V[4] = b1.x; V[5] = b1.y; V[6] = b1.z; V[7] = b1.w;
            lanes::align_nibbles32<true>(V, (uint32_t)(reinterpret_cast<uintptr_t>(sp) & 15), (uint32_t)(ni & 1), N);
        }
        // (bytes past the read end are whatever follows in the arena: they index valid table rows, are never stored, and are masked where it
        //  matters -- the tail search below and the range check in its slow path)
        const uint32_t f = fg & 0xffffu; const int g = (int)(fg >> 16) - 1;
        bool recal = A.clut != nullptr && nb > 0;
        int cov = 0;
        if (recal) {
            if (g < 0 || g >= A.n_rg) { errbits |= DERR_NORG; recal = false; }                 // readGroupCovariate panics, bqsr.go:38
            else { cov = A.rg_cov[g]; if (!A.cov_exists[cov]) recal = false; }                  // no recalibration, bqsr table empty (:950-953)
        }
        const bool rev = (f & F_REVERSED) != 0;
        // ---- word-parallel covariates (stored order; nibble k of word w <-> base 8 w + k) ----
        const uint32_t M1 = 0x11111111u;
        uint32_t C[4], Vd[4];      // 2-bit base codes (A C G T -> 0..3), valid flags (bit 0 of the nibble)
#pragma unroll
        for (int w = 0; w < 4; w++) {
            const uint32_t v = N[w];
            C[w] = (((v >> 1) & 0x77777777u) - ((v >> 3) & M1)) & 0x33333333u;
            uint32_t pc = v - ((v >> 1) & 0x55555555u); pc = (pc & 0x33333333u) + ((pc >> 2) & 0x33333333u);     // bits set per nibble
            const uint32_t t = pc ^ M1;                                                                           // zero iff exactly one
            Vd[w] = ~(t | (t >> 1) | (t >> 2)) & M1;
        }
        uint32_t inl[4];   // bases inside the read
        {
            const int full = nb >> 3, part = nb & 7;
#pragma unroll
            for (int w = 0; w < 4; w++) { inl[w] = w < full ? M1 : (w == full ? (M1 & ((1u << (4 * part)) - 1u)) : 0u); Vd[w] &= inl[w]; }
        }
        // low-quality tails (computeStrandedClippedSeq, bqsr.go:312-331): only when the read starts or ends with QUAL <= 2
        const bool is_last_lane = L > 0 && (L - 1) >= i0 && (L - 1) < i0 + 32;
        const uint32_t qfirst = Q[0] & 0xffu;
        uint32_t qlast = 0;
        if (is_last_lane) { const int jl = L - 1 - i0; qlast = (Q[jl >> 2] >> (8 * (jl & 3))) & 0xffu; }        // (dynamic word index: eight-way select, once per pass)
        const bool tail_here = recal && ((c == 0 && qfirst <= 2) || (is_last_lane && qlast <= 2));
        if (__any_sync(FULL_MASK, tail_here)) {
            uint32_t G = 0;
#pragma unroll
            for (int w = 0; w < 8; w++) { const uint32_t x = Q[w]; const uint32_t gt2 = (((x & 0x7f7f7f7fu) + 0x7d7d7d7du) | x) & 0x80808080u; G |= ((gt2 * 0x00204081u) >> 28) << (4 * w); }
            if (nb < 32) G &= nb > 0 ? ((1u << nb) - 1u) : 0u;
            const unsigned gb = __ballot_sync(FULL_MASK, G != 0) & gmask;
            const int lo_lane = gb ? __ffs((int)gb) - 1 : (int)lane, hi_lane = gb ? 31 - __clz((int)gb) : (int)lane;
            const int lf = G ? i0 + (__ffs((int)G) - 1) : 0x7fffffff, ll = G ? i0 + (31 - __clz((int)G)) : -1;
            const int lf_x = __shfl_sync(FULL_MASK, lf, lo_lane), ll_x = __shfl_sync(FULL_MASK, ll, hi_lane);    // (every lane takes part: groups without a set bit differ)
            const int leftPos = gb ? lf_x : 0x7fffffff, rightPos = gb ? ll_x : -1;
            // bases outside [leftPos, rightPos] read as N
#pragma unroll
            for (int w = 0; w < 4; w++) {
                const int lo = min(max(leftPos - i0 - 8 * w, 0), 8), hi = min(max(rightPos + 1 - i0 - 8 * w, 0), 8);     // nibbles [lo, hi) stay
                const uint32_t keep = hi > lo ? ((hi >= 8 ? 0xffffffffu : ((1u << (4 * hi)) - 1u)) & ~((1u << (4 * lo)) - 1u)) : 0u;
                Vd[w] &= keep;
            }
        }
        // previous base in sequencing direction: stored base j - 1 (forward) / j + 1 (reverse), across lanes at the word ends
        const uint32_t up_c = __shfl_up_sync(FULL_MASK, C[3], 1), up_v = __shfl_up_sync(FULL_MASK, Vd[3], 1);
        const uint32_t dn_c = __shfl_down_sync(FULL_MASK, C[0], 1), dn_v = __shfl_down_sync(FULL_MASK, Vd[0], 1);
        const uint32_t pc_in = c == 0 ? 0u : up_c, pv_in = c == 0 ? 0u : up_v, nc_in = (c == lpr - 1 || lane == 31) ? 0u : dn_c, nv_in = (c == lpr - 1 || lane == 31) ? 0u : dn_v;
        uint32_t X[4], NOK[4];     // context nibbles (prev | cur << 2, complemented for reverse reads, bqsr.go:64-76); "base has no context" flags
        const uint32_t cm = rev ? 0x33333333u : 0u;
#pragma unroll
        for (int w = 0; w < 4; w++) {
            const uint32_t pf = (C[w] << 4) | ((w ? C[w - 1] : pc_in) >> 28), pr = (C[w] >> 4) | ((w < 3 ? C[w + 1] : nc_in) << 28);
            const uint32_t vf = (Vd[w] << 4) | ((w ? Vd[w - 1] : pv_in) >> 28), vr = (Vd[w] >> 4) | ((w < 3 ? Vd[w + 1] : nv_in) << 28);
            const uint32_t P = rev ? pr : pf, PV = rev ? vr : vf;
            X[w] = ((P ^ cm) & 0x33333333u) | (((C[w] ^ cm) & 0x33333333u) << 2);
            NOK[w] = ~(Vd[w] & PV) & inl[w];
        }
        // ---- table look-ups ----
        uint32_t R[8];
#pragma unroll
        for (int w = 0; w < 8; w++) R[w] = Q[w];
        if (recal) {
            const int sign = (f & F_LAST) ? -1 : 1;
            const int step = rev ? -sign : sign;
            const int cyc0 = sign * (rev ? L - i0 : i0 + 1);                                       // cycle of stored base i0 (bqsr.go:376-387)
            if (L > (int)A.Lc) errbits |= DERR_CYCLE;                                             // (the host only selects this kernel when every cycle fits)
            const uint32_t cbase = lut_s + (uint32_t)(cyc0 + (int)A.Lc + 32) * A.blk + (uint32_t)cov * A.S17;
            const int stepb = step * (int)A.blk;
            uint32_t over = 0;
#pragma unroll
            for (int j = 0; j < 32; j++) {
                const uint32_t q = (Q[j >> 2] >> (8 * (j & 3))) & 0xffu;
                uint32_t row; asm volatile("ld.shared.u16 %0, [%1];" : "=r"(row) : "r"(rowtab_s + 2u * q));
                const uint32_t ctx = (X[j >> 3] >> (4 * (j & 7))) & 15u;
                uint32_t v; asm volatile("ld.shared.u8 %0, [%1];" : "=r"(v) : "r"(cbase + (uint32_t)(j * stepb) + (row & 0x7fffu) + ctx));
                R[j >> 2] = __byte_perm(R[j >> 2], v, (j & 3) == 0 ? 0x3214 : ((j & 3) == 1 ? 0x3240 : ((j & 3) == 2 ? 0x3410 : 0x4210)));
            }
            // QUAL > 93 is an error (bqsr.go:968 indexes a 94-entry table): any byte >= 64 sends the lane through the exact, masked check
#pragma unroll
            for (int w = 0; w < 8; w++) over |= Q[w];
            if (over & 0xc0c0c0c0u) {
#pragma unroll
                for (int w = 0; w < 8; w++) {
                    const int keep = nb - 4 * w;
                    const uint32_t v = keep >= 4 ? Q[w] : (keep <= 0 ? 0u : (Q[w] & (0xffffffffu >> (8 * (4 - keep)))));
                    if ((((v & 0x7f7f7f7fu) + 0x22222222u) | v) & 0x80808080u) errbits |= DERR_QUAL_RANGE;
                }
            }
            // bases without a context take column 16
#pragma unroll
            for (int i = 0; i < 8; i++) {
                uint32_t m = (NOK[i >> 1] >> (16 * (i & 1))) & 0x1111u;
                while (m) {
                    const int b = (__ffs((int)m) - 1) >> 2; m &= m - 1;
                    const int j = 4 * i + b;
                    const uint32_t q = (Q[i] >> (8 * b)) & 0xffu;
                    uint32_t row; asm volatile("ld.shared.u16 %0, [%1];" : "=r"(row) : "r"(rowtab_s + 2u * q));
                    uint32_t v; asm volatile("ld.shared.u8 %0, [%1];" : "=r"(v) : "r"(cbase + (uint32_t)(j * stepb) + (row & 0x7fffu) + 16u));
                    R[i] = (R[i] & ~(0xffu << (8 * b))) | (v << (8 * b));
                }
            }
            // QUAL values below 6 (and values without a table row) stay as they are (bqsr.go:968)
#pragma unroll
            for (int w = 0; w < 8; w++) {
                const uint32_t x = Q[w];
                const uint32_t ge6 = ((((x & 0x7f7f7f7fu) + 0x7a7a7a7au) | x) & 0x80808080u) >> 7;      // 1 per byte >= 6
                const uint32_t mk = ge6 * 0xffu;
                R[w] = (R[w] & mk) | (x & ~mk);
            }
        }
        // ---- park the 32 bytes in the warp's image of the output stream, then aligned 16-byte stores ----
        if (nb > 0) {
            const uint32_t dst = img_s + phase + (uint32_t)(ooff - o0) + (uint32_t)i0;
#pragma unroll
            for (int j = 0; j < 32; j++) if (j < nb) asm volatile("st.shared.u8 [%0], %1;" ::"r"(dst + j), "r"(R[j >> 2] >> (8 * (j & 3))) : "memory");
        }
        __syncwarp();
        {
            const uint32_t total = (uint32_t)(o1 - o0), end = phase + total;
            uint8_t* gbase = A.out + (o0 - phase);
            for (uint32_t m = lane; m * 16u < end; m += 32) {
                const uint32_t b0 = m * 16u;
                if (b0 >= phase && b0 + 16u <= end) *reinterpret_cast<uint4*>(gbase + b0) = *reinterpret_cast<const uint4*>(img + b0);
            }
            // the first and the last 16-byte chunk may be shared with a neighbouring pass: one byte per lane (lanes 0-15 the first, 16-31 the last)
            const uint32_t mlast = (end - 1u) >> 4;
            if (lane < 16) { const uint32_t t = lane; if ((phase != 0 || end < 16u) && t >= phase && t < end) gbase[t] = img[t]; }
            else { const uint32_t t = mlast * 16u + (lane - 16u); if (mlast > 0 && (end & 15u) && t < end) gbase[t] = img[t]; }
        }
        __syncwarp();
    }
    for (int o = 16; o; o >>= 1) errbits |= __shfl_xor_sync(FULL_MASK, errbits, o);
    if (errbits && lane == 0) atomicOr(A.err, errbits);
}
// QUAL bytes in output order without recalibration, any read length: one warp per read (the no-table path of elp_fetch for long reads)
__global__ void __launch_bounds__(256) qual_copy_kernel(uint64_t n, const int32_t* __restrict__ lseq, const uint64_t* __restrict__ qual_off, const uint64_t* __restrict__ out_off,
                                                        const uint8_t* __restrict__ qual, uint8_t* __restrict__ out) {
    const uint64_t k = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (k >= n) return;
    const int L = lseq[k];
    const uint8_t* src = qual + qual_off[k]; uint8_t* dst = out + out_off[k];
    for (int i = (int)lane_id(); i < L; i += 32) dst[i] = src[i];
}
}  // namespace

int run_apply_kernel(elp_ctx* c, bool with_lut) {
    const uint64_t n = c->n;
    uint64_t total = 0;
    if (n) {
        CUDA_TRY(c, cudaMemcpyAsync(&total, c->s_out_off.p + n, 8, cudaMemcpyDeviceToHost, c->stream));
        CUDA_TRY(c, cudaStreamSynchronize(c->stream));
    }
    CUDA_TRY(c, c->qual_out.reserve(total + 64, c->stream));
    c->qual_out_total = total;
    if (n) {
        static bool tables_set[64] = {false};
        if (!tables_set[c->device & 63]) {
            unsigned long long ge[CHUNK + 1], le[CHUNK + 1];
            for (int b = 0; b <= CHUNK; b++) { ge[b] = b == CHUNK ? 0ull : (ONES << (4 * b)); le[b] = b == 0 ? 0ull : (ONES >> (4 * (CHUNK - b))); }
            CUDA_TRY(c, cudaMemcpyToSymbol(c_ge, ge, sizeof ge)); CUDA_TRY(c, cudaMemcpyToSymbol(c_le, le, sizeof le));
            tables_set[c->device & 63] = true;
        }
        ApplyArgs A{};
        A.n = n; A.flag = c->s_flag.p; A.rg = c->s_rg.p; A.lseq = c->s_lseq.p; A.qual_off = c->s_qual_off.p; A.seq_off = c->s_seq_off.p; A.out_off = c->s_out_off.p;
        A.seq = c->seq.p; A.qual = c->qual.p; A.out = c->qual_out.p; A.rg_cov = c->d_rg_cov; A.n_rg = c->n_rg; A.cov_exists = c->d_cov_exists;
        A.lut = with_lut ? c->d_lut : nullptr; A.lut_maxcyc = c->lut_maxcyc; A.max_cycle = c->max_cycle; A.err = c->d_err;
        const double bytes = (double)n * (2 + 4 + 4 + 8 + 8 + 8) + (double)c->n_seq + 2.0 * (double)c->n_qual;
        // second-generation kernel: whenever the compact table fits shared memory and every cycle is inside it
        const char* force = getenv("ELPREP_B200_APPLY");
        const bool want_v2 = !(force && std::string(force) == "v1") && (!with_lut || (c->d_clut && c->clut_bytes && c->clut_Lc == c->lut_maxcyc && c->h_ranges.lseq_max <= c->clut_Lc)) && c->h_ranges.lseq_max <= 1024;
        if (want_v2) {
            Apply2Args B{};
            B.n = n; B.flag = c->s_flag.p; B.rg = c->s_rg.p; B.lseq = c->s_lseq.p; B.qual_off = c->s_qual_off.p; B.seq_off = c->s_seq_off.p; B.out_off = c->s_out_off.p;
            B.seq = c->seq.p; B.qual = c->qual.p; B.out = c->qual_out.p; B.rg_cov = c->d_rg_cov; B.n_rg = c->n_rg; B.cov_exists = c->d_cov_exists;
            B.clut = with_lut ? c->d_clut : nullptr; B.clut_bytes = with_lut ? c->clut_bytes : 0; B.blk = c->clut_blk; B.Lc = (uint32_t)c->clut_Lc; B.rowtab = c->d_rowtab; B.S17 = c->clut_S17;
            B.lpr = std::min(32, std::max(1, (c->h_ranges.lseq_max + 31) / 32)); B.rpw = 32 / B.lpr; B.err = c->d_err;
            if (!c->d_rowtab) { CUDA_TRY(c, cudaMalloc(&c->d_rowtab, 512)); CUDA_TRY(c, cudaMemsetAsync(c->d_rowtab, 0, 512, c->stream)); }
            B.rowtab = c->d_rowtab;
            int sms = 132; cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, c->device);
            const size_t smem = ((size_t)B.clut_bytes + 15) / 16 * 16 + (size_t)AP2_WARPS * (B.rpw * B.lpr * 32 + 32) + 16;
            CUDA_TRY(c, cudaFuncSetAttribute(bqsr_apply2_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
            const uint64_t n_pass = (n + B.rpw - 1) / B.rpw;
            const unsigned grid = (unsigned)std::min<uint64_t>((n_pass + AP2_WARPS - 1) / AP2_WARPS, (uint64_t)sms * 2);
            c->begin(with_lut ? "bqsr_apply" : "qual_materialize", bytes);
            bqsr_apply2_kernel<<<grid, AP2_WARPS * 32, smem, c->stream>>>(B);
            c->end(); LAUNCH_CHECK(c);
            int rc2 = check_device_errors(c);
            if (rc2) return rc2;
            c->qual_out_valid = true;
            return E_OK;
        }
        if (!with_lut && c->h_ranges.lseq_max > CHUNK * 32) {      // longer than either tiled kernel handles: plain per-read copy
            c->begin("qual_materialize", 2.0 * (double)c->n_qual + (double)n * 20);
            qual_copy_kernel<<<(unsigned)((n * 32 + 255) / 256), 256, 0, c->stream>>>(n, c->s_lseq.p, c->s_qual_off.p, c->s_out_off.p, c->qual.p, c->qual_out.p);
            c->end(); LAUNCH_CHECK(c);
            c->qual_out_valid = true;
            return E_OK;
        }
        // bqsr_apply_kernel's output image holds WARPS reads of at most CHUNK * 32 bases: longer reads are refused here, before
        // the launch (inside the kernel the block's slice of the output stream would overrun the image)
        if (c->h_ranges.lseq_max > CHUNK * 32)
            return c->fail(E_LIMIT, "BQSR: read longer than the device kernel supports (%d bases; without the shared-memory apply table the limit is %d)",
                           c->h_ranges.lseq_max, CHUNK * 32);
        A.lanes_per_read = std::min(32, std::max(1, (c->h_ranges.lseq_max + CHUNK - 1) / CHUNK));
        const uint64_t reads_per_block = (uint64_t)WARPS * (32 / A.lanes_per_read);
        // its own stats name, so that a caller can tell which apply kernel ran ("bqsr_apply" is bqsr_apply2_kernel)
        c->begin(with_lut ? "bqsr_apply_gmem" : "qual_materialize", bytes);
        bqsr_apply_kernel<<<(unsigned)((n + reads_per_block - 1) / reads_per_block), WARPS * 32, 0, c->stream>>>(A);
        c->end(); LAUNCH_CHECK(c);
    }
    int rc = check_device_errors(c);
    if (rc) return rc;
    c->qual_out_valid = true;
    return E_OK;
}

int phase_bqsr_apply(elp_ctx* c) {
    if (!c->sorted) return c->fail(E_STATE, "elp_bqsr_apply called before elp_sort_markdup");
    if (!c->finalized) return c->fail(E_STATE, "elp_bqsr_apply called before elp_bqsr_finalize");
    // the look-up table must cover every cycle of the reads now loaded (it was sized by elp_bqsr_finalize, possibly before they arrived)
    int rc = phase_adapt(c);
    if (rc) return rc;
    const int need = std::max(1, std::min(c->max_cycle, std::max(c->h_ranges.lseq_max, 1)));
    if (c->lut_maxcyc < need) { rc = build_apply_lut(c, need); if (rc) return rc; }
    rc = build_compact_lut(c);
    if (rc) return rc;
    return run_apply_kernel(c, true);
}
