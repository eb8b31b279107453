// markdup.cu -- duplicate marking on the device (replaces filters/mark-duplicates.go:36-445).
//
// The reference classifies reads one by one into three sharded concurrent maps with CAS "best" handles.  Here the
// same equivalence classes are formed by sorting exact packed keys (no hashing of group keys, so no collisions):
//   adapt_kernel        adaptAlignment (:153-156): unclipped 5' position (:79-110) + clamped phred sum (:36-68),
//                       plus a 39-bit (library, QNAME) hash for the mate join and the value ranges that size the keys
//   fragment groups     key (lib, refid, unclipped pos, strand | is_frag, score desc) -> radix sort of the group bits only ->
//                       frag_mark_kernel: one thread per group head walks its run (classifyFragment :210-254)
//   mate join           sort by the (lib,QNAME) hash, verify on bytes, pair up in arrival order
//                       (DeleteOrStore on pairFragment :336)
//   pair groups         key (lib, refid1, refid2, rev1, rev2, upos1, upos2), 64 bits when it fits, else 128 -> radix sort ->
//                       pair_mark_kernel (classifyPair :329-396): both mates of every loser get 0x400
// Results are deterministic; where the reference depends on goroutine scheduling (equal score AND equal QNAME) the
// outcome equals a single goroutine processing reads in arrival order (the later read/pair survives, :231-238,380-386).
#include "ctx.h"
#include <climits>
#include <algorithm>

namespace {

constexpr uint32_t NONE = 0xffffffffu;

__device__ __forceinline__ uint64_t mix64(uint64_t x) {
    x ^= x >> 33; x *= 0xff51afd7ed558ccdULL; x ^= x >> 33; x *= 0xc4ceb9fe1a85ec53ULL; x ^= x >> 33;
    return x;
}

// ---------------------------------------------------------------- K1 adapt
// adaptAlignment (mark-duplicates.go:153-156) for every read, one THREAD per read over tiles of consecutive reads.  The reads of a tile
// are consecutive in the QUAL, QNAME and CIGAR arenas (arrival order), so a tile's three byte strips are fetched with one TMA bulk copy
// each (cp.async.bulk, mbarrier-completed) into a four-deep shared-memory ring; the threads then read their read's bytes out of shared
// memory word by word (masked SWAR compares + __dp4a for the phred sum, a position-salted word mix for the (library, QNAME) hash).
// A tile whose strips do not fit its ring slot (very long reads) takes the same code with global loads.
constexpr int AD_T = 256, AD_STAGES = 4;
constexpr uint32_t AD_QCAP = 39 * 1024, AD_NCAP = 9 * 1024, AD_CCAP = 3 * 1024, AD_STAGE = AD_QCAP + AD_NCAP + AD_CCAP;

struct AdaptArgs {
    uint64_t n; int reads_per_tile;
    const uint16_t* flag; const int32_t *pos, *rg, *rg_lib; int n_rg;
    const uint64_t* cigar_off; const uint32_t* cigar; const uint64_t* qual_off; const uint8_t* qual; const uint64_t* qname_off; const uint8_t* qname;
    int32_t *upos, *score; uint64_t* qhash; DeviceRanges* ranges; uint32_t* err;
};

__device__ __forceinline__ uint32_t lds32(uint32_t a) { uint32_t v; asm volatile("ld.shared.u32 %0, [%1];" : "=r"(v) : "r"(a)); return v; }
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) { asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory"); }
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) { asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory"); }
__device__ __forceinline__ void mbar_arrive(uint32_t bar) { asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory"); }
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
    asm volatile("{\n .reg .pred P1;\n AD_WAIT:\n mbarrier.try_wait.parity.shared::cta.b64 P1, [%0], %1;\n @P1 bra AD_DONE;\n bra AD_WAIT;\n AD_DONE:\n }" ::"r"(bar), "r"(parity) : "memory");
}
// TMA 1-D bulk copy global -> shared, completion counted in bytes on an mbarrier (16-byte aligned addresses and size)
__device__ __forceinline__ void bulk_g2s(uint32_t dst, const void* src, uint32_t bytes, uint32_t bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(dst), "l"(src), "r"(bytes), "r"(bar) : "memory");
}

// word-granular byte-strip access: STAGED reads shared memory at (base + byte offset), otherwise global memory
template <bool STAGED> struct Strip {
    uint32_t sbase; const uint8_t* gbase;     // address of arena byte `origin` in shared memory / the arena itself
    uint64_t origin;
    __device__ __forceinline__ uint32_t word(uint64_t aligned_byte) const {     // 4-byte aligned arena offset
        if (STAGED) return lds32(sbase + (uint32_t)(aligned_byte - origin));
        return __ldg(reinterpret_cast<const uint32_t*>(gbase + aligned_byte));
    }
};

// computePhredScore (:57-68): sum over QUAL >= 15 of (q & 0x7f) (the table index byte(char << 1) wraps), bad: some byte > 93
template <bool STAGED> __device__ __forceinline__ uint32_t phred_score(const Strip<STAGED>& Q, uint64_t q0, uint64_t q1, unsigned lane, uint32_t& bad) {
    if (q1 <= q0) return 0;
    const uint64_t w0 = q0 & ~3ull;
    const uint32_t nw = (uint32_t)((((q1 - 1) & ~3ull) - w0) >> 2) + 1;
    const uint32_t first_mask = 0xffffffffu << (8 * (uint32_t)(q0 & 3)), last_mask = 0xffffffffu >> (8 * (3 - (uint32_t)((q1 - 1) & 3)));
    uint32_t s = 0;
    uint32_t k = lane % nw;                        // lanes start at different words: no shared-memory bank pile-up for power-of-two read lengths
    for (uint32_t t = 0; t < nw; t++) {
        uint32_t m = 0x7f7f7f7fu;
        if (k == 0) m &= first_mask;
        if (k == nw - 1) m &= last_mask;
        const uint32_t x = Q.word(w0 + 4ull * k) & m;            // bytes < 128: the adds below cannot carry across bytes
        bad |= (x + 0x22222222u) & 0x80808080u;
        const uint32_t ge15 = ((x + 0x71717171u) & 0x80808080u) >> 7;
        s = __dp4a(x & (ge15 * 0xffu), 0x01010101u, s);
        k = (k + 1 == nw) ? 0 : k + 1;
    }
    return s;
}
// (library, QNAME) hash for the mate join: a function of the name bytes only (equality is verified on bytes in join_kernel)
template <bool STAGED> __device__ __forceinline__ uint64_t qname_hash(const Strip<STAGED>& N, uint64_t n0, uint64_t n1) {
    uint64_t h = 0;
    if (n1 <= n0) return h;
    const uint32_t sh = 8 * (uint32_t)(n0 & 3);
    uint64_t a = n0 & ~3ull;
    uint32_t lo = N.word(a);
    for (uint64_t k = n0; k < n1; k += 4) {
        const uint32_t hi = (a + 4 < n1) ? N.word(a + 4) : 0u;   // only fetched when the name continues into the next word
        uint32_t wv = __funnelshift_r(lo, hi, sh);
        const uint32_t rem = (uint32_t)(n1 - k);
        if (rem < 4) wv &= 0xffffffffu >> (8 * (4 - rem));
        uint32_t m = (wv ^ ((uint32_t)(k - n0) * 0x9E3779B1u)) * 0x85EBCA6Bu;
        m ^= m >> 15; m *= 0xC2B2AE35u; m ^= m >> 13;
        h += (uint64_t)m * 0x9E3779B97F4A7C15ull;
        lo = hi; a += 4;
    }
    return h;
}
// computeUnclippedPosition (:79-110)
template <bool STAGED> __device__ __forceinline__ int32_t unclipped_pos(const Strip<STAGED>& C, uint64_t c0, uint64_t c1, int32_t p, bool reversed) {
    int32_t up = p;
    if (c1 <= c0) return up;
    if (reversed) {
        int32_t clipped = 1; up--;
        for (uint64_t k = c1; k-- > c0;) {
            const uint32_t op = C.word(4 * k); const uint32_t o = op & 15; const int32_t l = (int32_t)(op >> 4);
            const int32_t cl = (o == 4 || o == 5), r = (o == 0 || o == 2 || o == 3 || o == 7 || o == 8);
            clipped *= cl;
            up += (r | clipped) * l;
        }
    } else {
        for (uint64_t k = c0; k < c1; k++) { const uint32_t op = C.word(4 * k); const uint32_t o = op & 15; if (!(o == 4 || o == 5)) break; up -= (int32_t)(op >> 4); }
    }
    return up;
}

struct AdTile { uint64_t qb, nb, cb; uint32_t staged; };   // arena offsets of the first staged byte of each strip

__global__ void __launch_bounds__(AD_T, 1) adapt_kernel(AdaptArgs A) {
    extern __shared__ __align__(128) unsigned char ad_smem[];
    __shared__ __align__(8) uint64_t bars[AD_STAGES];
    __shared__ AdTile tinfo[AD_STAGES];
    const unsigned tid = threadIdx.x, lane = tid & 31;
    const uint32_t sm0 = (uint32_t)__cvta_generic_to_shared(ad_smem), bar0 = (uint32_t)__cvta_generic_to_shared(bars);
    const uint64_t R = (uint64_t)A.reads_per_tile, n_tiles = (A.n + R - 1) / R;
    if (tid == 0) { for (int s = 0; s < AD_STAGES; s++) mbar_init(bar0 + 8 * s, 1); asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
    __syncthreads();
    // thread 0: strips of tile t -> ring slot `slot`
    auto issue = [&](uint64_t t, int slot) {
        const uint64_t i0 = t * R, i1 = min(A.n, i0 + R);
        const uint64_t qa = A.qual_off[i0], qe = A.qual_off[i1], na = A.qname_off[i0], ne = A.qname_off[i1], ca = A.cigar_off[i0] * 4, ce = A.cigar_off[i1] * 4;
        const uintptr_t gq = reinterpret_cast<uintptr_t>(A.qual), gn = reinterpret_cast<uintptr_t>(A.qname), gc = reinterpret_cast<uintptr_t>(A.cigar);
        // windows aligned on 16-byte ADDRESSES (the arenas themselves are 256-byte aligned, so offsets and addresses agree mod 16)
        const uint64_t qb = qa & ~15ull, nb = na & ~15ull, cb = ca & ~15ull;
        const uint64_t qs = ((qe + 15) & ~15ull) - qb, ns = ((ne + 15) & ~15ull) - nb, cs = ((ce + 15) & ~15ull) - cb;
        const bool fits = qs <= AD_QCAP && ns <= AD_NCAP && cs <= AD_CCAP && ((gq | gn | gc) & 15) == 0;
        AdTile ti; ti.qb = qb; ti.nb = nb; ti.cb = cb; ti.staged = fits ? 1u : 0u;
        tinfo[slot] = ti;
        const uint32_t bar = bar0 + 8 * slot, dst = sm0 + (uint32_t)slot * AD_STAGE;
        if (fits) {
            mbar_expect_tx(bar, (uint32_t)(qs + ns + cs));
            if (qs) bulk_g2s(dst, A.qual + qb, (uint32_t)qs, bar);
            if (ns) bulk_g2s(dst + AD_QCAP, A.qname + nb, (uint32_t)ns, bar);
            if (cs) bulk_g2s(dst + AD_QCAP + AD_NCAP, reinterpret_cast<const uint8_t*>(A.cigar) + cb, (uint32_t)cs, bar);
        } else mbar_arrive(bar);
    };
    if (tid == 0) for (int s = 0; s < AD_STAGES - 1; s++) { const uint64_t t = (uint64_t)blockIdx.x + (uint64_t)s * gridDim.x; if (t < n_tiles) issue(t, s); }
    __syncthreads();

    int32_t pos_max = 0, upos_min = INT_MAX, upos_max = INT_MIN, score_max = 0, lseq_max = 0, pos_min = 0, qname_max = 0;
    uint32_t n_enter = 0, n_pairs = 0, errbits = 0;
    uint64_t it = 0;
    for (uint64_t t = blockIdx.x; t < n_tiles; t += gridDim.x, it++) {
        const int slot = (int)(it % AD_STAGES);
        // refill the slot that was consumed in the previous iteration (all threads passed its trailing __syncthreads)
        if (tid == 0) { const uint64_t tn = t + (uint64_t)(AD_STAGES - 1) * gridDim.x; if (tn < n_tiles) issue(tn, (int)((it + AD_STAGES - 1) % AD_STAGES)); }
        const uint64_t i = t * R + tid;
        const bool valid = tid < R && i < A.n;
        uint16_t f = 0; int32_t p = 0; uint64_t q0 = 0, q1 = 0, n0 = 0, n1 = 0, c0 = 0, c1 = 0; int32_t g = -1;
        if (valid) { f = A.flag[i]; p = A.pos[i]; q0 = A.qual_off[i]; q1 = A.qual_off[i + 1]; n0 = A.qname_off[i]; n1 = A.qname_off[i + 1]; c0 = A.cigar_off[i]; c1 = A.cigar_off[i + 1]; g = A.rg[i]; }
        mbar_wait(bar0 + 8 * slot, (uint32_t)((it / AD_STAGES) & 1));
        const AdTile ti = tinfo[slot];
        if (valid) {
            const int32_t len = (int32_t)(q1 - q0);
            qname_max = max(qname_max, (int32_t)(n1 - n0));
            pos_max = max(pos_max, p); pos_min = min(pos_min, p); lseq_max = max(lseq_max, len);
            const bool entering = (f & (F_UNMAPPED | F_SECONDARY | F_SUPPLEMENTARY)) == 0;          // mark-duplicates.go:436
            const bool true_pair = entering && (f & (F_MULTIPLE | F_NEXTUNMAPPED)) == F_MULTIPLE;   // :182-184
            int32_t up = 0, sc = 0; uint64_t qh = 0;
            if (entering) {
                uint32_t bad = 0; uint64_t h = 0;
                const uint32_t sbase = sm0 + (uint32_t)slot * AD_STAGE;
                if (ti.staged) {
                    const Strip<true> Q{sbase, nullptr, ti.qb}, N{sbase + AD_QCAP, nullptr, ti.nb}, C{sbase + AD_QCAP + AD_NCAP, nullptr, ti.cb};
                    sc = (int32_t)phred_score(Q, q0, q1, lane, bad);
                    up = unclipped_pos(C, c0, c1, p, (f & F_REVERSED) != 0);
                    if (true_pair) h = qname_hash(N, n0, n1);
                } else {
                    const Strip<false> Q{0, A.qual, 0}, N{0, A.qname, 0}, C{0, reinterpret_cast<const uint8_t*>(A.cigar), 0};
                    sc = (int32_t)phred_score(Q, q0, q1, lane, bad);
                    up = unclipped_pos(C, c0, c1, p, (f & F_REVERSED) != 0);
                    if (true_pair) h = qname_hash(N, n0, n1);
                }
                if (bad) errbits |= DERR_QUAL;
                const int32_t lib = (g >= 0 && g < A.n_rg) ? A.rg_lib[g] : -1;
                if (true_pair) { qh = mix64(h + (uint64_t)(uint32_t)(lib + 1) * 0x9E3779B97F4A7C15ull + (n1 - n0)); n_pairs++; }
                upos_min = min(upos_min, up); upos_max = max(upos_max, up); score_max = max(score_max, sc); n_enter++;
            }
            A.upos[i] = up; A.score[i] = sc; A.qhash[i] = qh;
        }
        __syncthreads();
    }
    // block reduction of the ranges, then one atomic per block
    __shared__ int32_t sh_i[8][7];
    __shared__ uint32_t sh_u[8][3];
    for (int o = 16; o; o >>= 1) {
        pos_max = max(pos_max, __shfl_xor_sync(FULL_MASK, pos_max, o)); pos_min = min(pos_min, __shfl_xor_sync(FULL_MASK, pos_min, o));
        upos_min = min(upos_min, __shfl_xor_sync(FULL_MASK, upos_min, o)); upos_max = max(upos_max, __shfl_xor_sync(FULL_MASK, upos_max, o));
        score_max = max(score_max, __shfl_xor_sync(FULL_MASK, score_max, o)); lseq_max = max(lseq_max, __shfl_xor_sync(FULL_MASK, lseq_max, o)); qname_max = max(qname_max, __shfl_xor_sync(FULL_MASK, qname_max, o));
        n_enter += __shfl_xor_sync(FULL_MASK, n_enter, o); n_pairs += __shfl_xor_sync(FULL_MASK, n_pairs, o); errbits |= __shfl_xor_sync(FULL_MASK, errbits, o);
    }
    const unsigned w = threadIdx.x >> 5;
    if (lane == 0) { sh_i[w][0] = pos_max; sh_i[w][1] = upos_min; sh_i[w][2] = upos_max; sh_i[w][3] = score_max; sh_i[w][4] = lseq_max; sh_i[w][5] = pos_min; sh_i[w][6] = qname_max; sh_u[w][0] = n_enter; sh_u[w][1] = n_pairs; sh_u[w][2] = errbits; }
    __syncthreads();
    if (threadIdx.x == 0) {
        const int nwb = blockDim.x >> 5;
        for (int k = 1; k < nwb; k++) {
            sh_i[0][0] = max(sh_i[0][0], sh_i[k][0]); sh_i[0][1] = min(sh_i[0][1], sh_i[k][1]); sh_i[0][2] = max(sh_i[0][2], sh_i[k][2]);
            sh_i[0][3] = max(sh_i[0][3], sh_i[k][3]); sh_i[0][4] = max(sh_i[0][4], sh_i[k][4]); sh_i[0][5] = min(sh_i[0][5], sh_i[k][5]); sh_i[0][6] = max(sh_i[0][6], sh_i[k][6]);
            sh_u[0][0] += sh_u[k][0]; sh_u[0][1] += sh_u[k][1]; sh_u[0][2] |= sh_u[k][2];
        }
        atomicMax(&A.ranges->pos_max, sh_i[0][0]); atomicMin(&A.ranges->upos_min, sh_i[0][1]); atomicMax(&A.ranges->upos_max, sh_i[0][2]);
        atomicMax(&A.ranges->score_max, sh_i[0][3]); atomicMax(&A.ranges->lseq_max, sh_i[0][4]); atomicMax(&A.ranges->qname_max, sh_i[0][6]);
        atomicAdd(&A.ranges->n_entering, sh_u[0][0]); atomicAdd(&A.ranges->n_true_pairs, sh_u[0][1]);
        if (sh_i[0][5] < 0) sh_u[0][2] |= DERR_QUAL_RANGE;   // negative POS: not representable in the compact sort key
        if (sh_u[0][2]) atomicOr(A.err, sh_u[0][2]);
    }
}

// ---------------------------------------------------------------- fragment groups
struct FragLayout { int bS, bU, bR, bL; int32_t upos_min, score_max; int key_bits; };

__global__ void __launch_bounds__(256) frag_keys_kernel(uint64_t n, const uint16_t* __restrict__ flag, const int32_t* __restrict__ refid, const int32_t* __restrict__ rg,
                                                         const int32_t* __restrict__ rg_lib, int n_rg, const int32_t* __restrict__ upos, const int32_t* __restrict__ score,
                                                         FragLayout L, uint64_t* __restrict__ keys, uint32_t* __restrict__ vals) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint16_t f = flag[i];
    uint64_t key;
    if ((f & (F_UNMAPPED | F_SECONDARY | F_SUPPLEMENTARY)) == 0) {
        const int32_t g = rg[i];
        const uint64_t lib = (uint64_t)(((g >= 0 && g < n_rg) ? rg_lib[g] : -1) + 1);
        const uint64_t is_frag = ((f & (F_MULTIPLE | F_NEXTUNMAPPED)) != F_MULTIPLE) ? 1 : 0;   // isTrueFragment :177-179
        key = (uint64_t)(uint32_t)(L.score_max - score[i]);
        int sh = L.bS;
        key |= is_frag << sh; sh += 1;
        key |= (uint64_t)((f & F_REVERSED) ? 1 : 0) << sh; sh += 1;
        key |= (uint64_t)(uint32_t)(upos[i] - L.upos_min) << sh; sh += L.bU;
        key |= (uint64_t)(uint32_t)(refid[i] + 1) << sh; sh += L.bR;
        key |= lib << sh;
    } else {
        key = L.key_bits >= 64 ? ~0ull : ((1ull << L.key_bits) - 1);   // sorts after every real key (library field holds an unused value)
    }
    keys[i] = key; vals[i] = (uint32_t)i;
}

// keys sorted by the group bits (>= bS + 1) only, so a group is in arrival order; score and is_frag are read from the low key bits
__global__ void __launch_bounds__(256) frag_mark_kernel(uint64_t m, const uint64_t* __restrict__ keys, const uint32_t* __restrict__ vals, int bS,
                                                         const uint64_t* __restrict__ qname_off, const uint8_t* __restrict__ qname, uint16_t* __restrict__ flag) {
    const uint64_t j = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= m) return;
    const uint64_t k0 = keys[j], g = k0 >> (bS + 1);
    if (j > 0 && (keys[j - 1] >> (bS + 1)) == g) return;   // not a group head
    if (j + 1 == m || (keys[j + 1] >> (bS + 1)) != g) return;   // a read alone in its group is never a duplicate
    const uint64_t smask = (1ull << bS) - 1;
    // winner among fragments = max score (smallest score_max - score), then smallest QNAME (:228-243); full ties: the later arrival survives
    bool has_pair = false;
    uint64_t e = j, win = j;
    uint64_t best = ~0ull;
    for (; e < m; e++) {
        const uint64_t k = keys[e];
        if ((k >> (bS + 1)) != g) break;
        if (((k >> bS) & 1) == 0) { has_pair = true; continue; }
        if (has_pair) continue;
        const uint64_t sc = k & smask;
        if (sc < best) { best = sc; win = e; }
        else if (sc == best) {
            const uint32_t a = vals[e], b = vals[win];
            if (qname_compare(qname, qname_off[a], qname_off[a + 1], qname_off[b], qname_off[b + 1]) <= 0) win = e;
        }
    }
    // a true-pair read in the group: every true fragment is a duplicate, pair reads are untouched (:225-227,245-252)
    for (uint64_t t = j; t < e; t++) {
        if (has_pair ? ((keys[t] >> bS) & 1) != 0 : t != win) atomic_or_u16(flag, vals[t], F_DUPLICATE);
    }
}

// ---------------------------------------------------------------- mate join
__global__ void __launch_bounds__(256) join_keys_kernel(uint64_t n, const uint16_t* __restrict__ flag, const uint64_t* __restrict__ qhash,
                                                         uint64_t* __restrict__ keys, uint32_t* __restrict__ vals, uint32_t* __restrict__ mate) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint16_t f = flag[i];
    const bool in = (f & (F_UNMAPPED | F_SECONDARY | F_SUPPLEMENTARY)) == 0 && (f & (F_MULTIPLE | F_NEXTUNMAPPED)) == F_MULTIPLE;
    keys[i] = in ? (qhash[i] & 0x7fffffffull) : (1ull << 31);      // 31 hash bits + the "not a true pair" bit = 32 key bits = 4 passes (equal-hash runs are verified on bytes)
    vals[i] = (uint32_t)i;
    mate[i] = NONE;
}

__device__ __forceinline__ int32_t lib_of(const int32_t* rg, const int32_t* rg_lib, int n_rg, uint32_t i) { const int32_t g = rg[i]; return (g >= 0 && g < n_rg) ? rg_lib[g] : -1; }

__global__ void __launch_bounds__(256) join_kernel(uint64_t m, const uint64_t* __restrict__ keys, const uint32_t* __restrict__ vals,
                                                    const int32_t* __restrict__ rg, const int32_t* __restrict__ rg_lib, int n_rg,
                                                    const uint64_t* __restrict__ qname_off, const uint8_t* __restrict__ qname, uint32_t* __restrict__ mate) {
    const uint64_t j = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= m) return;
    const uint64_t k0 = keys[j];
    if (j > 0 && keys[j - 1] == k0) return;
    uint64_t e = j + 1;
    while (e < m && keys[e] == k0) e++;
    if (e - j == 2) {   // the common case: both reads still unpaired (join_keys_kernel), all loads issued before any compare
        const uint32_t va = vals[j], vb = vals[j + 1];
        const int32_t ga = rg[va], gb = rg[vb];
        const uint64_t a0 = qname_off[va], a1 = qname_off[va + 1], b0 = qname_off[vb], b1 = qname_off[vb + 1];
        const int32_t la = (ga >= 0 && ga < n_rg) ? rg_lib[ga] : -1, lb = (gb >= 0 && gb < n_rg) ? rg_lib[gb] : -1;
        if (la == lb && qname_compare(qname, a0, a1, b0, b1) == 0) { mate[va] = vb; mate[vb] = va; }
        return;
    }
    // arrival order inside the run (stable sort): first unmatched same-(lib,QNAME) read stores, the next one deletes and pairs (:336)
    for (uint64_t a = j; a < e; a++) {
        const uint32_t va = vals[a];
        if (a > j && mate[va] != NONE) continue;   // the run's first read is still unpaired
        const int32_t la = lib_of(rg, rg_lib, n_rg, va);
        for (uint64_t b = a + 1; b < e; b++) {
            const uint32_t vb = vals[b];
            if (mate[vb] != NONE) continue;
            if (la != lib_of(rg, rg_lib, n_rg, vb)) continue;
            if (qname_compare(qname, qname_off[va], qname_off[va + 1], qname_off[vb], qname_off[vb + 1]) != 0) continue;
            mate[va] = vb; mate[vb] = va;
            break;
        }
    }
}

__global__ void __launch_bounds__(256) pair_flag_kernel(uint64_t n, const uint32_t* __restrict__ mate, uint32_t* __restrict__ flags) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint32_t m = mate[i];
    flags[i] = (m != NONE && m < i) ? 1u : 0u;   // the later mate triggers classifyPair
}

struct PairLayout { int bU, bR, bL; int32_t upos_min; int key_bits; };

__device__ __forceinline__ void put128(uint64_t& lo, uint64_t& hi, int& sh, uint64_t v, int bits) {
    if (bits == 0) return;
    if (sh < 64) { lo |= v << sh; if (sh + bits > 64) hi |= v >> (64 - sh); }
    else hi |= v << (sh - 64);
    sh += bits;
}

__global__ void __launch_bounds__(256) pair_keys_kernel(uint64_t n, const uint32_t* __restrict__ mate, const uint64_t* __restrict__ slot,
                                                         const uint16_t* __restrict__ flag, const int32_t* __restrict__ refid, const int32_t* __restrict__ rg,
                                                         const int32_t* __restrict__ rg_lib, int n_rg, const int32_t* __restrict__ upos, const int32_t* __restrict__ score,
                                                         PairLayout L, uint64_t* __restrict__ keys /*u64, or u128 as lo,hi*/, uint32_t* __restrict__ vals,
                                                         uint32_t* __restrict__ pair_a, uint32_t* __restrict__ pair_b, int32_t* __restrict__ pair_score) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint32_t m = mate[i];
    if (!(m != NONE && m < i)) return;
    const uint64_t p = slot[i];
    // classifyPair :342-361: aln1 = arriving read (i), aln2 = stored mate (m); swap into (refid, upos, fwd<rev) order
    uint32_t a1 = (uint32_t)i, a2 = m;
    int32_t r1 = refid[a1], r2 = refid[a2], p1 = upos[a1], p2 = upos[a2];
    uint32_t v1 = (flag[a1] & F_REVERSED) ? 1 : 0, v2 = (flag[a2] & F_REVERSED) ? 1 : 0;
    if (r1 > r2 || (r1 == r2 && (p1 > p2 || (p1 == p2 && v1 && !v2)))) {
        uint32_t t = a1; a1 = a2; a2 = t; int32_t ti = r1; r1 = r2; r2 = ti; ti = p1; p1 = p2; p2 = ti; t = v1; v1 = v2; v2 = t;
    }
    const int32_t g = rg[a1];
    const uint64_t lib = (uint64_t)(((g >= 0 && g < n_rg) ? rg_lib[g] : -1) + 1);
    uint64_t lo = 0, hi = 0; int sh = 0;
    put128(lo, hi, sh, (uint64_t)(uint32_t)(p2 - L.upos_min), L.bU);
    put128(lo, hi, sh, (uint64_t)(uint32_t)(p1 - L.upos_min), L.bU);
    put128(lo, hi, sh, v2, 1); put128(lo, hi, sh, v1, 1);
    put128(lo, hi, sh, (uint64_t)(uint32_t)(r2 + 1), L.bR); put128(lo, hi, sh, (uint64_t)(uint32_t)(r1 + 1), L.bR);
    put128(lo, hi, sh, lib, L.bL);
    if (L.key_bits <= 64) keys[p] = lo;
    else { keys[2 * p] = lo; keys[2 * p + 1] = hi; }
    vals[p] = (uint32_t)p;
    pair_a[p] = a1; pair_b[p] = a2; pair_score[p] = score[a1] + score[a2];
}

__device__ __forceinline__ bool same_key(const uint64_t* keys, uint64_t a, uint64_t b, int words) {
    return words == 1 ? keys[a] == keys[b] : (keys[2 * a] == keys[2 * b] && keys[2 * a + 1] == keys[2 * b + 1]);
}

// keys sorted by the signature only, so a group is in pair arrival order
__global__ void __launch_bounds__(256) pair_mark_kernel(uint64_t m, const uint64_t* __restrict__ keys, const uint32_t* __restrict__ vals, int words,
                                                         const uint32_t* __restrict__ pair_a, const uint32_t* __restrict__ pair_b, const int32_t* __restrict__ pair_score,
                                                         const uint64_t* __restrict__ qname_off, const uint8_t* __restrict__ qname, uint16_t* __restrict__ flag) {
    const uint64_t j = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= m) return;
    if (j > 0 && same_key(keys, j - 1, j, words)) return;   // not a group head
    if (j + 1 == m || !same_key(keys, j, j + 1, words)) return;   // a single pair (most groups): no score needed
    // winner = max score, then smallest aln1.QNAME (:375-395); full ties: the later pair survives
    uint64_t e = j + 1, win = j;
    int32_t best = pair_score[vals[j]];
    for (; e < m && same_key(keys, j, e, words); e++) {
        const int32_t sc = pair_score[vals[e]];
        if (sc > best) { best = sc; win = e; }
        else if (sc == best) {
            const uint32_t a = pair_a[vals[e]], b = pair_a[vals[win]];
            if (qname_compare(qname, qname_off[a], qname_off[a + 1], qname_off[b], qname_off[b + 1]) <= 0) win = e;
        }
    }
    for (uint64_t t = j; t < e; t++)
        if (t != win) { const uint32_t p = vals[t]; atomic_or_u16(flag, pair_a[p], F_DUPLICATE); atomic_or_u16(flag, pair_b[p], F_DUPLICATE); }
}

inline unsigned nblk(uint64_t n, int t) { return (unsigned)((n + t - 1) / t); }

}  // namespace

int check_device_errors(elp_ctx* c) {
    uint32_t e = 0;
    CUDA_TRY(c, cudaMemcpyAsync(&e, c->d_err, 4, cudaMemcpyDeviceToHost, c->stream));
    CUDA_TRY(c, cudaStreamSynchronize(c->stream));
    if (!e) return E_OK;
    CUDA_TRY(c, cudaMemsetAsync(c->d_err, 0, 4, c->stream));
    if (e & DERR_QUAL) return c->fail(E_QUAL, "Invalid QUAL character in a read entering duplicate marking");
    if (e & DERR_NORG) return c->fail(E_NORG, "Error: BQSR requires input with read groups. An alignment has no read group. Please fix input, e.g. rerun with the --replace-read-group option.");
    if (e & DERR_CYCLE) return c->fail(E_CYCLE, "cycle value exceeds maximum cycle value");
    if (e & DERR_CLIP) return c->fail(E_CLIP, "reference coordinate matches a non-existing base in read");
    if (e & DERR_REFEND) return c->fail(E_REFEND, "a recalibrated read extends past the end of its reference sequence");
    if (e & DERR_CIGAR_LIMIT) return c->fail(E_LIMIT, "BQSR: CIGAR with more operations than the device kernel supports");
    if (e & DERR_QUAL_RANGE) return c->fail(E_LIMIT, "value outside the supported range (negative POS, or QUAL > 93 in a recalibrated read)");
    if (e & DERR_TILE) return c->fail(E_TILE, "strconv.ParseInt: parsing a tile/x/y field of a QNAME: invalid syntax or value out of range");
    if (e & DERR_TILE_RANGE) return c->fail(E_LIMIT, "optical duplicates: tile/x/y value outside int32");
    if (e & DERR_BAM_CG) return c->fail(E_LIMIT, "BAM record uses the CG:B long-CIGAR convention, which the device parser does not handle");
    if (e & DERR_BAM_RG) return c->fail(E_BAM, "BAM record with an RG:Z value that is not an @RG ID of the header");
    if (e & DERR_BAM) return c->fail(E_BAM, "malformed BAM alignment record (field lengths and block_size do not add up)");
    if (e & DERR_READLEN_LIMIT) return c->fail(E_LIMIT, "BQSR: read longer than the device kernel supports");
    if (e & DERR_CLEANSAM) return c->fail(E_LIMIT, "Unexpected non-0 relative clipping position in CleanSam.");
    if (e & DERR_SPREAD_NAME) return c->fail(E_LIMIT, "cross-group pair exchange: QNAME longer than 92 bytes");
    return c->fail(E_CUDA, "unknown device error word 0x%x", e);
}

int phase_adapt(elp_ctx* c) {
    if (c->adapted) return E_OK;
    const uint64_t n = c->n;
    CUDA_TRY(c, c->upos.reserve(n + 1, c->stream));
    CUDA_TRY(c, c->score.reserve(n + 1, c->stream));
    CUDA_TRY(c, c->qhash.reserve(n + 1, c->stream));
    DeviceRanges init{}; init.pos_max = 0; init.upos_min = INT_MAX; init.upos_max = INT_MIN; init.score_max = 0; init.lseq_max = 0;
    { int rcu = upload_small(c, c->d_ranges, &init, sizeof init); if (rcu) return rcu; }
    if (n) {
        int sms = 132; cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, c->device);
        AdaptArgs A{};
        A.n = n; A.flag = c->flag.p; A.pos = c->pos.p; A.rg = c->rg.p; A.rg_lib = c->d_rg_lib; A.n_rg = c->n_rg; A.cigar_off = c->cigar_off.p; A.cigar = c->cigar.p;
        A.qual_off = c->qual_off.p; A.qual = c->qual.p; A.qname_off = c->qname_off.p; A.qname = c->qname.p; A.upos = c->upos.p; A.score = c->score.p; A.qhash = c->qhash.p;
        A.ranges = c->d_ranges; A.err = c->d_err;
        // reads per tile: as many as fit the ring slot on average (256 reads of 150 bases; fewer for longer reads)
        const double avg_q = (double)(c->n_qual - ARENA_FRONT_PAD) / (double)n + 1, avg_n = (double)c->n_qname / (double)n + 1, avg_c = 4.0 * (double)c->n_cigar / (double)n + 1;
        int rpt = (int)std::min({(double)AD_T, 0.94 * AD_QCAP / avg_q, 0.94 * AD_NCAP / avg_n, 0.94 * AD_CCAP / avg_c});
        A.reads_per_tile = std::max(32, rpt & ~31);
        const uint64_t n_tiles = (n + A.reads_per_tile - 1) / A.reads_per_tile;
        const unsigned grid = (unsigned)std::min<uint64_t>(n_tiles, (uint64_t)sms);
        const size_t smem = (size_t)AD_STAGES * AD_STAGE;
        CUDA_TRY(c, cudaFuncSetAttribute(adapt_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        double bytes = (double)n * (2 + 4 + 4 + 16 + 16 + 8 + 4 + 4 + 8) + (double)(c->n_qual - ARENA_FRONT_PAD) + (double)c->n_cigar * 4 + (double)c->n_qname;
        c->begin("adapt", bytes);
        adapt_kernel<<<grid, AD_T, smem, c->stream>>>(A);
        c->end(); LAUNCH_CHECK(c);
    }
    CUDA_TRY(c, cudaMemcpyAsync(&c->h_ranges, c->d_ranges, sizeof(DeviceRanges), cudaMemcpyDeviceToHost, c->stream));
    int rc = check_device_errors(c);   // synchronizes
    if (rc) return rc;
    if (c->h_ranges.n_entering == 0) { c->h_ranges.upos_min = 0; c->h_ranges.upos_max = 0; }
    c->adapted = true;
    return E_OK;
}

// pairs (classifyPair) over the local reads plus the ghost reads spread_exchange_begin appended (comm.cu); ghosts are true pairs by construction
static int mark_pairs(elp_ctx* c, bool optical, uint64_t nt, uint64_t n_true_pairs, int bU, int bR, int bL) {
    const DeviceRanges& R = c->h_ranges;
    int rc;
    if (n_true_pairs < 2) return optical ? phase_optical(c, 0, nullptr, nullptr, 0) : E_OK;
    CUDA_TRY(c, c->mate.reserve(nt + 4, c->stream));
    c->begin("join_keys", (double)nt * (2 + 8 + 8 + 4 + 4));
    join_keys_kernel<<<nblk(nt, 256), 256, 0, c->stream>>>(nt, c->flag.p, c->qhash.p, c->keys_a.p, c->vals_a.p, c->mate.p);
    c->end(); LAUNCH_CHECK(c);
    bool in_b = false;
    rc = radix_sort_u64(c, c->keys_a.p, c->keys_b.p, c->vals_a.p, c->vals_b.p, nt, 32, &in_b, "u64");   // 31 hash bits + 1: runs of equal hash are verified on bytes anyway
    if (rc) return rc;
    const uint64_t m = n_true_pairs;
    c->begin("join", (double)m * 12);
    join_kernel<<<nblk(m, 256), 256, 0, c->stream>>>(m, in_b ? c->keys_b.p : c->keys_a.p, in_b ? c->vals_b.p : c->vals_a.p, c->rg.p, c->d_rg_lib, c->n_rg, c->qname_off.p, c->qname.p, c->mate.p);
    c->end(); LAUNCH_CHECK(c);
    // deterministic pair list, ordered by the arrival of the later mate
    CUDA_TRY(c, c->scan_tmp.reserve(nt + 4, c->stream));
    uint64_t* slot = c->keys_b.p;   // nt+1 u64, free at this point
    c->begin("pair_flag", (double)nt * 8);
    pair_flag_kernel<<<nblk(nt, 256), 256, 0, c->stream>>>(nt, c->mate.p, c->scan_tmp.p);
    c->end(); LAUNCH_CHECK(c);
    rc = exclusive_scan_u32_to_u64(c, c->scan_tmp.p, slot, nt);
    if (rc) return rc;
    uint64_t npairs = 0;
    CUDA_TRY(c, cudaMemcpyAsync(&npairs, slot + nt, 8, cudaMemcpyDeviceToHost, c->stream));
    CUDA_TRY(c, cudaStreamSynchronize(c->stream));
    if (npairs >= (optical ? 1u : 2u)) {
        CUDA_TRY(c, c->pair_a.reserve(npairs + 4, c->stream)); CUDA_TRY(c, c->pair_b.reserve(npairs + 4, c->stream)); CUDA_TRY(c, c->pair_score.reserve(npairs + 4, c->stream));
        // the signature without the score; bU comes from the allreduced ranges, so every rank picks the same key width
        PairLayout L{}; L.bU = bU; L.bR = bR; L.bL = bL; L.upos_min = R.upos_min;
        L.key_bits = 2 * L.bU + 2 + 2 * L.bR + L.bL;
        if (L.key_bits > 128) return c->fail(E_LIMIT, "pair signature needs %d bits (>128)", L.key_bits);
        const int words = L.key_bits <= 64 ? 1 : 2;
        // keys live in keys_a (u128 as (lo,hi) pairs); slot[] occupies keys_b, so sort into a separate buffer
        CUDA_TRY(c, c->bytes_tmp.reserve((size_t)npairs * 8 * words + 64, c->stream));
        uint64_t* kb2 = reinterpret_cast<uint64_t*>(c->bytes_tmp.p);
        c->begin("pair_keys", (double)nt * 12 + (double)npairs * (2 * 18 + 8 * words + 16));
        pair_keys_kernel<<<nblk(nt, 256), 256, 0, c->stream>>>(nt, c->mate.p, slot, c->flag.p, c->refid.p, c->rg.p, c->d_rg_lib, c->n_rg, c->upos.p, c->score.p, L,
                                                              c->keys_a.p, c->vals_a.p, c->pair_a.p, c->pair_b.p, c->pair_score.p);
        c->end(); LAUNCH_CHECK(c);
        rc = words == 1 ? radix_sort_u64(c, c->keys_a.p, kb2, c->vals_a.p, c->vals_b.p, npairs, L.key_bits, &in_b, "u64")
                        : radix_sort_u128(c, c->keys_a.p, kb2, c->vals_a.p, c->vals_b.p, npairs, L.key_bits, &in_b, "u128");
        if (rc) return rc;
        const uint64_t* skeys = in_b ? kb2 : c->keys_a.p;
        const uint32_t* svals = in_b ? c->vals_b.p : c->vals_a.p;
        c->begin("pair_mark", (double)npairs * (8 * words + 8));
        pair_mark_kernel<<<nblk(npairs, 256), 256, 0, c->stream>>>(npairs, skeys, svals, words, c->pair_a.p, c->pair_b.p, c->pair_score.p,
                                                                  c->qname_off.p, c->qname.p, c->flag.p);
        c->end(); LAUNCH_CHECK(c);
        if (optical) return phase_optical(c, npairs, skeys, svals, words);
    }
    return optical ? phase_optical(c, 0, nullptr, nullptr, 0) : E_OK;
}

int phase_markdup(elp_ctx* c, bool optical) {
    int rc = phase_adapt(c);
    if (rc) return rc;
    // several GPUs (comm.cu): common key ranges, then the visiting mates of cross-group pairs arrive as ghost reads n .. n + n_ghost - 1.
    // Every rank makes the same collective calls in the same order, whatever its own reads look like.
    rc = comm_allreduce_ranges(c);
    if (rc) return rc;
    rc = spread_exchange_begin(c);
    if (rc) return rc;
    const uint64_t n = c->n, nt = n + c->n_ghost;
    const DeviceRanges& R = c->h_ranges;
    int rc_body = E_OK;
    if (nt == 0 || (R.n_entering == 0 && c->n_ghost == 0)) rc_body = optical ? phase_optical(c, 0, nullptr, nullptr, 0) : E_OK;
    else {
        rc_body = [&]() -> int {
            CUDA_TRY(c, c->keys_a.reserve(2 * nt + 4, c->stream)); CUDA_TRY(c, c->keys_b.reserve(2 * nt + 4, c->stream));
            CUDA_TRY(c, c->vals_a.reserve(nt + 4, c->stream)); CUDA_TRY(c, c->vals_b.reserve(nt + 4, c->stream));
            const int bR = bits_for((uint64_t)c->n_contigs), bL = bits_for((uint64_t)c->n_lib + 1);
            const int bU = bits_for((uint64_t)((int64_t)R.upos_max - (int64_t)R.upos_min));
            // both packed key layouts are checked before any marking kernel runs, so that a refusal leaves the FLAG column untouched
            {
                const int frag_bits = bits_for((uint64_t)R.score_max) + 2 + bU + bR + bL, pair_bits = 2 * bU + 2 + 2 * bR + bL;
                if (n && R.n_entering && frag_bits > 64) return c->fail(E_LIMIT, "fragment signature needs %d bits (>64): too many contigs/libraries for the packed key", frag_bits);
                if (pair_bits > 128) return c->fail(E_LIMIT, "pair signature needs %d bits (>128)", pair_bits);
            }
            // ---- fragments (classifyFragment): local reads only ----
            if (n && R.n_entering) {
                FragLayout L{}; L.bS = bits_for((uint64_t)R.score_max); L.bU = bU; L.bR = bR; L.bL = bL; L.upos_min = R.upos_min; L.score_max = R.score_max;
                L.key_bits = L.bS + 2 + L.bU + L.bR + L.bL;
                if (L.key_bits > 64) return c->fail(E_LIMIT, "fragment signature needs %d bits (>64): too many contigs/libraries for the packed key", L.key_bits);
                c->begin("frag_keys", (double)n * (2 + 4 + 4 + 4 + 4 + 8 + 4));
                frag_keys_kernel<<<nblk(n, 256), 256, 0, c->stream>>>(n, c->flag.p, c->refid.p, c->rg.p, c->d_rg_lib, c->n_rg, c->upos.p, c->score.p, L, c->keys_a.p, c->vals_a.p);
                c->end(); LAUNCH_CHECK(c);
                // only the group (bits from bS + 1 up) needs to be contiguous: frag_mark_kernel finds the winner from the low bits
                bool in_b = false;
                int r2 = radix_sort_u64(c, c->keys_a.p, c->keys_b.p, c->vals_a.p, c->vals_b.p, n, L.key_bits - (L.bS + 1), &in_b, "u64", L.bS + 1);
                if (r2) return r2;
                const uint64_t m = R.n_entering;
                c->begin("frag_mark", (double)m * 12);
                frag_mark_kernel<<<nblk(m, 256), 256, 0, c->stream>>>(m, in_b ? c->keys_b.p : c->keys_a.p, in_b ? c->vals_b.p : c->vals_a.p, L.bS, c->qname_off.p, c->qname.p, c->flag.p);
                c->end(); LAUNCH_CHECK(c);
            }
            return mark_pairs(c, optical, nt, (uint64_t)R.n_true_pairs + c->n_ghost, bU, bR, bL);
        }();
    }
    rc = spread_exchange_end(c);       // (also when the body failed: the other ranks are waiting in the same exchange)
    return rc_body ? rc_body : rc;
}
