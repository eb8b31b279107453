// coordsort.cu -- coordinate order on the device (replaces By(CoordinateLess).ParallelStableSort,
// sam/sam-types.go:425-473,599-641, called from the Finalize of (*sam.Sam).AddNodes, sam/filter-pipeline.go:113-117).
//
//  1. radix sort of the compact key (refid with -1 last | POS | strand)           -- the first three comparator clauses
//  2. runs of equal keys are ordered by the remaining clauses (QNAME bytes, modFlag, MAPQ, [NextREFID signed, PNEXT] if
//     both paired, TLEN): short runs by a per-run insertion sort, long runs (e.g. all unmapped reads) by a batched LSD
//     radix sort over 64-bit chunks of the composite secondary key.  Everything is stable: fully equal records keep
//     arrival order.
//  3. the fixed-width columns are gathered into output order once; the byte arenas (QNAME, CIGAR, SEQ, QUAL) stay where
//     they are and are reached through the gathered offsets (the reference sorts pointers, too).
// Deviation (malformed input only): an empty QNAME takes part in the comparison as the smallest string, whereas the
// reference skips the QNAME clause when either name is empty (:439), which is not a strict weak order.
#include "ctx.h"

namespace {

constexpr int SHORT_RUN = 32;

inline unsigned nblk(uint64_t n, int t) { return (unsigned)((n + t - 1) / t); }

struct CoordLayout { int bP, bR; int n_contigs; int key_bits; };

__global__ void __launch_bounds__(256) coord_keys_kernel(uint64_t n, const int32_t* __restrict__ refid, const int32_t* __restrict__ pos, const uint16_t* __restrict__ flag,
                                                          CoordLayout L, uint64_t* __restrict__ keys, uint32_t* __restrict__ vals) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int32_t r = refid[i];
    const uint64_t rr = (r < 0 || r >= L.n_contigs) ? (uint64_t)L.n_contigs : (uint64_t)r;   // refid -1 sorts last (:428-432)
    keys[i] = ((flag[i] & F_REVERSED) ? 1ull : 0ull) | ((uint64_t)(uint32_t)pos[i] << 1) | (rr << (1 + L.bP));
    vals[i] = (uint32_t)i;
}

__device__ __forceinline__ uint16_t mod_flag(uint16_t f) {   // sam-types.go:408-420
    if ((f & F_MULTIPLE) == 0) f &= ~(F_NEXTUNMAPPED | F_NEXTREVERSED);
    if (f & F_UNMAPPED) f &= ~F_REVERSED;
    if (f & F_NEXTUNMAPPED) f &= ~F_NEXTREVERSED;
    return f;
}

struct TieCols {
    const uint16_t* flag; const uint8_t* mapq; const int32_t *nref, *pnext, *tlen; const uint64_t* qname_off; const uint8_t* qname;
};

// the clauses of CoordinateLess after (refid, POS, strand): sam-types.go:439-472
__device__ __forceinline__ bool less2(const TieCols& c, uint32_t a, uint32_t b) {
    const int q = qname_compare(c.qname, c.qname_off[a], c.qname_off[a + 1], c.qname_off[b], c.qname_off[b + 1]);
    if (q) return q < 0;
    const uint16_t fa = c.flag[a], fb = c.flag[b];
    const uint16_t ma = mod_flag(fa), mb = mod_flag(fb);
    if (ma != mb) return ma < mb;
    if (c.mapq[a] != c.mapq[b]) return c.mapq[a] < c.mapq[b];
    if ((fa & F_MULTIPLE) && (fb & F_MULTIPLE)) {
        if (c.nref[a] != c.nref[b]) return c.nref[a] < c.nref[b];   // no special treatment of negative values
        if (c.pnext[a] != c.pnext[b]) return c.pnext[a] < c.pnext[b];
    }
    return c.tlen[a] < c.tlen[b];
}

// one thread per run head: short runs sorted in place, long runs only flagged
__global__ void __launch_bounds__(128) tie_short_kernel(uint64_t n, const uint64_t* __restrict__ keys, uint32_t* __restrict__ vals, TieCols c,
                                                         uint32_t* __restrict__ long_flag /* may be null */, uint32_t* __restrict__ n_long_elems) {
    const uint64_t j = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= n) return;
    const uint64_t k0 = keys[j];
    const bool head = (j == 0) || keys[j - 1] != k0;
    if (long_flag) long_flag[j] = 0;
    if (!head) return;
    uint64_t e = j + 1;
    while (e < n && e - j <= SHORT_RUN && keys[e] == k0) e++;
    const uint64_t t = e - j;
    if (t == 1) return;
    if (t > SHORT_RUN) return;   // flagged by tie_long_flag_kernel
    for (uint64_t x = j + 1; x < e; x++) {   // stable insertion sort
        const uint32_t v = vals[x];
        uint64_t y = x;
        while (y > j && less2(c, v, vals[y - 1])) { vals[y] = vals[y - 1]; y--; }
        vals[y] = v;
    }
}

// chunk key of the composite secondary key; chunk ids (least significant first):
//   0: TLEN   1: NextREFID|PNEXT (0 unless paired)   2: modFlag|MAPQ   3+k: QNAME bytes [8*(nq-1-k), +8) big-endian, zero padded
//   last: the primary coordinate key itself (keeps the runs apart and in place)
__device__ __forceinline__ uint64_t chunk_key(uint32_t a, int chunk, int nq, const TieCols& c, const int32_t* __restrict__ refid, const int32_t* __restrict__ pos,
                                              const CoordLayout& L) {
    uint64_t key;
    if (chunk == 0) key = (uint64_t)((uint32_t)c.tlen[a] ^ 0x80000000u);
    else if (chunk == 1) key = (c.flag[a] & F_MULTIPLE) ? (((uint64_t)((uint32_t)c.nref[a] ^ 0x80000000u) << 32) | (uint64_t)((uint32_t)c.pnext[a] ^ 0x80000000u)) : 0ull;
    else if (chunk == 2) key = ((uint64_t)mod_flag(c.flag[a]) << 8) | c.mapq[a];
    else if (chunk < 3 + nq) {
        const int qc = nq - 1 - (chunk - 3);
        const uint64_t q0 = c.qname_off[a], q1 = c.qname_off[a + 1], lo = q0 + (uint64_t)qc * 8;
        key = 0;
        if (lo < q1) {
            // every load is unconditional and inside the name (index clamped to its last byte); bytes past the end are masked to
            // zero afterwards.  Keep this form: on the H100 the equivalent per-byte form `o < q1 ? qname[o] : 0` gave nonzero key
            // bytes past the end of names shorter than the chunk, in whole warps, and long tie runs came out misordered
            // (tests/test_gpu_parity_large.py).  The two are the same function in C++ and no fault is visible in the SASS of the
            // old form, so what went wrong in its execution is not known.
            const uint64_t avail = q1 - lo;
            for (int b = 0; b < 8; b++) {
                const uint32_t byte = c.qname[min(lo + (uint64_t)b, q1 - 1)];
                key = (key << 8) | ((uint64_t)b < avail ? byte : 0u);
            }
        }
    } else {
        const int32_t r = refid[a];
        const uint64_t rr = (r < 0 || r >= L.n_contigs) ? (uint64_t)L.n_contigs : (uint64_t)r;
        key = ((c.flag[a] & F_REVERSED) ? 1ull : 0ull) | ((uint64_t)(uint32_t)pos[a] << 1) | (rr << (1 + L.bP));
    }
    return key;
}

__global__ void __launch_bounds__(256) chunk_keys_kernel(uint64_t m, const uint32_t* __restrict__ elem, int chunk, int nq, TieCols c,
                                                          const int32_t* __restrict__ refid, const int32_t* __restrict__ pos, CoordLayout L,
                                                          uint64_t* __restrict__ keys, uint32_t* __restrict__ vals) {
    const uint64_t k = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= m) return;
    const uint32_t a = elem[k];
    keys[k] = chunk_key(a, chunk, nq, c, refid, pos, L); vals[k] = a;
}

// flag[j] = 1 if j belongs to a run longer than SHORT_RUN (checked against the element SHORT_RUN places away on either side).
// Over the elements of all long runs, bits[ch] accumulates the OR and bits[n_chunks + ch] the AND of chunk key ch: a bit
// where the two differ is the only kind that can reorder anything in the tie rounds.
__global__ void __launch_bounds__(256) tie_long_flag_kernel(uint64_t n, const uint64_t* __restrict__ keys, const uint32_t* __restrict__ vals, uint32_t* __restrict__ long_flag,
                                                             int n_chunks, int nq, TieCols c, const int32_t* __restrict__ refid, const int32_t* __restrict__ pos,
                                                             CoordLayout L, unsigned long long* __restrict__ bits) {
    extern __shared__ unsigned long long s_bits[];   // [n_chunks] OR, [n_chunks] AND
    unsigned long long *s_or = s_bits, *s_and = s_bits + n_chunks;
    const uint64_t j = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    bool lng = false;
    if (j < n) {
        const uint64_t k0 = keys[j];
        // run length > SHORT_RUN  <=>  some window of SHORT_RUN+1 consecutive equal keys covers j
        uint64_t lo = j, hi = j;
        while (lo > 0 && j - lo < (uint64_t)SHORT_RUN && keys[lo - 1] == k0) lo--;
        while (hi + 1 < n && hi - lo < (uint64_t)SHORT_RUN && keys[hi + 1] == k0) hi++;
        lng = hi - lo >= (uint64_t)SHORT_RUN;
        long_flag[j] = lng ? 1u : 0u;
    }
    if (!__syncthreads_or(lng)) return;
    for (int ch = threadIdx.x; ch < n_chunks; ch += blockDim.x) { s_or[ch] = 0; s_and[ch] = ~0ull; }
    __syncthreads();
    const uint32_t a = lng ? vals[j] : 0u;
    const unsigned lane = threadIdx.x & 31;
    for (int ch = 0; ch < n_chunks; ch++) {
        const uint64_t k = lng ? chunk_key(a, ch, nq, c, refid, pos, L) : 0ull;
        uint64_t o = k, an = lng ? k : ~0ull;
        for (int d = 16; d; d >>= 1) { o |= __shfl_xor_sync(FULL_MASK, o, d); an &= __shfl_xor_sync(FULL_MASK, an, d); }
        if (lane == 0) { atomicOr(&s_or[ch], (unsigned long long)o); atomicAnd(&s_and[ch], (unsigned long long)an); }
    }
    __syncthreads();
    for (int ch = threadIdx.x; ch < n_chunks; ch += blockDim.x) { atomicOr(bits + ch, s_or[ch]); atomicAnd(bits + n_chunks + ch, s_and[ch]); }
}

__global__ void __launch_bounds__(256) compact_long_kernel(uint64_t n, const uint32_t* __restrict__ long_flag, const uint64_t* __restrict__ slot,
                                                            const uint32_t* __restrict__ vals, uint32_t* __restrict__ pos_list, uint32_t* __restrict__ elem) {
    const uint64_t j = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= n || !long_flag[j]) return;
    const uint64_t s = slot[j];
    pos_list[s] = (uint32_t)j; elem[s] = vals[j];
}

__global__ void __launch_bounds__(256) scatter_long_kernel(uint64_t m, const uint32_t* __restrict__ pos_list, const uint32_t* __restrict__ sorted_elem, uint32_t* __restrict__ vals) {
    const uint64_t k = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (k < m) vals[pos_list[k]] = sorted_elem[k];
}

__global__ void __launch_bounds__(256) iota_kernel(uint64_t n, uint32_t* __restrict__ v) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) v[i] = (uint32_t)i;
}

struct GatherCols {
    const int32_t *refid, *pos, *nref, *pnext, *tlen, *rg; const uint16_t* flag; const uint8_t* mapq;
    const uint64_t *qual_off, *seq_off, *cigar_off;
    int32_t *s_refid, *s_pos, *s_nref, *s_pnext, *s_tlen, *s_rg, *s_lseq; uint16_t* s_flag; uint8_t* s_mapq;
    uint64_t *s_qual_off, *s_seq_off, *s_cigar_off; uint32_t* s_ncigar;
    const uint8_t* optf; uint8_t* s_optf;
};

// The fixed-width columns of a read packed into one 64-byte row (streaming pass, coalesced), so that the permuted gather below
// touches two sectors per read instead of eleven:
//   u32[0..5] refid pos nref pnext tlen rg   [6] lseq  [7] ncigar  [8,9] qual_off  [10,11] seq_off  [12,13] cigar_off  [14] mapq
__global__ void __launch_bounds__(256) pack_rows_kernel(uint64_t n, GatherCols g, uint4* __restrict__ rows) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint64_t q0 = g.qual_off[i], q1 = g.qual_off[i + 1], c0 = g.cigar_off[i], c1 = g.cigar_off[i + 1], s0 = g.seq_off[i];
    uint4* r = rows + 4 * i;
    r[0] = make_uint4((uint32_t)g.refid[i], (uint32_t)g.pos[i], (uint32_t)g.nref[i], (uint32_t)g.pnext[i]);
    r[1] = make_uint4((uint32_t)g.tlen[i], (uint32_t)g.rg[i], (uint32_t)(q1 - q0), (uint32_t)(c1 - c0));
    r[2] = make_uint4((uint32_t)q0, (uint32_t)(q0 >> 32), (uint32_t)s0, (uint32_t)(s0 >> 32));
    r[3] = make_uint4((uint32_t)c0, (uint32_t)(c0 >> 32), (uint32_t)g.mapq[i], (uint32_t)g.optf[i]);
}

__global__ void __launch_bounds__(256) gather_cols_kernel(uint64_t n, const uint32_t* __restrict__ perm, GatherCols g, const uint4* __restrict__ rows) {
    const uint64_t k = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= n) return;
    const uint32_t i = perm[k];
    const uint4* r = rows + 4 * (uint64_t)i;
    const uint4 a = __ldg(r), b = __ldg(r + 1), c = __ldg(r + 2), d = __ldg(r + 3);
    g.s_refid[k] = (int32_t)a.x; g.s_pos[k] = (int32_t)a.y; g.s_nref[k] = (int32_t)a.z; g.s_pnext[k] = (int32_t)a.w; g.s_tlen[k] = (int32_t)b.x; g.s_rg[k] = (int32_t)b.y;
    g.s_flag[k] = g.flag[i];                       // FLAG from the column: duplicate marking set bits after the rows were packed
    g.s_mapq[k] = (uint8_t)d.z; g.s_optf[k] = (uint8_t)d.w;
    g.s_qual_off[k] = ((uint64_t)c.y << 32) | c.x; g.s_lseq[k] = (int32_t)b.z; g.s_seq_off[k] = ((uint64_t)c.w << 32) | c.z;
    g.s_cigar_off[k] = ((uint64_t)d.y << 32) | d.x; g.s_ncigar[k] = b.w;
}

__global__ void __launch_bounds__(256) lseq_u32_kernel(uint64_t n, const int32_t* __restrict__ lseq, uint32_t* __restrict__ out) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) out[i] = (uint32_t)lseq[i];
}

}  // namespace

int phase_coordinate_sort(elp_ctx* c, int order) {   // 0 keep, 1 coordinate, 2 queryname
    const bool sort = order == 1;
    const uint64_t n = c->n;
    int rc = phase_adapt(c);   // value ranges (pos_max) size the key
    if (rc) return rc;
    CUDA_TRY(c, c->perm.reserve(n + 4, c->stream));
    if (sort && n > 1) {
        CUDA_TRY(c, c->keys_a.reserve(2 * n + 4, c->stream)); CUDA_TRY(c, c->keys_b.reserve(2 * n + 4, c->stream));
        CUDA_TRY(c, c->vals_a.reserve(n + 4, c->stream)); CUDA_TRY(c, c->vals_b.reserve(n + 4, c->stream));
        CoordLayout L{}; L.n_contigs = c->n_contigs; L.bP = bits_for((uint64_t)c->h_ranges.pos_max); L.bR = bits_for((uint64_t)c->n_contigs);
        L.key_bits = 1 + L.bP + L.bR;
        c->begin("coord_keys", (double)n * (4 + 4 + 2 + 8 + 4));
        coord_keys_kernel<<<nblk(n, 256), 256, 0, c->stream>>>(n, c->refid.p, c->pos.p, c->flag.p, L, c->keys_a.p, c->vals_a.p);
        c->end(); LAUNCH_CHECK(c);
        bool in_b = false;
        rc = radix_sort_u64(c, c->keys_a.p, c->keys_b.p, c->vals_a.p, c->vals_b.p, n, L.key_bits, &in_b, "u64");
        if (rc) return rc;
        uint64_t* keys = in_b ? c->keys_b.p : c->keys_a.p;
        uint32_t* vals = in_b ? c->vals_b.p : c->vals_a.p;
        uint64_t* keys_free = in_b ? c->keys_a.p : c->keys_b.p;

        TieCols tc{c->flag.p, c->mapq.p, c->nref.p, c->pnext.p, c->tlen.p, c->qname_off.p, c->qname.p};
        const int nq = std::max(1, (int)((c->h_ranges.qname_max + 7) / 8));   // longest QNAME, from the adapt kernel's range reduction
        const int n_chunks = 3 + nq + 1;
        // long runs first (flags computed from the keys only), then short runs in place
        CUDA_TRY(c, c->scan_tmp.reserve(n + 4, c->stream));
        CUDA_TRY(c, c->tie_bits.reserve(2 * n_chunks, c->stream));
        CUDA_TRY(c, cudaMemsetAsync(c->tie_bits.p, 0, n_chunks * 8, c->stream));
        CUDA_TRY(c, cudaMemsetAsync(c->tie_bits.p + n_chunks, 0xff, n_chunks * 8, c->stream));
        c->begin("tie_long_flag", (double)n * 12);
        tie_long_flag_kernel<<<nblk(n, 256), 256, 2 * n_chunks * 8, c->stream>>>(n, keys, vals, c->scan_tmp.p, n_chunks, nq, tc, c->refid.p, c->pos.p, L,
                                                                  reinterpret_cast<unsigned long long*>(c->tie_bits.p));
        c->end(); LAUNCH_CHECK(c);
        uint64_t* slot = keys_free;   // n+1 u64
        rc = exclusive_scan_u32_to_u64(c, c->scan_tmp.p, slot, n);
        if (rc) return rc;
        uint64_t m = 0;
        std::vector<uint64_t> tie_bits(2 * n_chunks);
        CUDA_TRY(c, cudaMemcpyAsync(&m, slot + n, 8, cudaMemcpyDeviceToHost, c->stream));
        CUDA_TRY(c, cudaMemcpyAsync(tie_bits.data(), c->tie_bits.p, tie_bits.size() * 8, cudaMemcpyDeviceToHost, c->stream));
        CUDA_TRY(c, cudaStreamSynchronize(c->stream));
        c->begin("tie_short", (double)n * 12);
        tie_short_kernel<<<nblk(n, 128), 128, 0, c->stream>>>(n, keys, vals, tc, nullptr, nullptr);
        c->end(); LAUNCH_CHECK(c);
        if (m > 0) {
            // batched LSD sort of all long-run elements over the chunks of the secondary key
            CUDA_TRY(c, c->pair_a.reserve(m + 4, c->stream)); CUDA_TRY(c, c->pair_b.reserve(m + 4, c->stream));
            uint32_t* pos_list = c->pair_a.p; uint32_t* elem = c->pair_b.p;
            c->begin("tie_compact", (double)n * 16);
            compact_long_kernel<<<nblk(n, 256), 256, 0, c->stream>>>(n, c->scan_tmp.p, slot, vals, pos_list, elem);
            c->end(); LAUNCH_CHECK(c);
            CUDA_TRY(c, c->bytes_tmp.reserve((size_t)m * 16 + 64, c->stream));
            uint64_t* ka = reinterpret_cast<uint64_t*>(c->bytes_tmp.p);
            uint64_t* kb = ka + m;
            CUDA_TRY(c, c->mate.reserve(2 * m + 16, c->stream));
            uint32_t* va = c->mate.p; uint32_t* vb = c->mate.p + ((m + 3) & ~(uint64_t)3);   // 16-byte aligned: the sort stages payloads with 16-byte async copies
            for (int ch = 0; ch < n_chunks; ch++) {
                // a chunk whose bits are equal on every long-run element cannot reorder anything: skip it; sort the others only over
                // the range from their lowest to their highest differing bit
                const uint64_t diff = tie_bits[ch] ^ tie_bits[n_chunks + ch];
                if (diff == 0) continue;
                const int lo_bit = __builtin_ctzll(diff), hi_bit = 63 - __builtin_clzll(diff);
                c->begin("tie_chunk_keys", (double)m * 32);
                chunk_keys_kernel<<<nblk(m, 256), 256, 0, c->stream>>>(m, elem, ch, nq, tc, c->refid.p, c->pos.p, L, ka, va);
                c->end(); LAUNCH_CHECK(c);
                bool b2 = false;
                rc = radix_sort_u64(c, ka, kb, va, vb, m, hi_bit - lo_bit + 1, &b2, "u64", lo_bit);
                if (rc) return rc;
                CUDA_TRY(c, cudaMemcpyAsync(elem, b2 ? vb : va, m * 4, cudaMemcpyDeviceToDevice, c->stream));
            }
            c->begin("tie_scatter", (double)m * 12);
            scatter_long_kernel<<<nblk(m, 256), 256, 0, c->stream>>>(m, pos_list, elem, vals);
            c->end(); LAUNCH_CHECK(c);
        }
        CUDA_TRY(c, cudaMemcpyAsync(c->perm.p, vals, n * 4, cudaMemcpyDeviceToDevice, c->stream));

    } else if (order == 2 && n > 1) {
        // By(QNAMELess).ParallelStableSort (sam/sam-types.go:479-481, sam/filter-pipeline.go:119-123): stable LSD radix sort over
        // 8-byte big-endian chunks of the QNAME, last chunk first (names are zero padded: a prefix sorts before its extensions)
        CUDA_TRY(c, c->keys_a.reserve(2 * n + 4, c->stream)); CUDA_TRY(c, c->keys_b.reserve(2 * n + 4, c->stream));
        CUDA_TRY(c, c->vals_a.reserve(n + 4, c->stream)); CUDA_TRY(c, c->vals_b.reserve(n + 4, c->stream));
        TieCols tc{c->flag.p, c->mapq.p, c->nref.p, c->pnext.p, c->tlen.p, c->qname_off.p, c->qname.p};
        CoordLayout L{};
        const int nq = std::max(1, (int)((c->h_ranges.qname_max + 7) / 8));
        iota_kernel<<<nblk(n, 256), 256, 0, c->stream>>>(n, c->vals_a.p); c->launches++; LAUNCH_CHECK(c);
        const uint32_t* elem = c->vals_a.p;
        for (int ch = 0; ch < nq; ch++) {
            c->begin("qname_chunk_keys", (double)n * 32);
            chunk_keys_kernel<<<nblk(n, 256), 256, 0, c->stream>>>(n, elem, 3 + ch, nq, tc, c->refid.p, c->pos.p, L, c->keys_a.p, c->vals_a.p);
            c->end(); LAUNCH_CHECK(c);
            bool b2 = false;
            rc = radix_sort_u64(c, c->keys_a.p, c->keys_b.p, c->vals_a.p, c->vals_b.p, n, 64, &b2, "u64");
            if (rc) return rc;
            elem = b2 ? c->vals_b.p : c->vals_a.p;
        }
        CUDA_TRY(c, cudaMemcpyAsync(c->perm.p, elem, n * 4, cudaMemcpyDeviceToDevice, c->stream));
    } else if (n) {
        iota_kernel<<<nblk(n, 256), 256, 0, c->stream>>>(n, c->perm.p);
        c->launches++; LAUNCH_CHECK(c);
    }
    // gather the fixed-width columns into output order
    CUDA_TRY(c, c->s_refid.reserve(n + 4, c->stream)); CUDA_TRY(c, c->s_pos.reserve(n + 4, c->stream)); CUDA_TRY(c, c->s_nref.reserve(n + 4, c->stream));
    CUDA_TRY(c, c->s_pnext.reserve(n + 4, c->stream)); CUDA_TRY(c, c->s_tlen.reserve(n + 4, c->stream)); CUDA_TRY(c, c->s_rg.reserve(n + 4, c->stream));
    CUDA_TRY(c, c->s_lseq.reserve(n + 4, c->stream)); CUDA_TRY(c, c->s_flag.reserve(n + 4, c->stream)); CUDA_TRY(c, c->s_mapq.reserve(n + 4, c->stream)); CUDA_TRY(c, c->s_optf.reserve(n + 4, c->stream));
    CUDA_TRY(c, c->s_qual_off.reserve(n + 4, c->stream)); CUDA_TRY(c, c->s_seq_off.reserve(n + 4, c->stream)); CUDA_TRY(c, c->s_cigar_off.reserve(n + 4, c->stream));
    CUDA_TRY(c, c->s_ncigar.reserve(n + 4, c->stream)); CUDA_TRY(c, c->s_out_off.reserve(n + 4, c->stream));
    if (n) {
        GatherCols g{c->refid.p, c->pos.p, c->nref.p, c->pnext.p, c->tlen.p, c->rg.p, c->flag.p, c->mapq.p, c->qual_off.p, c->seq_off.p, c->cigar_off.p,
                     c->s_refid.p, c->s_pos.p, c->s_nref.p, c->s_pnext.p, c->s_tlen.p, c->s_rg.p, c->s_lseq.p, c->s_flag.p, c->s_mapq.p,
                     c->s_qual_off.p, c->s_seq_off.p, c->s_cigar_off.p, c->s_ncigar.p, c->optf.p, c->s_optf.p};
        // rows live in the key scratch (free here): 4 x uint4 per read
        CUDA_TRY(c, c->keys_a.reserve(8 * n + 8, c->stream));
        uint4* rows = reinterpret_cast<uint4*>(c->keys_a.p);
        c->begin("pack_rows", (double)n * (27 + 24 + 64));
        pack_rows_kernel<<<nblk(n, 256), 256, 0, c->stream>>>(n, g, rows);
        c->end(); LAUNCH_CHECK(c);
        c->begin("gather_cols", (double)n * (4 + 27 + 24 + 27 + 28 + 8));
        gather_cols_kernel<<<nblk(n, 256), 256, 0, c->stream>>>(n, c->perm.p, g, rows);
        c->end(); LAUNCH_CHECK(c);
        CUDA_TRY(c, c->scan_tmp.reserve(n + 4, c->stream));
        lseq_u32_kernel<<<nblk(n, 256), 256, 0, c->stream>>>(n, c->s_lseq.p, c->scan_tmp.p);
        c->launches++; LAUNCH_CHECK(c);
    }
    rc = exclusive_scan_u32_to_u64(c, c->scan_tmp.p, c->s_out_off.p, n);
    if (rc) return rc;
    c->sorted = true;
    c->qual_out_valid = false;
    return E_OK;
}
