// cleansam.cu -- filters.CleanSam (filters/simple-filters.go:292-306) on the device columns: MAPQ of unmapped reads becomes 0, and a mapped read
// whose alignment runs past the end of its contig has its CIGAR soft-clipped there by softClipEndOfRead / elementStradlessClippedRead
// (filters/utils.go:82-119) -- restated operation by operation, including the reference's own arithmetic (`pos += endPos`, the clipped length
// `ReadLengthFromCigar + clipFrom`): its results are the specification.  The CIGAR arena is packed, so a rewrite that changes operation
// counts re-packs it: count -> prefix sum -> write.
#include "../../include/elprep_b200.h"
#include "ctx.h"

namespace {

inline unsigned nblk(uint64_t n, int t) { return (unsigned)((n + t - 1) / t); }
__device__ __forceinline__ int cons_read(uint32_t o) { return o == 0 || o == 1 || o == 4 || o == 7 || o == 8; }
__device__ __forceinline__ int cons_ref(uint32_t o) { return o == 0 || o == 2 || o == 3 || o == 7 || o == 8; }
// int32 addition as Go does it: wraps (`pos += endPos` doubles pos, so a long CIGAR overflows it)
__device__ __forceinline__ int32_t wadd(int32_t a, int32_t b) { return (int32_t)((uint32_t)a + (uint32_t)b); }
__device__ __forceinline__ int32_t wsub(int32_t a, int32_t b) { return (int32_t)((uint32_t)a - (uint32_t)b); }

// walks one read; out == nullptr: only counts.  returns the new number of operations, or -1 if the read keeps its CIGAR
__device__ int clean_one(const uint32_t* __restrict__ cg, int nc, int32_t pos, int32_t refid, uint16_t flag, const int32_t* __restrict__ contig_len, int n_contigs,
                         uint32_t* __restrict__ out, uint32_t* __restrict__ err) {
    if (flag & F_UNMAPPED) return -1;
    const int32_t length = (refid >= 0 && refid < n_contigs) ? contig_len[refid] : 0;       // referenceSequenceTable[aln.RNAME]: 0 for a name that is not an @SQ
    int32_t reflen = 0, readlen = 0;
    for (int i = 0; i < nc; i++) { const uint32_t o = cg[i] & 15u; const int32_t l = (int32_t)(cg[i] >> 4); reflen = wadd(reflen, cons_ref(o) * l); readlen = wadd(readlen, cons_read(o) * l); }
    if (!(wsub(wadd(pos, reflen), 1) > length)) return -1;                                     // aln.End() > length
    int32_t clipFrom = wadd(wsub(length, pos), 1);
    // softClipEndOfRead
    int32_t p = 0; clipFrom = wsub(clipFrom, 1);
    int no = 0;
    for (int i = 0; i < nc; i++) {
        const uint32_t o = cg[i] & 15u; const int32_t l = (int32_t)(cg[i] >> 4);
        const int32_t endPos = wadd(p, cons_read(o) * l);
        if (endPos < clipFrom) { if (out) out[no] = cg[i]; no++; }
        else {
            int32_t clipped = wadd(readlen, clipFrom);
            const int32_t rel = wsub(clipFrom, p);
            // elementStradlessClippedRead
            if (cons_read(o)) {
                if (cons_ref(o)) { if (rel > 0) { if (out) out[no] = ((uint32_t)rel << 4) | o; no++; } }
                else clipped = wadd(clipped, rel);
            } else if (rel != 0) atomicOr(err, DERR_CLEANSAM);
            if (out) out[no] = ((uint32_t)clipped << 4) | 4u;
            no++;
            break;
        }
        p = wadd(p, endPos);
    }
    return no;
}

__global__ void __launch_bounds__(256) clean_count_kernel(uint64_t n, const uint16_t* __restrict__ flag, uint8_t* __restrict__ mapq, const int32_t* __restrict__ refid, const int32_t* __restrict__ pos,
                                                           const uint64_t* __restrict__ cigar_off, const uint32_t* __restrict__ cigar, const int32_t* __restrict__ contig_len, int n_contigs,
                                                           uint32_t* __restrict__ newcnt, uint32_t* __restrict__ n_changed, uint32_t* __restrict__ err) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint16_t f = flag[i];
    if (f & F_UNMAPPED) mapq[i] = 0;
    const uint64_t c0 = cigar_off[i]; const int nc = (int)(cigar_off[i + 1] - c0);
    const int k = clean_one(cigar + c0, nc, pos[i], refid[i], f, contig_len, n_contigs, nullptr, err);
    newcnt[i] = k < 0 ? (uint32_t)nc : (uint32_t)k;
    if (k >= 0) atomicAdd(n_changed, 1u);
}
__global__ void __launch_bounds__(256) clean_write_kernel(uint64_t n, const uint16_t* __restrict__ flag, const int32_t* __restrict__ refid, const int32_t* __restrict__ pos,
                                                           const uint64_t* __restrict__ cigar_off, const uint32_t* __restrict__ cigar, const int32_t* __restrict__ contig_len, int n_contigs,
                                                           const uint64_t* __restrict__ new_off, uint32_t* __restrict__ out, uint32_t* __restrict__ err) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint64_t c0 = cigar_off[i]; const int nc = (int)(cigar_off[i + 1] - c0);
    uint32_t* o = out + new_off[i];
    if (clean_one(cigar + c0, nc, pos[i], refid[i], flag[i], contig_len, n_contigs, o, err) < 0) for (int k = 0; k < nc; k++) o[k] = cigar[c0 + k];
}

}  // namespace

extern "C" int elp_clean_sam(elp_ctx* c, uint64_t* n_rewritten) {
    if (!c) return ELP_EINVAL;
    cudaSetDevice(c->device);
    if (c->sorted) return c->fail(E_STATE, "elp_clean_sam after elp_sort_markdup");
    if (n_rewritten) *n_rewritten = 0;
    const uint64_t n = c->n;
    if (!n) return ELP_OK;
    cudaStream_t s = c->stream;
    CUDA_TRY(c, c->scan_tmp.reserve(n + 8, s));
    uint32_t* d_changed = c->scan_tmp.p + n + 4;
    CUDA_TRY(c, cudaMemsetAsync(d_changed, 0, 4, s));
    c->begin("clean_sam_count", (double)n * 19 + (double)c->n_cigar * 4);
    clean_count_kernel<<<nblk(n, 256), 256, 0, s>>>(n, c->flag.p, c->mapq.p, c->refid.p, c->pos.p, c->cigar_off.p, c->cigar.p, c->d_contig_len, c->n_contigs, c->scan_tmp.p, d_changed, c->d_err);
    c->end(); LAUNCH_CHECK(c);
    uint32_t changed = 0;
    CUDA_TRY(c, cudaMemcpyAsync(&changed, d_changed, 4, cudaMemcpyDeviceToHost, s));
    int rc = check_device_errors(c);   // synchronizes
    if (rc) return rc;
    if (n_rewritten) *n_rewritten = changed;
    if (!changed) return ELP_OK;
    // re-pack the arena
    DBuf<uint64_t> new_off; DBuf<uint32_t> new_cigar;
    CUDA_TRY(c, new_off.reserve(n + 2, s));
    rc = exclusive_scan_u32_to_u64(c, c->scan_tmp.p, new_off.p, n);
    if (rc) { new_off.release(); return rc; }
    uint64_t total = 0;
    CUDA_TRY(c, cudaMemcpyAsync(&total, new_off.p + n, 8, cudaMemcpyDeviceToHost, s));
    CUDA_TRY(c, cudaStreamSynchronize(s));
    CUDA_TRY(c, new_cigar.reserve(std::max<uint64_t>(total + 16, c->cigar.cap), s));
    c->begin("clean_sam_write", (double)n * 26 + (double)c->n_cigar * 8);
    clean_write_kernel<<<nblk(n, 256), 256, 0, s>>>(n, c->flag.p, c->refid.p, c->pos.p, c->cigar_off.p, c->cigar.p, c->d_contig_len, c->n_contigs, new_off.p, new_cigar.p, c->d_err);
    c->end(); LAUNCH_CHECK(c);
    CUDA_TRY(c, cudaStreamSynchronize(s));
    std::swap(c->cigar.p, new_cigar.p); std::swap(c->cigar.cap, new_cigar.cap);
    std::swap(c->cigar_off.p, new_off.p); std::swap(c->cigar_off.cap, new_off.cap);
    new_cigar.release(); new_off.release();
    c->n_cigar = total; c->n_cleaned += changed; c->adapted = false;
    return ELP_OK;
}

// arrival-order CIGARs as the context now holds them (parity tests of elp_clean_sam): cigar_off[n+1] relative to the first operation, then the operations
extern "C" int elp_debug_cigar(elp_ctx* c, uint64_t* cigar_off, uint32_t* cigar, uint64_t capacity) {
    if (!c || !cigar_off) return ELP_EINVAL;
    cudaSetDevice(c->device);
    const uint64_t n = c->n;
    CUDA_TRY(c, cudaMemcpyAsync(cigar_off, c->cigar_off.p, (n + 1) * 8, cudaMemcpyDeviceToHost, c->stream));
    CUDA_TRY(c, cudaStreamSynchronize(c->stream));
    const uint64_t base = cigar_off[0], total = cigar_off[n] - base;
    for (uint64_t i = 0; i <= n; i++) cigar_off[i] -= base;
    if (total > capacity) return c->fail(E_INVAL, "elp_debug_cigar: %llu operations, capacity %llu", (unsigned long long)total, (unsigned long long)capacity);
    if (cigar && total) { CUDA_TRY(c, cudaMemcpyAsync(cigar, c->cigar.p + base, total * 4, cudaMemcpyDeviceToHost, c->stream)); CUDA_TRY(c, cudaStreamSynchronize(c->stream)); }
    return ELP_OK;
}
