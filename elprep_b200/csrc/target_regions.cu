// target_regions.cu -- `--target-regions` of `elprep filter ... --bqsr`: RemoveNonOverlappingReads (filters/simple-filters.go:308-328) over
// the reads in output order, after duplicate marking and the duplication metrics and before the BQSR gather
// (runBestPracticesPipelineIntermediateSam, cmd/filter.go:171-180; the tables-only worker, :288-296).
//
//   target_keep      one thread per output record: keep flag of intervals.Overlap(ivals[RNAME], POS, alnEnd), warp-aggregated kept count
//   (scan)           exclusive_scan_u32_to_u64 of the flags
//   target_compact   perm compacted in order into the sort scratch, which then becomes perm
//   target_pack_rows, target_gather_cols   the output-order columns rebuilt from the compacted perm (build_output_columns, coordsort.cu)
//   target_summary   over the kept reads: the longest read and the QUAL presence bitmap, which pick the gather and apply kernels
// Nothing runs after the predicate when every read is kept.
#include <algorithm>
#include <utility>
#include "../../include/elprep_b200.h"
#include "ctx.h"
#include "regions.cuh"

namespace {

// alnStart = POS; alnEnd = End() for a mapped read whose CIGAR has read bases, else POS (:318-324).  The sums are Go's int32 sums: they wrap.
__global__ void __launch_bounds__(256) target_keep_kernel(uint64_t n, const int32_t* __restrict__ refid, const int32_t* __restrict__ pos, const uint16_t* __restrict__ flag,
                                                           const uint64_t* __restrict__ cigar_off, const uint32_t* __restrict__ ncigar, const uint32_t* __restrict__ cigar,
                                                           const int32_t* const* __restrict__ regions, const uint64_t* __restrict__ n_regions, int n_contigs,
                                                           uint32_t* __restrict__ keep, unsigned long long* __restrict__ n_keep) {
    const uint64_t k = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    bool kp = false;
    if (k < n) {
        const int32_t r = refid[k], p = pos[k];
        int32_t a_end = p;
        if (!(flag[k] & F_UNMAPPED)) {
            const uint32_t* cg = cigar + cigar_off[k];
            const uint32_t nc = ncigar[k];
            uint32_t rl = 0, fl = 0;
            for (uint32_t q = 0; q < nc; q++) {
                const uint32_t op = cg[q], o = op & 15u, ln = op >> 4;
                if (o == 0 || o == 1 || o == 4 || o == 7 || o == 8) rl += ln;
                if (o == 0 || o == 2 || o == 3 || o == 7 || o == 8) fl += ln;
            }
            if ((int32_t)rl > 0) a_end = (int32_t)((uint32_t)p + fl - 1u);   // aln.End(), sam/sam-types.go:769-775
        }
        kp = r >= 0 && r < n_contigs && overlap_any(regions[r], n_regions[r], p, a_end);   // RNAME * and contigs without regions: Overlap(nil) is false
        keep[k] = kp ? 1u : 0u;
    }
    const unsigned b = __ballot_sync(FULL_MASK, kp);
    if ((threadIdx.x & 31) == 0 && b) atomicAdd(n_keep, (unsigned long long)__popc(b));
}

__global__ void __launch_bounds__(256) target_compact_kernel(uint64_t n, const uint32_t* __restrict__ keep, const uint64_t* __restrict__ slot, const uint32_t* __restrict__ perm,
                                                              uint32_t* __restrict__ out) {
    const uint64_t k = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (k < n && keep[k]) out[slot[k]] = perm[k];
}

// one warp per kept read (grid-stride): the longest read and which QUAL values occur, in the bitmap layout of qual_presence_kernel (api.cu)
__global__ void __launch_bounds__(256) target_summary_kernel(uint64_t n, const int32_t* __restrict__ lseq, const uint64_t* __restrict__ qual_off, const uint8_t* __restrict__ qual,
                                                              uint32_t* __restrict__ present, int32_t* __restrict__ lseq_max) {
    unsigned long long lo = 0, hi = 0;
    uint32_t other = 0;
    int32_t lm = 0;
    const unsigned lane = threadIdx.x & 31;
    const uint64_t w0 = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5, nw = ((uint64_t)gridDim.x * blockDim.x) >> 5;
    for (uint64_t k = w0; k < n; k += nw) {
        const int32_t L = lseq[k];
        lm = max(lm, L);
        const uint8_t* q = qual + qual_off[k];
        for (int32_t i = (int32_t)lane; i < L; i += 32) { const uint32_t v = q[i]; lo |= 1ull << v; hi |= 1ull << (v - 64u); other |= v & 0x80u; }   // shifts >= 64 give 0
    }
    for (int o = 16; o; o >>= 1) { lo |= __shfl_xor_sync(FULL_MASK, lo, o); hi |= __shfl_xor_sync(FULL_MASK, hi, o); other |= __shfl_xor_sync(FULL_MASK, other, o); }
    if (lane == 0) {
        if ((uint32_t)lo) atomicOr(present, (uint32_t)lo);
        if ((uint32_t)(lo >> 32)) atomicOr(present + 1, (uint32_t)(lo >> 32));
        if ((uint32_t)hi) atomicOr(present + 2, (uint32_t)hi);
        if ((uint32_t)(hi >> 32) || other) atomicOr(present + 3, (uint32_t)(hi >> 32) | (other ? 0x80000000u : 0u));   // bit 127: some byte >= 128
        if (lm) atomicMax(lseq_max, lm);
    }
}

}  // namespace

int phase_target_filter(elp_ctx* c, uint64_t* n_removed) {
    if (!c->sorted) return c->fail(E_STATE, "elp_filter_target_regions before elp_sort_markdup (the reads are filtered after duplicate marking)");
    if (c->gathered) return c->fail(E_STATE, "elp_filter_target_regions after elp_bqsr_gather, elp_bqsr_tables_put or elp_bqsr_apply (the filter runs before the BQSR gather)");
    const uint64_t n = c->n_sorted;
    uint64_t kept = n;
    if (n) {
        cudaStream_t s = c->stream;
        TRY(table_upload(c, c->bqsr_regions));
        TRY(grow(c, c->scan_tmp, n + 8));
        // the kept count lives in the BQSR gather's small words (cleared by the gather before its own use)
        unsigned long long* d_kept = reinterpret_cast<unsigned long long*>(c->d_bq_small.p);
        CUDA_TRY(c, cudaMemsetAsync(d_kept, 0, 8, s));
        const double cigar_bytes = 4.0 * (double)c->n_cigar * (double)n / (double)std::max<uint64_t>(c->n, 1);
        c->begin("target_keep", (double)n * (4 + 4 + 2 + 8 + 4 + 4) + cigar_bytes);
        target_keep_kernel<<<nblk(n, 256), 256, 0, s>>>(n, c->s_refid.p, c->s_pos.p, c->s_flag.p, c->s_cigar_off.p, c->s_ncigar.p, c->cigar.p,
                                                         c->bqsr_regions.d_ptrs.p, c->bqsr_regions.d_n.p, c->n_contigs, c->scan_tmp.p, d_kept);
        c->end(); LAUNCH_CHECK(c);
        unsigned long long hk = 0;
        CUDA_TRY(c, cudaMemcpyAsync(&hk, d_kept, 8, cudaMemcpyDeviceToHost, s));
        CUDA_TRY(c, cudaStreamSynchronize(s));
        kept = hk;
        if (kept < n) {
            TRY(grow(c, c->keys_b, n + 2)); TRY(grow(c, c->vals_a, n + 4));
            TRY(exclusive_scan_u32_to_u64(c, c->scan_tmp.p, c->keys_b.p, n));
            c->begin("target_compact", (double)n * (4 + 8 + 4) + 4.0 * (double)kept);
            target_compact_kernel<<<nblk(n, 256), 256, 0, s>>>(n, c->scan_tmp.p, c->keys_b.p, c->perm.p, c->vals_a.p);
            c->end(); LAUNCH_CHECK(c);
            std::swap(c->perm, c->vals_a);   // the compacted order becomes perm; the old one is sort scratch from here on
            TRY(build_output_columns(c, c->perm.p, kept, true));
            // whole-context summaries the BQSR phases choose kernels and table sizes by, now over the kept reads: lseq_max (h_ranges, which
            // phase_adapt keeps while `adapted` holds: no read can be appended after the sort) and the QUAL presence bitmap
            CUDA_TRY(c, cudaMemsetAsync(c->d_qpresent.p, 0, 16, s));
            CUDA_TRY(c, cudaMemsetAsync(&c->d_ranges.p->lseq_max, 0, 4, s));
            if (kept) {
                int sms = 132; cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, c->device);
                const double qual_bytes = (double)(c->n_qual - ARENA_FRONT_PAD) * (double)kept / (double)std::max<uint64_t>(c->n, 1);
                c->begin("target_summary", (double)kept * (4 + 8) + qual_bytes);
                target_summary_kernel<<<(unsigned)std::min<uint64_t>(nblk(kept * 32, 256), (uint64_t)sms * 16), 256, 0, s>>>(kept, c->s_lseq.p, c->s_qual_off.p, c->qual.p,
                                                                                                                      c->d_qpresent.p, &c->d_ranges.p->lseq_max);
                c->end(); LAUNCH_CHECK(c);
            }
            int32_t lm = 0;
            CUDA_TRY(c, cudaMemcpyAsync(&lm, &c->d_ranges.p->lseq_max, 4, cudaMemcpyDeviceToHost, s));
            CUDA_TRY(c, cudaMemcpyAsync(c->h_qpresent, c->d_qpresent.p, 16, cudaMemcpyDeviceToHost, s));
            CUDA_TRY(c, cudaStreamSynchronize(s));
            c->h_ranges.lseq_max = lm;
            c->n_sorted = kept;
            c->out_sel_valid = false;      // the record filters' selection indexes the old order
            c->qual_out_valid = false;     // so does the materialised QUAL stream
        }
    }
    if (n_removed) *n_removed = n - kept;
    return E_OK;
}

extern "C" {

int elp_set_bqsr_target_regions(elp_ctx* c, int32_t contig, const int32_t* se, uint64_t n_intervals, int already_flat) {
    if (!c) return ELP_EINVAL;
    cudaSetDevice(c->device);
    return region_set(c, c->bqsr_regions, "elp_set_bqsr_target_regions", contig, se, n_intervals, already_flat);
}

int elp_filter_target_regions(elp_ctx* c, uint64_t* n_removed) {
    if (!c) return ELP_EINVAL;
    cudaSetDevice(c->device);
    return phase_target_filter(c, n_removed);
}

uint64_t elp_n_sorted(const elp_ctx* c) { return c ? (c->sorted ? c->n_sorted : c->n) : 0; }

}  // extern "C"
