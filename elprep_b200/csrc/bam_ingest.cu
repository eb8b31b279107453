// bam_ingest.cu -- BAM alignment records straight into the device columns (SURVEY.md §8f row 1; replaces the host-side
// parseBamAlignment, sam/bam-files.go:314-400, for the fields this path uses).
//
// The caller hands over the decompressed BAM record bytes as they sit in the file (each record preceded by its 4-byte
// block_size) plus the byte offset of every record.  Two kernels:
//   bam_fixed_kernel  one thread per record: the fixed-offset little-endian fields (:300-312) -> refid, pos (+1), flag, mapq,
//                     nref, pnext (+1), tlen columns; the lengths of the four variable parts; the RG:Z tag located by walking
//                     the typed optional fields (sam/bam-files.go optionalBAMFieldParseTable) and matched against @RG IDs
//   bam_copy_kernel   one warp per record: QNAME bytes (without the NUL), CIGAR words (already `len<<4|op`), SEQ nibbles
//                     and QUAL bytes (phred without +33) are byte-for-byte the device layout -> four segmented copies
// Offsets come from device prefix sums of the lengths.  The raw records stay in a device arena so that the write phase can
// hand them back (elp_fetch_bam): output order, FLAG and QUAL patched, everything else -- names, CIGAR, tags -- untouched
// (the counterpart of formatting every *sam.Alignment again, sam/bam-files.go:635-735).  Not handled (error return): the CG:B long-CIGAR convention (:376-392),
// an RG:Z value that is not an @RG ID of the header.
#include <algorithm>
#include "ctx.h"
#include "../../include/elprep_b200.h"

namespace {

inline unsigned nblk(uint64_t n, int t) { return (unsigned)((n + t - 1) / t); }

__device__ __forceinline__ uint32_t rd32(const uint8_t* p) { return (uint32_t)p[0] | ((uint32_t)p[1] << 8) | ((uint32_t)p[2] << 16) | ((uint32_t)p[3] << 24); }
__device__ __forceinline__ uint32_t rd16(const uint8_t* p) { return (uint32_t)p[0] | ((uint32_t)p[1] << 8); }

struct BamArgs {
    uint64_t n, n0;                       // records in this call, reads already in the context
    const uint8_t* raw; const uint64_t* start; uint64_t n_bytes;   // start[i]: offset of record i's block_size field
    int chained;                          // start[] has n + 1 entries and start[i + 1] must be the end of record i (no filter ran)
    int32_t *refid, *pos, *nref, *pnext, *tlen, *rg; uint16_t* flag; uint8_t* mapq; uint8_t* optf;
    uint32_t *len_qname, *len_cigar, *len_seq, *len_qual;   // [n] lengths, scanned afterwards
    const uint8_t* rg_names; const uint32_t* rg_name_off; int n_rg; int n_contigs;
    uint32_t* err;
};

// fixed part: block_size(4) refID(4) pos(4) l_read_name(1) mapq(1) bin(2) n_cigar_op(2) flag(2) l_seq(4) next_refID(4) next_pos(4) tlen(4)
constexpr int BAM_FIXED = 36;

__global__ void __launch_bounds__(256) bam_fixed_kernel(BamArgs A) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= A.n) return;
    const uint64_t st = A.start[i];
    const uint8_t* r = A.raw + st;
    uint32_t bad = 0;
    const uint64_t rec_len = (st + 4 <= A.n_bytes) ? (uint64_t)rd32(r) + 4 : 0;      // block_size counts the bytes after itself
    if (rec_len < BAM_FIXED || st + rec_len > A.n_bytes || (A.chained && A.start[i + 1] != st + rec_len)) { atomicOr(A.err, DERR_BAM); A.len_qname[i] = A.len_cigar[i] = A.len_seq[i] = A.len_qual[i] = 0; return; }
    const int32_t refid = (int32_t)rd32(r + 4), pos = (int32_t)rd32(r + 8);
    const uint32_t l_name = r[12], mapq = r[13], n_cig = rd16(r + 16), flag = rd16(r + 18);
    const int32_t l_seq = (int32_t)rd32(r + 20), nref = (int32_t)rd32(r + 24), pnext = (int32_t)rd32(r + 28), tlen = (int32_t)rd32(r + 32);
    // all lengths in 64 bits: a crafted l_seq near INT_MAX must not wrap (l_seq > rec_len is malformed whatever else the record says)
    const uint64_t lsq = l_seq < 0 ? 0ull : (uint64_t)(uint32_t)l_seq;
    const uint64_t var = (uint64_t)l_name + 4ull * n_cig + ((lsq + 1) >> 1) + lsq;
    if (l_name < 1 || l_seq < 0 || lsq > rec_len || BAM_FIXED + var > rec_len || refid >= A.n_contigs || nref >= A.n_contigs) bad = 1;
    const uint64_t k = A.n0 + i;
    A.refid[k] = refid < 0 ? -1 : refid; A.pos[k] = pos + 1; A.flag[k] = (uint16_t)flag; A.mapq[k] = (uint8_t)mapq;
    A.nref[k] = nref < 0 ? -1 : nref; A.pnext[k] = pnext + 1; A.tlen[k] = tlen;
    int32_t rg = -1; uint8_t optf = 0;
    if (!bad) {
        // optional fields: tag[2] type[1] value (sam/bam-files.go:369-397)
        uint64_t x = BAM_FIXED + var;
        while (x + 3 <= rec_len) {
            const uint8_t t0 = r[x], t1 = r[x + 1], ty = r[x + 2];
            x += 3;
            if (t0 == 's' && t1 == 'r') optf |= 1;          // the sr tag of `elprep split` (sam/split-merge.go:286-293)
            uint64_t sz = 0; bool str = false;
            switch (ty) {
                case 'A': case 'c': case 'C': sz = 1; break;
                case 's': case 'S': sz = 2; break;
                case 'i': case 'I': case 'f': sz = 4; break;
                case 'Z': case 'H': str = true; break;
                case 'B': {
                    if (x + 5 > rec_len) { bad = 1; break; }
                    const uint8_t sub = r[x]; const uint64_t cnt = rd32(r + x + 1);
                    const uint64_t es = (sub == 'c' || sub == 'C') ? 1 : ((sub == 's' || sub == 'S') ? 2 : ((sub == 'i' || sub == 'I' || sub == 'f') ? 4 : 0));
                    if (!es) bad = 1;
                    if (t0 == 'C' && t1 == 'G') bad = 2;     // long-CIGAR convention: not supported here
                    if (cnt * es > rec_len) { bad = 1; break; }    // (cnt < 2^32, es <= 4: no overflow; bounded before it is added to x)
                    sz = 5 + cnt * es; break;
                }
                default: bad = 1;
            }
            if (bad) break;
            if (str) {
                uint64_t e = x;
                while (e < rec_len && r[e] != 0) e++;
                if (e >= rec_len) { bad = 1; break; }
                if (t0 == 'R' && t1 == 'G' && ty == 'Z') {
                    rg = -2;                                   // present but (so far) unknown
                    for (int g = 0; g < A.n_rg; g++) {
                        const uint32_t a = A.rg_name_off[g], b = A.rg_name_off[g + 1];
                        if ((uint64_t)(b - a) != e - x) continue;
                        bool same = true;
                        for (uint32_t q = 0; q < b - a && same; q++) same = A.rg_names[a + q] == r[x + q];
                        if (same) { rg = g; break; }
                    }
                }
                x = e + 1;
            } else { if (x + sz > rec_len) { bad = 1; break; } x += sz; }
        }
        if (x != rec_len && !bad) bad = 1;
    }
    if (rg == -2) { atomicOr(A.err, DERR_BAM_RG); rg = -1; }
    if (bad) atomicOr(A.err, bad == 2 ? DERR_BAM_CG : DERR_BAM);
    A.rg[k] = rg; A.optf[k] = optf;
    A.len_qname[i] = bad ? 0 : l_name - 1; A.len_cigar[i] = bad ? 0 : n_cig;
    A.len_seq[i] = bad ? 0 : (uint32_t)((l_seq + 1) >> 1); A.len_qual[i] = bad ? 0 : (uint32_t)l_seq;
}

// ---- fused per-record filters of the ingest (SURVEY.md 8f row 4; filters/simple-filters.go:71-103,332-347) ----
// keep[i] = 1 iff record i passes every requested predicate; also checks that the caller's offsets follow the block_size chain
// intervals.Overlap (intervals/intervals.go:146-164) over one contig's flattened, start-sorted (start, end) pairs
__device__ bool overlap_any(const int32_t* __restrict__ iv, uint64_t n, int32_t start, int32_t end) {
    int64_t left = 0, right = (int64_t)n - 1;
    while (left <= right) {
        const int64_t mid = (left + right) / 2;
        const int32_t is = iv[2 * mid], ie = iv[2 * mid + 1];
        if (is > end - 1) right = mid - 1;
        else if (ie <= start - 1) left = mid + 1;
        else return true;
    }
    return false;
}
// integer value of an optional field at r[x] (x behind tag and type), by BAM type; false for a non-integer type
__device__ __forceinline__ bool tag_int(const uint8_t* r, uint64_t x, uint8_t ty, int64_t* v) {
    switch (ty) {
        case 'c': *v = (int8_t)r[x]; return true;
        case 'C': *v = r[x]; return true;
        case 's': *v = (int16_t)rd16(r + x); return true;
        case 'S': *v = rd16(r + x); return true;
        case 'i': *v = (int32_t)rd32(r + x); return true;
        case 'I': *v = rd32(r + x); return true;
        default: return false;
    }
}

__global__ void __launch_bounds__(256) bam_keep_kernel(uint64_t n, const uint8_t* __restrict__ raw, const uint64_t* __restrict__ rec_off, uint64_t n_bytes,
                                                        uint32_t mask, int32_t min_mapq, const int32_t* const* __restrict__ regions, const uint64_t* __restrict__ n_regions, int n_contigs,
                                                        uint32_t* __restrict__ keep, uint32_t* __restrict__ err) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint64_t st = rec_off[i], len = rec_off[i + 1] - st;
    const uint8_t* r = raw + st;
    if (len < BAM_FIXED || (uint64_t)rd32(r) + 4 != len) { atomicOr(err, DERR_BAM); keep[i] = 0; return; }
    const int32_t refid = (int32_t)rd32(r + 4), pos = (int32_t)rd32(r + 8) + 1;
    const uint32_t l_name = r[12], mapq = r[13], n_cig = rd16(r + 16), flag = rd16(r + 18);
    bool k = true;
    if ((mask & ELP_FILTER_UNMAPPED) && (flag & F_UNMAPPED)) k = false;                                           // RemoveUnmappedReads :73-75
    if ((mask & ELP_FILTER_UNMAPPED_STRICT) && ((flag & F_UNMAPPED) || pos == 0 || refid < 0)) k = false;          // RemoveUnmappedReadsStrict :79-83
    if ((int32_t)mapq < min_mapq) k = false;                                                                      // RemoveMappingQualityLessThan :332-347
    if (k && (mask & ELP_FILTER_NON_EXACT)) {                                                                     // RemoveNonExactMappingReads :90-99: only M and S
        const uint64_t c0 = BAM_FIXED + (uint64_t)l_name;
        if (c0 + 4ull * n_cig > len) { atomicOr(err, DERR_BAM); keep[i] = 0; return; }
        for (uint32_t q = 0; q < n_cig; q++) { const uint32_t o = r[c0 + 4 * q] & 15u; if (o != 0 && o != 4) { k = false; break; } }
    }
    if ((mask & ELP_FILTER_DUPLICATES) && (flag & F_DUPLICATE)) k = false;                                        // RemoveDuplicateReads :131-133 (flags of the input)
    if (k && (mask & (ELP_FILTER_NON_EXACT_STRICT | ELP_FILTER_TARGET_REGIONS))) {
        const int32_t l_seq = (int32_t)rd32(r + 20);
        const uint64_t c0 = BAM_FIXED + (uint64_t)l_name, lsq = l_seq < 0 ? 0ull : (uint64_t)(uint32_t)l_seq;
        const uint64_t tags0 = c0 + 4ull * n_cig + ((lsq + 1) >> 1) + lsq;
        if (l_seq < 0 || tags0 > len) { atomicOr(err, DERR_BAM); keep[i] = 0; return; }
        if (mask & ELP_FILTER_TARGET_REGIONS) {                                                                   // RemoveNonOverlappingReads :310-328
            int32_t a_end = pos;
            if (!(flag & F_UNMAPPED)) {
                int32_t rl = 0, fl = 0;
                for (uint32_t q = 0; q < n_cig; q++) { const uint32_t op = rd32(r + c0 + 4 * q); const uint32_t o = op & 15u; const int32_t ln = (int32_t)(op >> 4);
                    if (o == 0 || o == 1 || o == 4 || o == 7 || o == 8) rl += ln; if (o == 0 || o == 2 || o == 3 || o == 7 || o == 8) fl += ln; }
                if (rl > 0) a_end = pos + fl - 1;                                                                 // aln.End(), sam/sam-types.go:769-775
            }
            if (refid < 0 || refid >= n_contigs || !regions || !overlap_any(regions[refid], n_regions[refid], pos, a_end)) k = false;   // no regions for RNAME: Overlap(nil) is false
        }
        if (k && (mask & ELP_FILTER_NON_EXACT_STRICT)) {                                                          // RemoveNonExactMappingReadsStrict :115-136: X0=1, X1=0, XM=0, XO=0, XG=0
            int64_t want[5] = {1, 0, 0, 0, 0}; uint32_t seen = 0; bool good = true;
            uint64_t x = tags0;
            while (x + 3 <= len && good) {
                const uint8_t t0 = r[x], t1 = r[x + 1], ty = r[x + 2];
                x += 3;
                int which = -1;
                if (t0 == 'X') which = t1 == '0' ? 0 : (t1 == '1' ? 1 : (t1 == 'M' ? 2 : (t1 == 'O' ? 3 : (t1 == 'G' ? 4 : -1))));
                uint64_t sz = 0;
                switch (ty) {
                    case 'A': case 'c': case 'C': sz = 1; break;
                    case 's': case 'S': sz = 2; break;
                    case 'i': case 'I': case 'f': sz = 4; break;
                    case 'Z': case 'H': { uint64_t e = x; while (e < len && r[e] != 0) e++; sz = e - x + 1; break; }
                    case 'B': { if (x + 5 > len) { sz = len; break; } const uint8_t sub = r[x]; const uint64_t cnt = rd32(r + x + 1);
                                sz = 5 + cnt * ((sub == 'c' || sub == 'C') ? 1 : ((sub == 's' || sub == 'S') ? 2 : 4)); break; }
                    default: sz = len;                                                                            // malformed: bam_fixed_kernel reports it
                }
                if (x + sz > len) break;
                if (which >= 0 && !(seen & (1u << which))) {                                                      // (TAGS.Get returns the first occurrence)
                    int64_t v;
                    seen |= 1u << which;
                    if (!tag_int(r, x, ty, &v) || v != want[which]) good = false;                                 // a non-integer value is treated as a mismatch (the Go type assertion would panic)
                }
                x += sz;
            }
            if (!good || seen != 31u) k = false;
        }
    }
    keep[i] = k ? 1u : 0u;
}
__global__ void __launch_bounds__(256) bam_compact_kernel(uint64_t n, const uint32_t* __restrict__ keep, const uint64_t* __restrict__ slot, const uint64_t* __restrict__ rec_off,
                                                           uint64_t* __restrict__ start) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n && keep[i]) start[slot[i]] = rec_off[i];
}

struct CopyArgs {
    uint64_t n, n0;
    const uint8_t* raw; const uint64_t* start;
    const uint64_t *qname_off, *cigar_off, *seq_off, *qual_off;   // arena-global, indexed n0 + i
    uint8_t* qname; uint32_t* cigar; uint8_t* seq; uint8_t* qual;
};

__global__ void __launch_bounds__(256) bam_copy_kernel(CopyArgs A) {
    const unsigned lane = threadIdx.x & 31;
    const uint64_t i = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (i >= A.n) return;
    const uint64_t k = A.n0 + i;
    const uint8_t* r = A.raw + A.start[i];
    const uint64_t q0 = A.qname_off[k], q1 = A.qname_off[k + 1], c0 = A.cigar_off[k], c1 = A.cigar_off[k + 1];
    const uint64_t s0 = A.seq_off[k], s1 = A.seq_off[k + 1], u0 = A.qual_off[k], u1 = A.qual_off[k + 1];
    if (q1 == q0 && c1 == c0 && s1 == s0 && u1 == u0) return;      // rejected record
    const uint8_t* p = r + BAM_FIXED;
    for (uint64_t t = lane; t < q1 - q0; t += 32) A.qname[q0 + t] = p[t];
    p += (q1 - q0) + 1;                                               // NUL
    for (uint64_t t = lane; t < c1 - c0; t += 32) A.cigar[c0 + t] = rd32(p + 4 * t);
    p += 4 * (c1 - c0);
    for (uint64_t t = lane; t < s1 - s0; t += 32) A.seq[s0 + t] = p[t];
    p += s1 - s0;
    for (uint64_t t = lane; t < u1 - u0; t += 32) A.qual[u0 + t] = p[t];
}

__global__ void __launch_bounds__(256) add_base_u64_kernel(uint64_t n, uint64_t* __restrict__ v, uint64_t base) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) v[i] += base;
}

// ---- egress ----
__global__ void __launch_bounds__(256) bam_out_len_kernel(uint64_t n, const uint32_t* __restrict__ perm, const uint64_t* __restrict__ all_start, const uint8_t* __restrict__ all,
                                                           uint32_t* __restrict__ len) {
    const uint64_t k = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (k < n) len[k] = rd32(all + all_start[perm[k]]) + 4;
}
// one warp per output record: copy the stored record, patch FLAG (bytes 18..19 of the record with its block_size) and QUAL
__global__ void __launch_bounds__(256) bam_out_copy_kernel(uint64_t n, uint64_t first, const uint32_t* __restrict__ perm, const uint64_t* __restrict__ all_start,
                                                            const uint8_t* __restrict__ all, const uint64_t* __restrict__ out_off, uint8_t* __restrict__ out,
                                                            const uint16_t* __restrict__ s_flag, const uint64_t* __restrict__ s_out_off, const uint8_t* __restrict__ qual_out) {
    const unsigned lane = threadIdx.x & 31;
    const uint64_t kk = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (kk >= n) return;
    const uint64_t k = first + kk;
    const uint32_t i = perm[k];
    const uint8_t* r = all + all_start[i];
    const uint64_t len = (uint64_t)rd32(r) + 4;
    uint8_t* o = out + out_off[kk];
    const uint32_t l_name = r[12], n_cig = rd16(r + 16);
    const int32_t l_seq = (int32_t)rd32(r + 20);
    const uint64_t q0 = BAM_FIXED + (uint64_t)l_name + 4ull * n_cig + (uint64_t)((l_seq + 1) >> 1), q1 = q0 + (uint64_t)l_seq;
    const uint16_t f = s_flag[k];
    const uint8_t* nq = qual_out ? qual_out + s_out_off[k] : nullptr;
    for (uint64_t t = lane; t < len; t += 32) {
        uint8_t v = r[t];
        if (t == 18) v = (uint8_t)(f & 0xff); else if (t == 19) v = (uint8_t)(f >> 8);
        else if (nq && t >= q0 && t < q1) v = nq[t - q0];
        o[t] = v;
    }
}

template <class T> int grow(elp_ctx* c, DBuf<T>& b, size_t need, size_t keep) {
    cudaError_t e = b.reserve(need, c->stream, keep);
    if (e != cudaSuccess) return c->fail(e == cudaErrorMemoryAllocation ? E_NOMEM : E_CUDA, "device allocation of %zu bytes failed: %s", need * sizeof(T), cudaGetErrorString(e));
    return E_OK;
}
#define TRY(x) do { int rc__ = (x); if (rc__) return rc__; } while (0)

}  // namespace

static int upload_regions(elp_ctx* c) {
    if (!c->regions_dirty && c->d_region_ptrs) return E_OK;
    const int nc = std::max(1, c->n_contigs);
    if ((int)c->d_regions.size() != c->n_contigs) { c->d_regions.assign(c->n_contigs, nullptr); c->n_regions.assign(c->n_contigs, 0); }
    if (!c->d_region_ptrs) { CUDA_TRY(c, cudaMalloc(&c->d_region_ptrs, nc * sizeof(void*))); CUDA_TRY(c, cudaMalloc(&c->d_n_regions, nc * 8)); }
    if (c->n_contigs) {
        CUDA_TRY(c, cudaMemcpy(c->d_region_ptrs, c->d_regions.data(), c->n_contigs * sizeof(void*), cudaMemcpyHostToDevice));
        CUDA_TRY(c, cudaMemcpy(c->d_n_regions, c->n_regions.data(), c->n_contigs * 8, cudaMemcpyHostToDevice));
    }
    c->regions_dirty = false;
    return E_OK;
}

extern "C" int elp_append_bam(elp_ctx* c, const uint8_t* records, uint64_t n_bytes, const uint64_t* record_off, uint64_t n_records) {
    if (!c || (!records && n_bytes)) return ELP_EINVAL;
    cudaSetDevice(c->device);
    std::lock_guard<std::mutex> lk(c->append_mu);
    if (c->sorted) return c->fail(E_STATE, "elp_append_bam after elp_sort_markdup (call elp_reset first)");
    // record offsets: given, or found by walking the block_size chain
    std::vector<uint64_t> walked;
    if (!record_off) {
        uint64_t x = 0;
        while (x + 4 <= n_bytes) {
            walked.push_back(x);
            const uint32_t bs = (uint32_t)records[x] | ((uint32_t)records[x + 1] << 8) | ((uint32_t)records[x + 2] << 16) | ((uint32_t)records[x + 3] << 24);
            x += 4ull + bs;
        }
        if (x != n_bytes) return c->fail(E_INVAL, "elp_append_bam: the block_size chain does not end at n_bytes");
        walked.push_back(n_bytes);
        n_records = walked.size() - 1;
        record_off = walked.data();
    }
    const uint64_t nrec = n_records;
    if (nrec == 0) return ELP_OK;
    if (record_off[nrec] != n_bytes) return c->fail(E_INVAL, "elp_append_bam: record_off[n_records] must equal n_bytes");
    for (uint64_t i = 0; i < nrec; i++) if (record_off[i + 1] < record_off[i] || record_off[i + 1] > n_bytes) return c->fail(E_INVAL, "elp_append_bam: record_off must be non-decreasing and within n_bytes");
    if (c->n + nrec >= (1ull << 32)) return c->fail(E_LIMIT, "more than 2^32-1 reads in one context");
    TRY(grow(c, c->bam_raw, n_bytes + 64, 0)); TRY(grow(c, c->bam_off, nrec + 2, 0));
    CUDA_TRY(c, cudaMemcpyAsync(c->bam_raw.p, records, n_bytes, cudaMemcpyHostToDevice, c->stream));
    CUDA_TRY(c, cudaMemcpyAsync(c->bam_off.p, record_off, (nrec + 1) * 8, cudaMemcpyHostToDevice, c->stream));
    return bam_ingest_core(c, n_bytes, nrec);
}

// The device-resident part of elp_append_bam, shared with elp_append_sam: nrec records (n_bytes in all) already sit in bam_raw, and
// bam_off[0..nrec] holds their chained offsets (bam_off[nrec] == n_bytes).  The caller holds append_mu and has checked the phase
// and the 2^32 read limit.  From here on: ingest filters, fixed fields and RG:Z, segmented copies, QUAL presence, the bam_all arena.
int bam_ingest_core(elp_ctx* c, uint64_t n_bytes, uint64_t nrec) {
    uint64_t bn = nrec;                                       // becomes the number of records that pass the filters
    const uint64_t n0 = c->n;
    cudaStream_t s = c->stream;
    TRY(grow(c, c->bam_start, nrec + 2, 0));
    const uint64_t* d_start = c->bam_off.p;                   // without filters: record i is read n0 + i
    if (c->filter_mask || c->filter_min_mapq > 0) {
        TRY(grow(c, c->scan_tmp, nrec + 8, 0)); TRY(grow(c, c->off_stage, nrec + 2, 0));
        c->begin("bam_keep", (double)nrec * 48);
        if (c->filter_mask & ELP_FILTER_TARGET_REGIONS) { int rcr = upload_regions(c); if (rcr) return rcr; }
        bam_keep_kernel<<<nblk(nrec, 256), 256, 0, s>>>(nrec, c->bam_raw.p, c->bam_off.p, n_bytes, c->filter_mask, c->filter_min_mapq, c->d_region_ptrs, c->d_n_regions, c->n_contigs, c->scan_tmp.p, c->d_err);
        c->end(); LAUNCH_CHECK(c);
        TRY(exclusive_scan_u32_to_u64(c, c->scan_tmp.p, c->off_stage.p, nrec));
        bam_compact_kernel<<<nblk(nrec, 256), 256, 0, s>>>(nrec, c->scan_tmp.p, c->off_stage.p, c->bam_off.p, c->bam_start.p); c->launches++;
        LAUNCH_CHECK(c);
        uint64_t kept = 0;
        CUDA_TRY(c, cudaMemcpyAsync(&kept, c->off_stage.p + nrec, 8, cudaMemcpyDeviceToHost, s));
        int rc0 = check_device_errors(c);   // synchronizes
        if (rc0) return rc0;
        bn = kept; d_start = c->bam_start.p;
        c->n_filtered += nrec - kept;
        if (bn == 0) return ELP_OK;
    }
    const uint64_t n1 = n0 + bn;
    // @RG ID strings for the RG:Z match
    if (!c->d_rg_names && c->n_rg) {
        std::vector<uint8_t> names; std::vector<uint32_t> off(1, 0);
        for (auto& id : c->rg_ids) { names.insert(names.end(), id.begin(), id.end()); off.push_back((uint32_t)names.size()); }
        CUDA_TRY(c, cudaMalloc(&c->d_rg_names, std::max<size_t>(names.size(), 1)));
        CUDA_TRY(c, cudaMalloc(&c->d_rg_name_off, off.size() * 4));
        CUDA_TRY(c, cudaMemcpy(c->d_rg_names, names.data(), names.size(), cudaMemcpyHostToDevice));
        CUDA_TRY(c, cudaMemcpy(c->d_rg_name_off, off.data(), off.size() * 4, cudaMemcpyHostToDevice));
    }
    TRY(grow(c, c->refid, n1 + 1, n0)); TRY(grow(c, c->pos, n1 + 1, n0)); TRY(grow(c, c->nref, n1 + 1, n0)); TRY(grow(c, c->pnext, n1 + 1, n0)); TRY(grow(c, c->tlen, n1 + 1, n0));
    TRY(grow(c, c->rg, n1 + 1, n0)); TRY(grow(c, c->flag, n1 + 2, n0)); TRY(grow(c, c->mapq, n1 + 1, n0)); TRY(grow(c, c->optf, n1 + 1, n0));
    TRY(grow(c, c->qname_off, n1 + 2, n0 + 1)); TRY(grow(c, c->cigar_off, n1 + 2, n0 + 1)); TRY(grow(c, c->qual_off, n1 + 2, n0 + 1)); TRY(grow(c, c->seq_off, n1 + 2, n0 + 1));
    TRY(grow(c, c->scan_tmp, 4 * (bn + 4) + 8, 0));   // (the keep flags above are dead by now)
    BamArgs A{};
    A.n = bn; A.n0 = n0; A.raw = c->bam_raw.p; A.start = d_start; A.n_bytes = n_bytes; A.chained = d_start == c->bam_off.p;
    A.refid = c->refid.p; A.pos = c->pos.p; A.nref = c->nref.p; A.pnext = c->pnext.p; A.tlen = c->tlen.p; A.rg = c->rg.p; A.flag = c->flag.p; A.mapq = c->mapq.p; A.optf = c->optf.p;
    A.len_qname = c->scan_tmp.p; A.len_cigar = c->scan_tmp.p + (bn + 4); A.len_seq = c->scan_tmp.p + 2 * (bn + 4); A.len_qual = c->scan_tmp.p + 3 * (bn + 4);
    A.rg_names = c->d_rg_names; A.rg_name_off = c->d_rg_name_off; A.n_rg = c->n_rg; A.n_contigs = c->n_contigs; A.err = c->d_err;
    c->begin("bam_fixed", (double)bn * 36 + (double)n_bytes * 0.2);
    bam_fixed_kernel<<<nblk(bn, 256), 256, 0, s>>>(A);
    c->end(); LAUNCH_CHECK(c);
    // offsets = arena base + exclusive prefix sums of the lengths
    const uint64_t bases[4] = {c->n_qname, c->n_cigar, c->n_seq, c->n_qual};
    uint64_t* outs[4] = {c->qname_off.p + n0, c->cigar_off.p + n0, c->seq_off.p + n0, c->qual_off.p + n0};
    const uint32_t* lens[4] = {A.len_qname, A.len_cigar, A.len_seq, A.len_qual};
    uint64_t ends[4];
    for (int a = 0; a < 4; a++) {
        TRY(exclusive_scan_u32_to_u64(c, lens[a], outs[a], bn));
        if (bases[a]) { add_base_u64_kernel<<<nblk(bn + 1, 256), 256, 0, s>>>(bn + 1, outs[a], bases[a]); c->launches++; }
        CUDA_TRY(c, cudaMemcpyAsync(&ends[a], outs[a] + bn, 8, cudaMemcpyDeviceToHost, s));
    }
    LAUNCH_CHECK(c);
    int rc = check_device_errors(c);   // synchronizes
    if (rc) return rc;
    TRY(grow(c, c->qname, ends[0] + 64, c->n_qname)); TRY(grow(c, c->cigar, ends[1] + 16, c->n_cigar));
    TRY(grow(c, c->seq, ends[2] + 64, c->n_seq)); TRY(grow(c, c->qual, ends[3] + 64, c->n_qual));
    CopyArgs B{};
    B.n = bn; B.n0 = n0; B.raw = c->bam_raw.p; B.start = d_start;
    B.qname_off = c->qname_off.p; B.cigar_off = c->cigar_off.p; B.seq_off = c->seq_off.p; B.qual_off = c->qual_off.p;
    B.qname = c->qname.p; B.cigar = c->cigar.p; B.seq = c->seq.p; B.qual = c->qual.p;
    c->begin("bam_copy", 2.0 * (double)n_bytes);
    bam_copy_kernel<<<nblk(bn * 32, 256), 256, 0, s>>>(B);
    c->end(); LAUNCH_CHECK(c);
    TRY(qual_presence_update(c, c->n_qual, ends[3] - c->n_qual));
    CUDA_TRY(c, cudaStreamSynchronize(s));   // the caller's buffer may be released after return (cgo pointer rules)
    // keep the raw records for elp_fetch_bam (only meaningful while every read of the context came in as BAM)
    if (c->bam_reads == n0) {
        TRY(grow(c, c->bam_all, c->n_bam + n_bytes + 64, c->n_bam)); TRY(grow(c, c->bam_all_off, n1 + 2, n0));
        CUDA_TRY(c, cudaMemcpyAsync(c->bam_all.p + c->n_bam, c->bam_raw.p, n_bytes, cudaMemcpyDeviceToDevice, s));
        CUDA_TRY(c, cudaMemcpyAsync(c->bam_all_off.p + n0, d_start, bn * 8, cudaMemcpyDeviceToDevice, s));      // start of every kept record
        if (c->n_bam) { add_base_u64_kernel<<<nblk(bn, 256), 256, 0, s>>>(bn, c->bam_all_off.p + n0, c->n_bam); c->launches++; }
        CUDA_TRY(c, cudaStreamSynchronize(s));
        c->n_bam += n_bytes; c->bam_reads = n1;
    }
    c->n = n1; c->n_qname = ends[0]; c->n_cigar = ends[1]; c->n_seq = ends[2]; c->n_qual = ends[3];
    c->adapted = false;
    return ELP_OK;
}

static int bam_out_prepare(elp_ctx* c, uint64_t first, uint64_t n, uint64_t* total) {
    if (!c->sorted) return c->fail(E_STATE, "elp_fetch_bam before elp_sort_markdup");
    if (c->bam_reads != c->n) return c->fail(E_STATE, "elp_fetch_bam: not every read of this context came in through elp_append_bam");
    if (first + n > c->n) return c->fail(E_INVAL, "elp_fetch_bam: range [%llu,%llu) exceeds %llu reads", (unsigned long long)first, (unsigned long long)(first + n), (unsigned long long)c->n);
    TRY(grow(c, c->scan_tmp, n + 8, 0)); TRY(grow(c, c->off_stage, n + 2, 0));
    bam_out_len_kernel<<<nblk(n, 256), 256, 0, c->stream>>>(n, c->perm.p + first, c->bam_all_off.p, c->bam_all.p, c->scan_tmp.p); c->launches++;
    LAUNCH_CHECK(c);
    TRY(exclusive_scan_u32_to_u64(c, c->scan_tmp.p, c->off_stage.p, n));
    CUDA_TRY(c, cudaMemcpyAsync(total, c->off_stage.p + n, 8, cudaMemcpyDeviceToHost, c->stream));
    CUDA_TRY(c, cudaStreamSynchronize(c->stream));
    return E_OK;
}

extern "C" uint64_t elp_fetch_bam_bytes(elp_ctx* c, uint64_t first, uint64_t n) {
    if (!c || n == 0) return 0;
    cudaSetDevice(c->device);
    uint64_t total = 0;
    if (bam_out_prepare(c, first, n, &total)) return 0;
    return total;
}

extern "C" int elp_fetch_bam(elp_ctx* c, uint64_t first, uint64_t n, uint8_t* out, uint64_t capacity, uint64_t* record_off) {
    if (c && c->n_cleaned) return c->fail(E_STATE, "elp_fetch_bam: elp_clean_sam rewrote %llu CIGARs; the stored records still carry the old ones (use elp_fetch)", (unsigned long long)c->n_cleaned);
    if (!c || (!out && n)) return ELP_EINVAL;
    cudaSetDevice(c->device);
    if (n == 0) { if (record_off) record_off[0] = 0; return ELP_OK; }
    uint64_t total = 0;
    TRY(bam_out_prepare(c, first, n, &total));
    if (total > capacity) return c->fail(E_INVAL, "elp_fetch_bam: output buffer too small (%llu > %llu)", (unsigned long long)total, (unsigned long long)capacity);
    TRY(grow(c, c->bam_raw, total + 64, 0));      // staging for the formatted records
    c->begin("bam_format", 2.0 * (double)total);
    bam_out_copy_kernel<<<nblk(n * 32, 256), 256, 0, c->stream>>>(n, first, c->perm.p, c->bam_all_off.p, c->bam_all.p, c->off_stage.p, c->bam_raw.p, c->s_flag.p, c->s_out_off.p,
                                                                  c->qual_out_valid ? c->qual_out.p : nullptr);
    c->end(); LAUNCH_CHECK(c);
    CUDA_TRY(c, cudaMemcpyAsync(out, c->bam_raw.p, total, cudaMemcpyDeviceToHost, c->stream));
    if (record_off) CUDA_TRY(c, cudaMemcpyAsync(record_off, c->off_stage.p, (n + 1) * 8, cudaMemcpyDeviceToHost, c->stream));
    CUDA_TRY(c, cudaStreamSynchronize(c->stream));
    return ELP_OK;
}

extern "C" int elp_set_target_regions(elp_ctx* c, int32_t contig, const int32_t* se, uint64_t n_intervals, int already_flat) {
    if (!c) return ELP_EINVAL;
    cudaSetDevice(c->device);
    if (contig < 0 || contig >= c->n_contigs) return c->fail(E_INVAL, "elp_set_target_regions: contig %d out of range", contig);
    if ((int)c->d_regions.size() != c->n_contigs) { c->d_regions.assign(c->n_contigs, nullptr); c->n_regions.assign(c->n_contigs, 0); }
    std::vector<std::pair<int32_t, int32_t>> iv(n_intervals);
    for (uint64_t i = 0; i < n_intervals; i++) iv[i] = {se[2 * i], se[2 * i + 1]};
    uint64_t n = n_intervals;
    if (!already_flat && n > 1) {   // intervals.ParallelSortByStart + ParallelFlatten (intervals/intervals.go:88-117)
        std::stable_sort(iv.begin(), iv.end(), [](const std::pair<int32_t, int32_t>& a, const std::pair<int32_t, int32_t>& b) { return a.first < b.first; });
        uint64_t m = 0;
        for (uint64_t i = 0; i < n; i++) { if (m > 0 && iv[i].first <= iv[m - 1].second) { if (iv[i].second > iv[m - 1].second) iv[m - 1].second = iv[i].second; } else iv[m++] = iv[i]; }
        n = m;
    }
    if (c->d_regions[contig]) { cudaFree(c->d_regions[contig]); c->d_regions[contig] = nullptr; }
    if (n) { CUDA_TRY(c, cudaMalloc(&c->d_regions[contig], n * 8)); CUDA_TRY(c, cudaMemcpy(c->d_regions[contig], iv.data(), n * 8, cudaMemcpyHostToDevice)); }
    c->n_regions[contig] = n; c->regions_dirty = true;
    return ELP_OK;
}

extern "C" int elp_set_ingest_filter(elp_ctx* c, uint32_t mask, int32_t min_mapq) {
    if (!c) return ELP_EINVAL;
    if (mask & ~(uint32_t)(ELP_FILTER_UNMAPPED | ELP_FILTER_UNMAPPED_STRICT | ELP_FILTER_NON_EXACT | ELP_FILTER_DUPLICATES | ELP_FILTER_NON_EXACT_STRICT | ELP_FILTER_TARGET_REGIONS)) return c->fail(E_INVAL, "elp_set_ingest_filter: unknown filter bits 0x%x", mask);
    c->filter_mask = mask; c->filter_min_mapq = min_mapq;
    return ELP_OK;
}
extern "C" uint64_t elp_n_filtered(const elp_ctx* c) { return c ? c->n_filtered : 0; }
