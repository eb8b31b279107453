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
// hand them back (elp_fetch_bam): output order, MAPQ, FLAG and QUAL patched, everything else -- names, CIGAR, tags -- untouched
// (the counterpart of formatting every *sam.Alignment again, sam/bam-files.go:635-735).  Not handled (error return): the CG:B long-CIGAR convention (:376-392),
// an RG:Z value that is not an @RG ID of the header (unless --replace-read-group puts every read in the one @RG, elp_set_replace_read_group).
#include <algorithm>
#include "ctx.h"
#include "regions.cuh"
#include "tagwalk.cuh"
#include "../../include/elprep_b200.h"

namespace {

__device__ __forceinline__ uint32_t rd32(const uint8_t* p) { return (uint32_t)p[0] | ((uint32_t)p[1] << 8) | ((uint32_t)p[2] << 16) | ((uint32_t)p[3] << 24); }
__device__ __forceinline__ uint32_t rd16(const uint8_t* p) { return (uint32_t)p[0] | ((uint32_t)p[1] << 8); }

struct BamArgs {
    uint64_t n, n0;                       // records in this call, reads already in the context
    const uint8_t* raw; const uint64_t* start; uint64_t n_bytes;   // start[i]: offset of record i's block_size field
    int chained;                          // start[] has n + 1 entries and start[i + 1] must be the end of record i (no filter ran)
    int clear_dup;                        // ClearDuplicateFlag: 0x400 cleared in the FLAG column (the stored record keeps its bytes)
    int rg_replace;                       // --replace-read-group: every read gets read group 0, whatever RG field its record has
    int32_t *refid, *pos, *nref, *pnext, *tlen, *rg; uint16_t* flag; uint8_t* mapq; uint8_t* optf;
    uint32_t *len_qname, *len_cigar, *len_seq, *len_qual;   // [n] lengths, scanned afterwards
    const uint8_t* rg_names; const uint32_t* rg_name_off; int n_rg;
    int n_ref;                            // refID / next_refID bound of the records (ingest_ref_bound)
    const int32_t* remap;                 // elp_set_input_dictionary: refID -> output contig of the columns, or null (off)
    uint32_t* err;
};

// fixed part: block_size(4) refID(4) pos(4) l_read_name(1) mapq(1) bin(2) n_cigar_op(2) flag(2) l_seq(4) next_refID(4) next_pos(4) tlen(4)
constexpr int BAM_FIXED = 36;

struct RgNames { const uint8_t* names; const uint32_t* off; int n; };

// The structure of one record of rec_len >= BAM_FIXED bytes, as parseBamAlignment (sam/bam-files.go:314-400) reads it: the variable
// lengths against block_size, contig ids, every optional field.  Returns 1 for a malformed record, else 2 for a well-formed one that
// uses the CG:B long-CIGAR convention, else 0; *rg_out: the @RG index of RG:Z, -1 without one, -2 for a value that is no @RG ID;
// *optf_out: the sr bit.  Every record of a call goes through it, whether the ingest filters keep it or not: a malformed record fails
// the call whatever filters are set, as the reference parses a record before any filter sees it.  CG:B and an unknown RG:Z value are
// well-formed (the reference reads them); they are refused only in the records that become reads, where the device cannot represent them.
__device__ uint32_t check_record(const uint8_t* r, uint64_t rec_len, int n_contigs, RgNames G, int32_t* rg_out, uint8_t* optf_out) {
    uint32_t bad = 0;
    const int32_t refid = (int32_t)rd32(r + 4);
    const uint32_t l_name = r[12], n_cig = rd16(r + 16);
    const int32_t l_seq = (int32_t)rd32(r + 20), nref = (int32_t)rd32(r + 24);
    // all lengths in 64 bits: a crafted l_seq near INT_MAX must not wrap (l_seq > rec_len is malformed whatever else the record says)
    const uint64_t lsq = l_seq < 0 ? 0ull : (uint64_t)(uint32_t)l_seq;
    const uint64_t var = (uint64_t)l_name + 4ull * n_cig + ((lsq + 1) >> 1) + lsq;
    if (l_name < 1 || l_seq < 0 || lsq > rec_len || BAM_FIXED + var > rec_len || refid >= n_contigs || nref >= n_contigs) bad = 1;
    int32_t rg = -1; uint8_t optf = 0; bool cg = false;
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
                    if (t0 == 'C' && t1 == 'G') cg = true;   // long-CIGAR convention: not supported here
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
                    for (int g = 0; g < G.n; g++) {
                        const uint32_t a = G.off[g], b = G.off[g + 1];
                        if ((uint64_t)(b - a) != e - x) continue;
                        bool same = true;
                        for (uint32_t q = 0; q < b - a && same; q++) same = G.names[a + q] == r[x + q];
                        if (same) { rg = g; break; }
                    }
                }
                x = e + 1;
            } else { if (x + sz > rec_len) { bad = 1; break; } x += sz; }
        }
        if (x != rec_len && !bad) bad = 1;
    }
    *rg_out = rg; *optf_out = optf;
    return bad ? bad : (cg ? 2u : 0u);
}

__global__ void __launch_bounds__(256) bam_fixed_kernel(BamArgs A) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= A.n) return;
    const uint64_t st = A.start[i];
    const uint8_t* r = A.raw + st;
    const uint64_t rec_len = (st + 4 <= A.n_bytes) ? (uint64_t)rd32(r) + 4 : 0;      // block_size counts the bytes after itself
    if (rec_len < BAM_FIXED || st + rec_len > A.n_bytes || (A.chained && A.start[i + 1] != st + rec_len)) { atomicOr(A.err, DERR_BAM); A.len_qname[i] = A.len_cigar[i] = A.len_seq[i] = A.len_qual[i] = 0; return; }
    const int32_t refid = (int32_t)rd32(r + 4), pos = (int32_t)rd32(r + 8);
    const uint32_t l_name = r[12], mapq = r[13], n_cig = rd16(r + 16), flag = rd16(r + 18);
    const int32_t l_seq = (int32_t)rd32(r + 20), nref = (int32_t)rd32(r + 24), pnext = (int32_t)rd32(r + 28), tlen = (int32_t)rd32(r + 32);
    const uint64_t k = A.n0 + i;
    // (remap is read only inside the bound: check_record below fails a record outside it)
    const int32_t ro = refid < 0 ? -1 : (!A.remap ? refid : (refid < A.n_ref ? A.remap[refid] : -1));
    const int32_t no = nref < 0 ? -1 : (!A.remap ? nref : (nref < A.n_ref ? A.remap[nref] : -1));
    A.refid[k] = ro; A.pos[k] = pos + 1; A.flag[k] = (uint16_t)(A.clear_dup ? flag & ~(uint32_t)F_DUPLICATE : flag); A.mapq[k] = (uint8_t)mapq;
    A.nref[k] = no; A.pnext[k] = pnext + 1; A.tlen[k] = tlen;
    int32_t rg; uint8_t optf;
    const uint32_t bad = check_record(r, rec_len, A.n_ref, RgNames{A.rg_names, A.rg_name_off, A.n_rg}, &rg, &optf);
    if (A.rg_replace) rg = 0;                  // (the record's RG fields are rewritten at egress; a value that is no @RG ID is not refused)
    else if (rg == -2) { atomicOr(A.err, DERR_BAM_RG); rg = -1; }
    if (bad) atomicOr(A.err, bad == 2 ? DERR_BAM_CG : DERR_BAM);
    A.rg[k] = rg; A.optf[k] = optf;
    A.len_qname[i] = bad ? 0 : l_name - 1; A.len_cigar[i] = bad ? 0 : n_cig;
    A.len_seq[i] = bad ? 0 : (uint32_t)((l_seq + 1) >> 1); A.len_qual[i] = bad ? 0 : (uint32_t)l_seq;
}

// ---- fused per-record filters of the ingest (SURVEY.md 8f row 4; filters/simple-filters.go:71-103,332-347) ----
// keep[i] = 1 iff record i passes every requested predicate; also checks that the caller's offsets follow the block_size chain
// (overlap_any: regions.cuh)
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
                                                        int n_ref, const int32_t* __restrict__ remap, bool drop_unmapped_ref, RgNames G, uint32_t* __restrict__ keep, uint32_t* __restrict__ err) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint64_t st = rec_off[i], len = rec_off[i + 1] - st;
    const uint8_t* r = raw + st;
    if (len < BAM_FIXED || (uint64_t)rd32(r) + 4 != len) { atomicOr(err, DERR_BAM); keep[i] = 0; return; }
    {   // the reference parses a record before any filter sees it: a malformed record fails the call even when a filter would drop it.
        // (CG:B and an unknown RG:Z are left to bam_fixed_kernel, which sees the records that are kept.)
        int32_t rg; uint8_t optf;
        if (check_record(r, len, n_ref, G, &rg, &optf) == 1) { atomicOr(err, DERR_BAM); keep[i] = 0; return; }
    }
    // from here on the record is well-formed: every length fits in len
    const int32_t refid = (int32_t)rd32(r + 4), pos = (int32_t)(rd32(r + 8) + 1u);                                 // int32 + 1 wraps as in Go
    const uint32_t l_name = r[12], mapq = r[13], n_cig = rd16(r + 16), flag = rd16(r + 18);
    // remap (elp_set_input_dictionary): the output contig of refid; with REPLACE (drop set) a read whose RNAME is not in the new dictionary
    // is dropped (ReplaceReferenceSequenceDictionary :49-57)
    const int32_t ro = (remap && refid >= 0) ? remap[refid] : refid;
    bool k = !(drop_unmapped_ref && refid >= 0 && ro < 0);
    if ((mask & ELP_FILTER_UNMAPPED) && (flag & F_UNMAPPED)) k = false;                                           // RemoveUnmappedReads :73-75
    if ((mask & ELP_FILTER_UNMAPPED_STRICT) && ((flag & F_UNMAPPED) || pos == 0 || refid < 0)) k = false;          // RemoveUnmappedReadsStrict :79-83
    if ((int32_t)mapq < min_mapq) k = false;                                                                      // RemoveMappingQualityLessThan :332-347 (min_mapq as elp_set_ingest_filter stores it)
    if (k && (mask & ELP_FILTER_NON_EXACT)) {                                                                     // RemoveNonExactMappingReads :90-99: only M and S
        const uint64_t c0 = BAM_FIXED + (uint64_t)l_name;
        for (uint32_t q = 0; q < n_cig; q++) { const uint32_t o = r[c0 + 4 * q] & 15u; if (o != 0 && o != 4) { k = false; break; } }
    }
    if ((mask & ELP_FILTER_DUPLICATES) && (flag & F_DUPLICATE)) k = false;                                        // RemoveDuplicateReads :131-133 (flags of the input)
    if (k && (mask & (ELP_FILTER_NON_EXACT_STRICT | ELP_FILTER_TARGET_REGIONS))) {
        const uint64_t lsq = rd32(r + 20);
        const uint64_t c0 = BAM_FIXED + (uint64_t)l_name;
        const uint64_t tags0 = c0 + 4ull * n_cig + ((lsq + 1) >> 1) + lsq;
        if (mask & ELP_FILTER_TARGET_REGIONS) {                                                                   // RemoveNonOverlappingReads :310-328
            int32_t a_end = pos;
            if (!(flag & F_UNMAPPED)) {
                uint32_t rl = 0, fl = 0;                                                                          // int32 sums of Go, wrapping: kept unsigned
                for (uint32_t q = 0; q < n_cig; q++) { const uint32_t op = rd32(r + c0 + 4 * q); const uint32_t o = op & 15u; const uint32_t ln = op >> 4;
                    if (o == 0 || o == 1 || o == 4 || o == 7 || o == 8) rl += ln; if (o == 0 || o == 2 || o == 3 || o == 7 || o == 8) fl += ln; }
                if ((int32_t)rl > 0) a_end = (int32_t)((uint32_t)pos + fl - 1u);                                  // aln.End(), sam/sam-types.go:769-775
            }
            if (ro < 0 || ro >= n_contigs || !regions || !overlap_any(regions[ro], n_regions[ro], pos, a_end)) k = false;   // no regions for RNAME: Overlap(nil) is false
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
                    case 'B': { const uint8_t sub = r[x]; const uint64_t cnt = rd32(r + x + 1);
                                sz = 5 + cnt * ((sub == 'c' || sub == 'C') ? 1 : ((sub == 's' || sub == 'S') ? 2 : 4)); break; }
                    default: sz = len;                                                                            // (check_record refused the record)
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
// output record k of a call: first + kk, or sel[first + kk] when the record filters of elp_set_output_filter select the records
__device__ __forceinline__ uint64_t out_pos(const uint32_t* __restrict__ sel, uint64_t first, uint64_t kk) { return sel ? sel[first + kk] : first + kk; }
__global__ void __launch_bounds__(256) bam_out_len_kernel(uint64_t n, uint64_t first, const uint32_t* __restrict__ sel, const uint32_t* __restrict__ perm, const uint64_t* __restrict__ all_start,
                                                           const uint8_t* __restrict__ all, uint32_t* __restrict__ len) {
    const uint64_t kk = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (kk < n) len[kk] = rd32(all + all_start[perm[out_pos(sel, first, kk)]]) + 4;
}
// elp_set_input_dictionary: lanes 4..7 and 24..27 rewrite the bytes of refID and next_refID as the output contig (-1 where there is none),
// after they copied the stored bytes there in their first step of the per-byte loop
__device__ __forceinline__ void patch_refids(const uint8_t* r, uint8_t* o, const int32_t* __restrict__ remap) {
    const unsigned lane = threadIdx.x & 31;
    if ((lane >= 4 && lane < 8) || (lane >= 24 && lane < 28)) {
        const int32_t id = (int32_t)rd32(r + (lane & ~3u));
        const uint32_t v = (uint32_t)(id < 0 ? -1 : remap[id]);
        o[lane] = (uint8_t)(v >> (8 * (lane & 3u)));
    }
}
// one warp per output record: copy the stored record, patch MAPQ (byte 13 of the record with its block_size; elp_clean_sam sets it to 0
// for unmapped reads, otherwise it equals the stored byte), FLAG (bytes 18..19) and QUAL
__global__ void __launch_bounds__(256) bam_out_copy_kernel(uint64_t n, uint64_t first, const uint32_t* __restrict__ sel, const uint32_t* __restrict__ perm, const uint64_t* __restrict__ all_start,
                                                            const uint8_t* __restrict__ all, const uint64_t* __restrict__ out_off, uint8_t* __restrict__ out,
                                                            const uint16_t* __restrict__ s_flag, const uint8_t* __restrict__ s_mapq, const uint64_t* __restrict__ s_out_off, const uint8_t* __restrict__ qual_out,
                                                            const int32_t* __restrict__ remap) {
    const unsigned lane = threadIdx.x & 31;
    const uint64_t kk = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (kk >= n) return;
    const uint64_t k = out_pos(sel, first, kk);
    const uint32_t i = perm[k];
    const uint8_t* r = all + all_start[i];
    const uint64_t len = (uint64_t)rd32(r) + 4;
    uint8_t* o = out + out_off[kk];
    const uint32_t l_name = r[12], n_cig = rd16(r + 16);
    const int32_t l_seq = (int32_t)rd32(r + 20);
    const uint64_t q0 = BAM_FIXED + (uint64_t)l_name + 4ull * n_cig + (uint64_t)((l_seq + 1) >> 1), q1 = q0 + (uint64_t)l_seq;
    const uint16_t f = s_flag[k];
    const uint8_t mq = s_mapq[k];
    const uint8_t* nq = qual_out ? qual_out + s_out_off[k] : nullptr;
    for (uint64_t t = lane; t < len; t += 32) {
        uint8_t v = r[t];
        if (t == 18) v = (uint8_t)(f & 0xff); else if (t == 19) v = (uint8_t)(f >> 8);
        else if (nq && t >= q0 && t < q1) v = nq[t - q0];
        o[t] = v;
    }
    if (lane == 13) o[13] = mq;                  // (this lane copied byte 13 in its first step: outside the per-byte loop, no extra compare there)
    if (remap) patch_refids(r, o, remap);
}

// ---- write-phase filters (elp_set_output_filter; cmd/filter.go:803-902) ----
// keep[k] = 1 iff output record k passes RemoveDuplicateReads (the FLAG after marking) and RemoveOptionalReads (no sr tag)
__global__ void __launch_bounds__(256) out_select_kernel(uint64_t n, uint32_t mask, const uint16_t* __restrict__ s_flag, const uint8_t* __restrict__ s_optf, uint32_t* __restrict__ keep) {
    const uint64_t k = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= n) return;
    bool ok = true;
    if ((mask & ELP_OUT_REMOVE_DUPLICATES) && (s_flag[k] & F_DUPLICATE)) ok = false;               // simple-filters.go:138-140
    if ((mask & ELP_OUT_REMOVE_OPTIONAL_READS) && (s_optf[k] & ELP_OPT_SR)) ok = false;            // :146-152
    keep[k] = ok ? 1u : 0u;
}
__global__ void __launch_bounds__(256) out_compact_kernel(uint64_t n, const uint32_t* __restrict__ keep, const uint64_t* __restrict__ slot, uint32_t* __restrict__ sel) {
    const uint64_t k = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (k < n && keep[k]) sel[slot[k]] = (uint32_t)k;
}

// start of the optional fields of a stored record
__device__ __forceinline__ uint64_t tags_start(const uint8_t* r) {
    const uint64_t l_seq = rd32(r + 20);
    return BAM_FIXED + (uint64_t)r[12] + 4ull * rd16(r + 16) + ((l_seq + 1) >> 1) + l_seq;
}

// RemoveOptionalFields / KeepOptionalFields (simple-filters.go:235-288) on BAM records, after SetRG when --replace-read-group is on
// (tagwalk::out_fields), one warp per output record; drop may be null (no field filter: only the RG field changes).
// measure: the record's length with the fields it is written with
__global__ void __launch_bounds__(256) bam_out_fields_measure_kernel(uint64_t n, uint64_t first, const uint32_t* __restrict__ sel, const uint32_t* __restrict__ perm,
                                                                     const uint64_t* __restrict__ all_start, const uint8_t* __restrict__ all, const uint32_t* __restrict__ drop,
                                                                     tagwalk::RgSet g, uint32_t* __restrict__ len) {
    const uint64_t kk = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (kk >= n) return;
    const uint8_t* r = all + all_start[perm[out_pos(sel, first, kk)]];
    const uint64_t rec = (uint64_t)rd32(r) + 4;
    const uint64_t t0 = tags_start(r);
    uint64_t x = t0;
    tagwalk::out_fields(r, t0, rec, drop, g, [&](uint64_t t, uint64_t fe, bool repl) { x += repl ? tagwalk::rg_field_bytes(g) : fe - t; });
    if ((threadIdx.x & 31) == 0) len[kk] = (uint32_t)x;
}
// emit: the fixed part and the variable fields with block_size, MAPQ, FLAG, QUAL (and, with remap, refID / next_refID) patched, then the
// fields in their order
__global__ void __launch_bounds__(256) bam_out_fields_emit_kernel(uint64_t n, uint64_t first, const uint32_t* __restrict__ sel, const uint32_t* __restrict__ perm,
                                                                  const uint64_t* __restrict__ all_start, const uint8_t* __restrict__ all, const uint32_t* __restrict__ drop,
                                                                  tagwalk::RgSet g, const uint64_t* __restrict__ out_off, uint8_t* __restrict__ out,
                                                                  const uint16_t* __restrict__ s_flag, const uint8_t* __restrict__ s_mapq, const uint64_t* __restrict__ s_out_off, const uint8_t* __restrict__ qual_out,
                                                                  const int32_t* __restrict__ remap) {
    const unsigned lane = threadIdx.x & 31;
    const uint64_t kk = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (kk >= n) return;
    const uint64_t k = out_pos(sel, first, kk);
    const uint8_t* r = all + all_start[perm[k]];
    const uint64_t rec = (uint64_t)rd32(r) + 4, t0 = tags_start(r);
    uint8_t* o = out + out_off[kk];
    const uint32_t bs = (uint32_t)(out_off[kk + 1] - out_off[kk] - 4);
    const int32_t l_seq = (int32_t)rd32(r + 20);
    const uint64_t q1 = t0, q0 = q1 - (uint64_t)l_seq;
    const uint16_t f = s_flag[k];
    const uint8_t mq = s_mapq[k];
    const uint8_t* nq = qual_out ? qual_out + s_out_off[k] : nullptr;
    for (uint64_t t = lane; t < t0; t += 32) {
        uint8_t v = r[t];
        if (t < 4) v = (uint8_t)(bs >> (8 * t));
        else if (t == 18) v = (uint8_t)(f & 0xff); else if (t == 19) v = (uint8_t)(f >> 8);
        else if (nq && t >= q0) v = nq[t - q0];
        o[t] = v;
    }
    if (lane == 13) o[13] = mq;                  // (as in bam_out_copy_kernel)
    if (remap) patch_refids(r, o, remap);
    uint64_t x = t0;
    tagwalk::out_fields(r, t0, rec, drop, g, [&](uint64_t t, uint64_t fe, bool repl) {
        if (repl) { tagwalk::rg_field_write(o + x, g); x += tagwalk::rg_field_bytes(g); return; }
        for (uint64_t j = lane; j < fe - t; j += 32) o[x + j] = r[t + j];
        x += fe - t;
    });
}

}  // namespace

// ---- region tables (RegionTable, ctx.h): the ingest filter's, the one of elp_filter_target_regions and the BQSR known sites ----
// one contig's regions: sorted by start and flattened unless already_flat (intervals.ParallelSortByStart + ParallelFlatten, intervals/intervals.go:88-117)
int region_set(elp_ctx* c, RegionTable& t, const char* who, int32_t contig, const int32_t* se, uint64_t n_intervals, int already_flat) {
    if (contig < 0 || contig >= c->n_contigs) return c->fail(E_INVAL, "%s: contig %d out of range", who, contig);
    if (n_intervals && !se) return c->fail(E_INVAL, "%s: null interval array", who);
    std::vector<std::pair<int32_t, int32_t>> iv(n_intervals);
    for (uint64_t i = 0; i < n_intervals; i++) iv[i] = {se[2 * i], se[2 * i + 1]};
    uint64_t n = n_intervals;
    if (!already_flat && n > 1) {
        std::stable_sort(iv.begin(), iv.end(), [](const std::pair<int32_t, int32_t>& a, const std::pair<int32_t, int32_t>& b) { return a.first < b.first; });
        uint64_t m = 0;
        for (uint64_t i = 0; i < n; i++) { if (m > 0 && iv[i].first <= iv[m - 1].second) { if (iv[i].second > iv[m - 1].second) iv[m - 1].second = iv[i].second; } else iv[m++] = iv[i]; }
        n = m;
    }
    t.clear(contig);
    if (n) {
        DBuf<int32_t>& own = t.own[contig];
        CUDA_TRY(c, own.fit(2 * n));
        CUDA_TRY(c, cudaMemcpyAsync(own.p, iv.data(), n * 8, cudaMemcpyHostToDevice, c->stream));
        CUDA_TRY(c, cudaStreamSynchronize(c->stream));
        t.d[contig] = own.p; t.n[contig] = n;
    }
    return ELP_OK;
}

extern "C" int elp_append_bam(elp_ctx* c, const uint8_t* records, uint64_t n_bytes, const uint64_t* record_off, uint64_t n_records) {
    if (!c || (!records && n_bytes)) return ELP_EINVAL;
    cudaSetDevice(c->device);
    std::lock_guard<std::mutex> lk(c->append_mu);
    if (c->sorted) return c->fail(E_STATE, "elp_append_bam after elp_sort_markdup (call elp_reset first)");
    if (c->bgzf_open) return c->fail(E_STATE, "elp_append_bam while a BGZF file is open (elp_append_bgzf_end first)");
    TRY(relabel_check_selected(c, "elp_append_bam"));
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

// @RG ID strings for the RG:Z match at ingest and the RG:Z value of --replace-read-group at egress, uploaded once per context
int rg_names_upload(elp_ctx* c) {
    if (c->d_rg_names.p || !c->n_rg) return E_OK;
    std::vector<uint8_t> names; std::vector<uint32_t> off(1, 0);
    for (auto& id : c->rg_ids) { names.insert(names.end(), id.begin(), id.end()); off.push_back((uint32_t)names.size()); }
    CUDA_TRY(c, c->d_rg_names.fit(std::max<size_t>(names.size(), 1)));
    CUDA_TRY(c, c->d_rg_name_off.fit(off.size()));
    CUDA_TRY(c, cudaMemcpy(c->d_rg_names.p, names.data(), names.size(), cudaMemcpyHostToDevice));
    CUDA_TRY(c, cudaMemcpy(c->d_rg_name_off.p, off.data(), off.size() * 4, cudaMemcpyHostToDevice));
    return E_OK;
}

// The device-resident part of elp_append_bam, shared with elp_append_sam: nrec records (n_bytes in all) already sit in bam_raw, and
// bam_off[0..nrec] holds their chained offsets (bam_off[nrec] == n_bytes).  The caller holds append_mu and has checked the phase
// and the 2^32 read limit.  From here on: ingest filters, fixed fields and RG:Z, segmented copies, QUAL presence, the bam_all arena.
int bam_ingest_core(elp_ctx* c, uint64_t n_bytes, uint64_t nrec, bool sam_records) {
    uint64_t bn = nrec;                                       // becomes the number of records that pass the filters
    const uint64_t n0 = c->n;
    cudaStream_t s = c->stream;
    // several inputs (merge_inputs.cu): the records as the merged header writes them, in the rewrite's buffer; bam_off follows them
    const uint8_t* raw = c->bam_raw.p;
    if (relabel_on(c)) TRY(relabel_records(c, &raw, c->bam_off.p, &n_bytes, nrec, sam_records));
    TRY(grow(c, c->bam_start, nrec + 2, 0));
    const uint64_t* d_start = c->bam_off.p;                   // without filters: record i is read n0 + i
    TRY(rg_names_upload(c));
    const int n_ref = ingest_ref_bound(c, sam_records);
    if (ingest_keep_on(c)) {
        TRY(grow(c, c->scan_tmp, nrec + 8, 0)); TRY(grow(c, c->off_stage, nrec + 2, 0));
        c->begin("bam_keep", (double)nrec * 48);
        if (c->filter_mask & ELP_FILTER_TARGET_REGIONS) TRY(table_upload(c, c->regions));
        bam_keep_kernel<<<nblk(nrec, 256), 256, 0, s>>>(nrec, raw, c->bam_off.p, n_bytes, c->filter_mask, c->filter_min_mapq, c->regions.d_ptrs.p, c->regions.d_n.p, c->n_contigs,
                                                        n_ref, ingest_remap(c), (c->dict_mode & ELP_DICT_REPLACE) != 0, RgNames{c->d_rg_names.p, c->d_rg_name_off.p, c->n_rg}, c->scan_tmp.p, c->d_err.p);
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
    TRY(grow(c, c->refid, n1 + 1, n0)); TRY(grow(c, c->pos, n1 + 1, n0)); TRY(grow(c, c->nref, n1 + 1, n0)); TRY(grow(c, c->pnext, n1 + 1, n0)); TRY(grow(c, c->tlen, n1 + 1, n0));
    TRY(grow(c, c->rg, n1 + 1, n0)); TRY(grow(c, c->flag, n1 + 2, n0)); TRY(grow(c, c->mapq, n1 + 1, n0)); TRY(grow(c, c->optf, n1 + 1, n0));
    TRY(grow(c, c->qname_off, n1 + 2, n0 + 1)); TRY(grow(c, c->cigar_off, n1 + 2, n0 + 1)); TRY(grow(c, c->qual_off, n1 + 2, n0 + 1)); TRY(grow(c, c->seq_off, n1 + 2, n0 + 1));
    TRY(grow(c, c->scan_tmp, 4 * (bn + 4) + 8, 0));   // (the keep flags above are dead by now)
    BamArgs A{};
    A.n = bn; A.n0 = n0; A.raw = raw; A.start = d_start; A.n_bytes = n_bytes; A.chained = d_start == c->bam_off.p; A.clear_dup = c->clear_dup; A.rg_replace = c->rg_replace;
    A.refid = c->refid.p; A.pos = c->pos.p; A.nref = c->nref.p; A.pnext = c->pnext.p; A.tlen = c->tlen.p; A.rg = c->rg.p; A.flag = c->flag.p; A.mapq = c->mapq.p; A.optf = c->optf.p;
    A.len_qname = c->scan_tmp.p; A.len_cigar = c->scan_tmp.p + (bn + 4); A.len_seq = c->scan_tmp.p + 2 * (bn + 4); A.len_qual = c->scan_tmp.p + 3 * (bn + 4);
    A.rg_names = c->d_rg_names.p; A.rg_name_off = c->d_rg_name_off.p; A.n_rg = c->n_rg; A.n_ref = n_ref; A.remap = ingest_remap(c); A.err = c->d_err.p;
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
    B.n = bn; B.n0 = n0; B.raw = raw; B.start = d_start;
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
        CUDA_TRY(c, cudaMemcpyAsync(c->bam_all.p + c->n_bam, raw, n_bytes, cudaMemcpyDeviceToDevice, s));
        CUDA_TRY(c, cudaMemcpyAsync(c->bam_all_off.p + n0, d_start, bn * 8, cudaMemcpyDeviceToDevice, s));      // start of every kept record
        if (c->n_bam) { add_base_u64_kernel<<<nblk(bn, 256), 256, 0, s>>>(bn, c->bam_all_off.p + n0, c->n_bam); c->launches++; }
        CUDA_TRY(c, cudaStreamSynchronize(s));
        c->n_bam += n_bytes; c->bam_reads = n1;
    }
    c->n = n1; c->n_qname = ends[0]; c->n_cigar = ends[1]; c->n_seq = ends[2]; c->n_qual = ends[3];
    c->adapted = false;
    return ELP_OK;
}

// The selection of the record filters: sel[j] is the output position of the j-th record that passes (in output order).  Built once per
// sort and setting, on the first filtered fetch; without record bits there is none (sel null, every record passes).
int out_select(elp_ctx* c, const uint32_t** sel, uint64_t* n_out) {
    *sel = nullptr; *n_out = c->n_sorted;
    if (!c->out_mask) return E_OK;
    if (!c->out_sel_valid) {
        const uint64_t n = c->n_sorted;
        uint64_t kept = 0;
        if (n) {
            cudaStream_t s = c->stream;
            TRY(grow(c, c->scan_tmp, n + 8, 0)); TRY(grow(c, c->off_stage, n + 2, 0)); TRY(grow(c, c->out_sel, n + 1, 0));
            c->begin("out_select", 7.0 * (double)n);
            out_select_kernel<<<nblk(n, 256), 256, 0, s>>>(n, c->out_mask, c->s_flag.p, c->s_optf.p, c->scan_tmp.p);
            c->end(); LAUNCH_CHECK(c);
            TRY(exclusive_scan_u32_to_u64(c, c->scan_tmp.p, c->off_stage.p, n));
            c->begin("out_select", 12.0 * (double)n + 4.0 * (double)n);
            out_compact_kernel<<<nblk(n, 256), 256, 0, s>>>(n, c->scan_tmp.p, c->off_stage.p, c->out_sel.p);
            c->end(); LAUNCH_CHECK(c);
            CUDA_TRY(c, cudaMemcpyAsync(&kept, c->off_stage.p + n, 8, cudaMemcpyDeviceToHost, s));
            CUDA_TRY(c, cudaStreamSynchronize(s));
        }
        c->n_out = kept; c->out_sel_valid = true;
    }
    *sel = c->out_sel.p; *n_out = c->n_out;
    return E_OK;
}

// the RG:Z value the egress writes (elp_set_replace_read_group), or off
tagwalk::RgSet rg_set(const elp_ctx* c) {
    return c->rg_replace ? tagwalk::RgSet{c->d_rg_names.p, (uint32_t)c->rg_ids[0].size(), true} : tagwalk::RgSet{nullptr, 0, false};
}

// record lengths of the call (as the field filter and the read-group replacement write them, when set) scanned into off_stage[0..n], *total bytes
static int bam_out_prepare(elp_ctx* c, uint64_t first, uint64_t n, uint64_t* total, const uint32_t** sel) {
    if (!c->sorted) return c->fail(E_STATE, "elp_fetch_bam before elp_sort_markdup");
    if (c->bam_reads != c->n) return c->fail(E_STATE, "elp_fetch_bam: not every read of this context came in through elp_append_bam");
    uint64_t n_out = 0;
    TRY(out_select(c, sel, &n_out));
    if (first + n > n_out) {
        if (*sel) return c->fail(E_INVAL, "elp_fetch_bam: range [%llu,%llu) exceeds the %llu output records that pass the record filters (elp_n_output)", (unsigned long long)first, (unsigned long long)(first + n), (unsigned long long)n_out);
        return c->fail(E_INVAL, "elp_fetch_bam: range [%llu,%llu) exceeds %llu reads", (unsigned long long)first, (unsigned long long)(first + n), (unsigned long long)n_out);
    }
    TRY(grow(c, c->scan_tmp, n + 8, 0)); TRY(grow(c, c->off_stage, n + 2, 0));
    if (c->out_fields || c->rg_replace) {
        c->begin("bam_out_fields_measure", (double)c->n_bam * (double)n / (double)std::max<uint64_t>(c->n, 1) + 4.0 * (double)n);
        bam_out_fields_measure_kernel<<<nblk(n * 32, 256), 256, 0, c->stream>>>(n, first, *sel, c->perm.p, c->bam_all_off.p, c->bam_all.p, c->out_fields ? c->d_out_drop.p : nullptr,
                                                                                 rg_set(c), c->scan_tmp.p);
        c->end();
    } else {
        bam_out_len_kernel<<<nblk(n, 256), 256, 0, c->stream>>>(n, first, *sel, c->perm.p, c->bam_all_off.p, c->bam_all.p, c->scan_tmp.p); c->launches++;
    }
    LAUNCH_CHECK(c);
    TRY(exclusive_scan_u32_to_u64(c, c->scan_tmp.p, c->off_stage.p, n));
    CUDA_TRY(c, cudaMemcpyAsync(total, c->off_stage.p + n, 8, cudaMemcpyDeviceToHost, c->stream));
    CUDA_TRY(c, cudaStreamSynchronize(c->stream));
    return E_OK;
}

// the records of the call (bam_out_prepare ran: off_stage holds their offsets, total their bytes) formatted at dst
static int bam_out_format(elp_ctx* c, uint64_t first, uint64_t n, const uint32_t* sel, uint64_t total, uint8_t* dst) {
    if (c->out_fields || c->rg_replace) {
        c->begin("bam_out_fields_emit", (double)c->n_bam * (double)n / (double)std::max<uint64_t>(c->n, 1) + (double)total);
        bam_out_fields_emit_kernel<<<nblk(n * 32, 256), 256, 0, c->stream>>>(n, first, sel, c->perm.p, c->bam_all_off.p, c->bam_all.p, c->out_fields ? c->d_out_drop.p : nullptr,
                                                                             rg_set(c), c->off_stage.p, dst,
                                                                             c->s_flag.p, c->s_mapq.p, c->s_out_off.p, c->qual_out_valid ? c->qual_out.p : nullptr, ingest_remap(c));
    } else {
        c->begin("bam_format", 2.0 * (double)total);
        bam_out_copy_kernel<<<nblk(n * 32, 256), 256, 0, c->stream>>>(n, first, sel, c->perm.p, c->bam_all_off.p, c->bam_all.p, c->off_stage.p, dst, c->s_flag.p, c->s_mapq.p, c->s_out_off.p,
                                                                      c->qual_out_valid ? c->qual_out.p : nullptr, ingest_remap(c));
    }
    c->end(); LAUNCH_CHECK(c);
    return E_OK;
}

extern "C" uint64_t elp_fetch_bam_bytes(elp_ctx* c, uint64_t first, uint64_t n) {
    if (!c || n == 0) return 0;
    cudaSetDevice(c->device);
    uint64_t total = 0; const uint32_t* sel = nullptr;
    if (bam_out_prepare(c, first, n, &total, &sel)) return 0;
    return total;
}

extern "C" int elp_fetch_bam(elp_ctx* c, uint64_t first, uint64_t n, uint8_t* out, uint64_t capacity, uint64_t* record_off) {
    if (c && c->n_cleaned) return c->fail(E_STATE, "elp_fetch_bam: elp_clean_sam rewrote %llu CIGARs; the stored records still carry the old ones (use elp_fetch)", (unsigned long long)c->n_cleaned);
    if (!c || (!out && n)) return ELP_EINVAL;
    cudaSetDevice(c->device);
    if (n == 0) { if (record_off) record_off[0] = 0; return ELP_OK; }
    uint64_t total = 0; const uint32_t* sel = nullptr;
    TRY(bam_out_prepare(c, first, n, &total, &sel));
    if (total > capacity) return c->fail(E_INVAL, "elp_fetch_bam: output buffer too small (%llu > %llu)", (unsigned long long)total, (unsigned long long)capacity);
    TRY(grow(c, c->bam_raw, total + 64, 0));      // staging for the formatted records
    TRY(bam_out_format(c, first, n, sel, total, c->bam_raw.p));
    CUDA_TRY(c, cudaMemcpyAsync(out, c->bam_raw.p, total, cudaMemcpyDeviceToHost, c->stream));
    if (record_off) CUDA_TRY(c, cudaMemcpyAsync(record_off, c->off_stage.p, (n + 1) * 8, cudaMemcpyDeviceToHost, c->stream));
    CUDA_TRY(c, cudaStreamSynchronize(c->stream));
    return ELP_OK;
}

// the records of elp_fetch_bam(first, n) behind the caller's prefix in bam_raw, deflated there (bgzf_deflate.cu): the records never leave the
// device uncompressed
extern "C" int elp_fetch_bgzf(elp_ctx* c, uint64_t first, uint64_t n, const uint8_t* prefix, uint64_t n_prefix, int write_eof, uint8_t* out, uint64_t capacity, uint64_t* out_n) {
    if (c && c->n_cleaned) return c->fail(E_STATE, "elp_fetch_bgzf: elp_clean_sam rewrote %llu CIGARs; the stored records still carry the old ones (use elp_fetch)", (unsigned long long)c->n_cleaned);
    if (!c || !out || !out_n || (!prefix && n_prefix)) return ELP_EINVAL;
    cudaSetDevice(c->device);
    uint64_t total = 0; const uint32_t* sel = nullptr;
    if (n) TRY(bam_out_prepare(c, first, n, &total, &sel));
    const uint64_t all = n_prefix + total, need = elp_bgzf_deflate_bound(all);
    if (capacity < need) return c->fail(E_INVAL, "elp_fetch_bgzf: output buffer too small (%llu < elp_bgzf_deflate_bound = %llu)", (unsigned long long)capacity, (unsigned long long)need);
    TRY(grow(c, c->bam_raw, all + 64, 0));
    if (n_prefix) CUDA_TRY(c, cudaMemcpyAsync(c->bam_raw.p, prefix, n_prefix, cudaMemcpyHostToDevice, c->stream));
    if (n) TRY(bam_out_format(c, first, n, sel, total, c->bam_raw.p + n_prefix));
    return bgzf_deflate_run(c, c->bam_raw.p, all, write_eof, out, out_n);
}

extern "C" int elp_set_target_regions(elp_ctx* c, int32_t contig, const int32_t* se, uint64_t n_intervals, int already_flat) {
    if (!c) return ELP_EINVAL;
    cudaSetDevice(c->device);
    return region_set(c, c->regions, "elp_set_target_regions", contig, se, n_intervals, already_flat);
}

extern "C" int elp_set_ingest_filter(elp_ctx* c, uint32_t mask, int32_t min_mapq) {
    if (!c) return ELP_EINVAL;
    if (mask & ~(uint32_t)(ELP_FILTER_UNMAPPED | ELP_FILTER_UNMAPPED_STRICT | ELP_FILTER_NON_EXACT | ELP_FILTER_DUPLICATES | ELP_FILTER_NON_EXACT_STRICT | ELP_FILTER_TARGET_REGIONS | ELP_FILTER_CLEAR_DUPLICATE_FLAG)) return c->fail(E_INVAL, "elp_set_ingest_filter: unknown filter bits 0x%x", mask);
    c->filter_mask = mask & ~(uint32_t)ELP_FILTER_CLEAR_DUPLICATE_FLAG;   // (the clear drops no record)
    // RemoveMappingQualityLessThan(mq int): 0 no filter, above 255 every read dropped, else MAPQ >= byte(mq) -- so -1 keeps MAPQ 255 only
    c->filter_min_mapq = min_mapq == 0 ? 0 : (min_mapq > 255 ? 256 : (int32_t)((uint32_t)min_mapq & 255u));
    c->clear_dup = (mask & ELP_FILTER_CLEAR_DUPLICATE_FLAG) != 0;
    return ELP_OK;
}

// a 2-byte tag string as its index in the tag table; -1 for any other length (it matches no field, as an interned symbol would not)
static int32_t tag_index(const char* s) { return (s && s[0] && s[1] && !s[2]) ? (int32_t)((uint8_t)s[0] | ((uint32_t)(uint8_t)s[1] << 8)) : -1; }

extern "C" int elp_set_output_filter(elp_ctx* c, uint32_t mask, const char* const* remove_tags, int32_t n_remove, const char* const* keep_tags, int32_t n_keep) {
    if (!c) return ELP_EINVAL;
    cudaSetDevice(c->device);
    if (mask & ~(uint32_t)(ELP_OUT_REMOVE_DUPLICATES | ELP_OUT_REMOVE_OPTIONAL_READS | ELP_OUT_KEEP_FIELDS)) return c->fail(E_INVAL, "elp_set_output_filter: unknown filter bits 0x%x", mask);
    if (n_remove < 0 || n_keep < 0 || (n_remove && !remove_tags) || (n_keep && !keep_tags)) return c->fail(E_INVAL, "elp_set_output_filter: bad tag list");
    if (n_keep && !(mask & ELP_OUT_KEEP_FIELDS)) return c->fail(E_INVAL, "elp_set_output_filter: keep_tags without ELP_OUT_KEEP_FIELDS");
    // one decision per tag: RemoveOptionalFields(remove_tags), then KeepOptionalFields(keep_tags) -- dropped by either, dropped
    std::vector<uint32_t> drop(2048, 0u);
    for (int32_t i = 0; i < n_remove; i++) { const int32_t t = tag_index(remove_tags[i]); if (t >= 0) drop[t >> 5] |= 1u << (t & 31); }
    if (mask & ELP_OUT_KEEP_FIELDS) {
        std::vector<uint32_t> keep(2048, 0u);
        for (int32_t i = 0; i < n_keep; i++) { const int32_t t = tag_index(keep_tags[i]); if (t >= 0) keep[t >> 5] |= 1u << (t & 31); }
        for (int w = 0; w < 2048; w++) drop[w] |= ~keep[w];
    }
    bool any = false;
    for (uint32_t w : drop) any |= w != 0;
    if (any) {
        CUDA_TRY(c, c->d_out_drop.fit(2048));
        CUDA_TRY(c, cudaMemcpyAsync(c->d_out_drop.p, drop.data(), 2048 * 4, cudaMemcpyHostToDevice, c->stream));
        CUDA_TRY(c, cudaStreamSynchronize(c->stream));   // (drop is pageable host memory)
    }
    c->out_mask = mask & ~(uint32_t)ELP_OUT_KEEP_FIELDS; c->out_fields = any; c->out_sel_valid = false;
    return ELP_OK;
}

extern "C" int elp_set_replace_read_group(elp_ctx* c, int on) {
    if (!c) return ELP_EINVAL;
    cudaSetDevice(c->device);
    if (c->n || c->sorted || c->bgzf_open) return c->fail(E_STATE, "elp_set_replace_read_group: the context holds reads (call it after elp_create or elp_reset)");
    if (on && c->n_rg != 1) return c->fail(E_INVAL, "elp_set_replace_read_group: the context must be created with exactly one @RG, the replacement (it has %d)", c->n_rg);
    if (on) TRY(rg_names_upload(c));
    c->rg_replace = on != 0;
    return ELP_OK;
}

// the names elp_fetch_sam prints for a stored refID: the input name table, with "chr" prefixed under RENAME (RenameChromosomes runs on
// RNAME / RNEXT before the output is formatted); elp_config's names while the setting is off
std::vector<std::string> sam_print_names(const elp_ctx* c) {
    if (!c->dict_mode) return c->contig_names;
    std::vector<std::string> v;
    for (const std::string& s : c->in_tab) v.push_back((c->dict_mode & ELP_DICT_RENAME_CHROMOSOMES) ? "chr" + s : s);
    return v;
}

extern "C" int elp_set_input_dictionary(elp_ctx* c, uint32_t mode, const char* const* names, const int32_t* lengths, int32_t n) {
    if (!c) return ELP_EINVAL;
    cudaSetDevice(c->device);
    if (mode & ~(uint32_t)(ELP_DICT_RENAME_CHROMOSOMES | ELP_DICT_REPLACE)) return c->fail(E_INVAL, "elp_set_input_dictionary: unknown mode bits 0x%x", mode);
    if (n < 0 || (n && (!names || !lengths))) return c->fail(E_INVAL, "elp_set_input_dictionary: bad input dictionary (n = %d)", n);
    if (mode && relabel_on(c)) return c->fail(E_INVAL, "elp_set_input_dictionary: the context has inputs or tag renames (elp_add_input, elp_set_tag_rename); the two do not combine");
    if (c->n || c->sorted || c->bgzf_open) return c->fail(E_STATE, "elp_set_input_dictionary: the context holds reads (call it after elp_create or elp_reset)");
    if (mode && !c->has_contig_names) return c->fail(E_INVAL, "elp_set_input_dictionary: the context was created without elp_config.contig_names");
    const bool rename = (mode & ELP_DICT_RENAME_CHROMOSOMES) != 0, replace = (mode & ELP_DICT_REPLACE) != 0;
    std::vector<std::string> in;
    for (int32_t i = 0; i < n; i++) {
        if (!names[i]) return c->fail(E_INVAL, "elp_set_input_dictionary: input name %d is null", i);
        in.push_back(names[i]);
    }
    if (rename && !replace) {
        if (n != c->n_contigs) return c->fail(E_INVAL, "elp_set_input_dictionary: RENAME_CHROMOSOMES alone: the input has %d @SQ, elp_config %d contigs", n, c->n_contigs);
        for (int32_t i = 0; i < n; i++)
            if (c->contig_names[i] != "chr" + in[i])
                return c->fail(E_INVAL, "elp_set_input_dictionary: RENAME_CHROMOSOMES alone: contig %d of elp_config is '%s', not 'chr%s'", i, c->contig_names[i].c_str(), in[i].c_str());
    }
    c->sam_out.reset();                      // (elp_fetch_sam's name table follows the setting)
    c->in_dict = NameDictBufs();
    c->in_tab.clear(); c->in_len.clear(); c->n_in = 0; c->dict_mode = 0;
    if (!mode) return ELP_OK;
    auto renamed = [&](const std::string& s) { return rename ? "chr" + s : s; };
    std::map<std::string, int32_t> last_out, last_in_len;   // AddREFID: the last of equal names wins; CleanSam's table likewise
    for (int j = 0; j < c->n_contigs; j++) last_out[c->contig_names[j]] = j;
    for (int32_t i = 0; i < n; i++) last_in_len[renamed(in[i])] = lengths[i];
    std::vector<int32_t> remap;
    for (int32_t i = 0; i < n; i++) {
        if (!replace) { remap.push_back(i); continue; }
        auto it = last_out.find(renamed(in[i]));
        remap.push_back(it == last_out.end() ? -1 : it->second);
    }
    std::vector<std::string> tab = in;
    if (replace) {   // the SAM extension: replacement names no input name reaches, as the RNAME text that renames to them
        std::map<std::string, int> known;
        for (const std::string& s : in) known.emplace(s, 0);
        for (int j = 0; j < c->n_contigs; j++) {
            const std::string& N = c->contig_names[j];
            if (rename && N.compare(0, 3, "chr") != 0) continue;   // unreachable: every renamed RNAME starts with "chr"
            const std::string text = rename ? N.substr(3) : N;
            if (text == "*" || !known.emplace(text, 0).second) continue;
            tab.push_back(text); remap.push_back(last_out[N]);
        }
    }
    remap.push_back(-1);                     // elp_append_sam under REPLACE: an RNAME that reaches nothing
    std::vector<int32_t> clean_len(std::max(1, c->n_contigs), 0);
    for (int j = 0; j < c->n_contigs; j++) { auto it = last_in_len.find(c->contig_names[j]); if (it != last_in_len.end()) clean_len[j] = it->second; }
    CUDA_TRY(c, c->d_remap.fit(remap.size()));
    CUDA_TRY(c, c->d_clean_len.fit(clean_len.size()));
    CUDA_TRY(c, cudaMemcpy(c->d_remap.p, remap.data(), remap.size() * 4, cudaMemcpyHostToDevice));
    CUDA_TRY(c, cudaMemcpy(c->d_clean_len.p, clean_len.data(), clean_len.size() * 4, cudaMemcpyHostToDevice));
    c->in_tab = tab; c->in_len.assign(lengths, lengths + n); c->n_in = n; c->dict_mode = mode;
    return ELP_OK;
}

extern "C" uint64_t elp_n_output(elp_ctx* c) {
    if (!c || !c->sorted) return 0;
    cudaSetDevice(c->device);
    const uint32_t* sel = nullptr; uint64_t n_out = 0;
    if (out_select(c, &sel, &n_out)) return 0;
    return n_out;
}
extern "C" uint64_t elp_n_filtered(const elp_ctx* c) { return c ? c->n_filtered : 0; }
