// sam_format.cu -- SAM text alignment lines of the stored records in output order (replaces FormatAlignment, sam/sam-files.go:563-598,
// with formatSamTag :485-546 and cigarToString :548-557, applied to parseBamAlignment, sam/bam-files.go:317-400, of every record a
// BAM-in or SAM-in run writes to a SAM file).
//
// Line k is FormatAlignment(parseBamAlignment(stored record of perm[k])) with the context's FLAG and MAPQ and, once elp_bqsr_apply has run, the
// recalibrated QUAL: the bytes elp_fetch_bam returns, written as text.  One warp per line; one device function (format_line) in three modes:
//   sam_out_measure  byte length of every line, number of float values (f fields and B:f elements) in it
//   sam_out_float    only when a line holds a float value: the float bits into one list (the host formats them, gofloat.hpp), then the
//                    text lengths added to the line lengths
//   sam_out_emit     every line at its scanned offset
// Nothing of a line is held in registers or shared memory: fields are written while the record is walked, so lines have no length limit.
#include <algorithm>
#include <string>
#include <thread>
#include <vector>
#include "ctx.h"
#include "gofloat.hpp"
#include "pool.hpp"
#include "tagwalk.cuh"
#include "../../include/elprep_b200.h"

struct SamOutState {
    uint8_t* d_names = nullptr; uint32_t* d_name_off = nullptr; int32_t* d_canon = nullptr;   // @SQ names, and per contig the first index with its name
    DBuf<uint32_t> nf, fbits; DBuf<uint64_t> fbase, foff; DBuf<uint8_t> ftext;               // float values: count per line, slots, texts
    unsigned long long* d_small = nullptr;                                                   // [0] error bits, [1] float values
};

void sam_out_release(elp_ctx* c) {
    SamOutState* S = c->sam_out;
    if (!S) return;
    S->nf.release(); S->fbits.release(); S->fbase.release(); S->foff.release(); S->ftext.release();
    void* singles[] = {S->d_names, S->d_name_off, S->d_canon, S->d_small};
    for (void* p : singles) if (p) cudaFree(p);
    delete S;
    c->sam_out = nullptr;
}

namespace {

inline unsigned nblk(uint64_t n, int t) { return (unsigned)((n + t - 1) / t); }
template <class T> int grow(elp_ctx* c, DBuf<T>& b, size_t need, size_t keep) {
    cudaError_t e = b.reserve(need, c->stream, keep);
    if (e != cudaSuccess) return c->fail(e == cudaErrorMemoryAllocation ? E_NOMEM : E_CUDA, "device allocation of %zu bytes failed: %s", need * sizeof(T), cudaGetErrorString(e));
    return E_OK;
}
#define TRY(x) do { int rc__ = (x); if (rc__) return rc__; } while (0)

enum { FM_MEASURE = 0, FM_LIST = 1, FM_EMIT = 2 };
enum : unsigned long long { FE_CIGAR_OP = 1, FE_LINE_LIMIT = 2 };

struct FmtArgs {
    uint64_t n, first;                                                    // lines [first, first + n) of the output order (of sel when sel is set)
    const uint32_t* sel;                                                  // output positions of the records the record filters keep, or null
    const uint32_t* drop;                                                 // 65 536-bit tag table of the field filter, or null
    const uint32_t* perm; const uint64_t* all_start; const uint8_t* all;
    const uint16_t* flag; const uint8_t* mapq;                            // in output order: FLAG after marking, MAPQ after elp_clean_sam
    const uint64_t* qoff; const uint8_t* qual;                            // qual: recalibrated QUAL in output order, or null (stored QUAL)
    const uint8_t* names; const uint32_t* name_off; const int32_t* canon; int n_contigs;   // canon[n_contigs]: the canon of "*" (-1 if no @SQ has that name)
    uint32_t* len; uint32_t* nf;                                          // measure: line length, float values per line
    const uint64_t* fbase; uint32_t* fbits;                               // list: slot of a line's first float value, float bits
    const uint8_t* ftext; const uint64_t* foff;                           // emit: float texts by slot
    const uint64_t* line_off; uint8_t* out;                               // emit
    unsigned long long* small;
};

__device__ __forceinline__ uint32_t rd32(const uint8_t* p) { return (uint32_t)p[0] | ((uint32_t)p[1] << 8) | ((uint32_t)p[2] << 16) | ((uint32_t)p[3] << 24); }
__device__ __forceinline__ uint32_t rd16(const uint8_t* p) { return (uint32_t)p[0] | ((uint32_t)p[1] << 8); }

// decimal digits of v from the powers of ten; sdig: strconv.AppendInt length of a value in [-2^31, 2^32)
__device__ __forceinline__ int ndig(uint32_t v) {
    constexpr uint32_t P10[9] = {10u, 100u, 1000u, 10000u, 100000u, 1000000u, 10000000u, 100000000u, 1000000000u};
    int d = 1;
#pragma unroll
    for (int i = 0; i < 9; i++) d += v >= P10[i];
    return d;
}
__device__ __forceinline__ int sdig(int64_t v) { return v < 0 ? 1 + ndig((uint32_t)(-v)) : ndig((uint32_t)v); }
// the nd = sdig(v) characters of v, from the last digit backward
__device__ __forceinline__ void put_dec(uint8_t* o, int64_t v, int nd) {
    uint32_t a = (uint32_t)(v < 0 ? -v : v);
    const int lo = v < 0 ? 1 : 0;
    if (lo) o[0] = '-';
    for (int i = nd - 1; i >= lo; i--) { o[i] = (uint8_t)('0' + a % 10u); a /= 10u; }
}

__device__ __forceinline__ int warp_incl(int v) {
    const unsigned lane = threadIdx.x & 31;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) { const int u = __shfl_up_sync(FULL_MASK, v, d); if (lane >= (unsigned)d) v += u; }
    return v;
}

struct Ident { __device__ uint32_t operator()(uint32_t v) const { return v; } };
struct Phred33 { __device__ uint32_t operator()(uint32_t v) const { return __vadd4(v, 0x21212121u); } };   // + 33 per byte, wrapping (0xff -> ' ')
struct Lower { __device__ uint32_t operator()(uint32_t v) const { return v | (__vcmpgeu4(v, 0x41414141u) & __vcmpleu4(v, 0x5a5a5a5au) & 0x20202020u); } };

// dst[i] = f(src[i]) for i < n over the warp; f maps 4 packed bytes at once.  The body is stored as aligned words, each assembled from
// the two aligned source words it straddles (an aligned word that holds a byte of src lies inside src's allocation).
template <class F> __device__ __forceinline__ void warp_map(uint8_t* dst, const uint8_t* src, uint64_t n, F f) {
    const unsigned lane = threadIdx.x & 31;
    const uint64_t h4 = (4 - (reinterpret_cast<uintptr_t>(dst) & 3)) & 3, head = n < h4 ? n : h4;
    if (lane < head) dst[lane] = (uint8_t)f((uint32_t)src[lane]);
    const uint64_t nw = (n - head) >> 2;
    const uint8_t* s = src + head;
    const uint32_t sh = (uint32_t)(reinterpret_cast<uintptr_t>(s) & 3) * 8;
    const uint32_t* a = reinterpret_cast<const uint32_t*>(reinterpret_cast<uintptr_t>(s) & ~(uintptr_t)3);
    uint32_t* d = reinterpret_cast<uint32_t*>(dst + head);
    for (uint64_t w = lane; w < nw; w += 32) d[w] = f(sh ? __funnelshift_r(a[w], a[w + 1], sh) : a[w]);
    const uint64_t t0 = head + 4 * nw;
    if (t0 + lane < n) dst[t0 + lane] = (uint8_t)f((uint32_t)src[t0 + lane]);
}

// name of contig id, or "*" for id < 0
__device__ __forceinline__ const uint8_t* name_of(const FmtArgs& A, int32_t id, uint32_t* len) {
    if (id < 0) { *len = 1; return reinterpret_cast<const uint8_t*>("*"); }
    *len = A.name_off[id + 1] - A.name_off[id];
    return A.names + A.name_off[id];
}

// one float value: slot s of the host-formatted list.  Returns its text length (0 while measuring: added once the texts exist).
template <int M> __device__ __forceinline__ int float_text(const FmtArgs& A, uint64_t s, uint32_t bits, uint8_t* o) {
    if (M == FM_LIST) { A.fbits[s] = bits; return 0; }
    if (M == FM_MEASURE) return 0;
    const uint64_t a = A.foff[s], b = A.foff[s + 1];
    for (uint64_t j = a; j < b; j++) o[j - a] = A.ftext[j];
    return (int)(b - a);
}

// FormatAlignment of output line A.first + kk.  All lanes run the same control flow; lane 0 writes the short serial parts, the warp the long ones.
template <int M> __device__ void format_line(const FmtArgs& A, uint64_t kk, const uint8_t* tbl) {
    constexpr bool W = M == FM_EMIT;
    const unsigned lane = threadIdx.x & 31;
    const uint64_t k = A.sel ? A.sel[A.first + kk] : A.first + kk;
    const uint8_t* r = A.all + A.all_start[A.perm[k]];
    const uint64_t rec = (uint64_t)rd32(r) + 4;
    const uint32_t l_name = r[12], mapq = A.mapq[k], ncig = rd16(r + 16), flag = A.flag[k];
    const int32_t refid = (int32_t)rd32(r + 4), nref = (int32_t)rd32(r + 24), tlen = (int32_t)rd32(r + 32);
    const int32_t pos1 = (int32_t)(rd32(r + 8) + 1u), pnext1 = (int32_t)(rd32(r + 28) + 1u);   // int32(x) + 1 wraps as in Go
    const uint64_t L = rd32(r + 20);                                      // l_seq >= 0 (checked at ingest)
    const uint64_t lq = l_name - 1;
    uint32_t lrn, lrx;
    const uint8_t* rn = name_of(A, refid, &lrn);
    // RNEXT: "*" below 0, "=" when its NAME equals RNAME's (parseBamAlignment :340-347 compares strings), else the name
    const uint8_t* rx;
    if (nref >= 0 && A.canon[nref] == A.canon[refid < 0 ? A.n_contigs : refid]) { rx = reinterpret_cast<const uint8_t*>("="); lrx = 1; }
    else rx = name_of(A, nref, &lrx);
    uint8_t* o = W ? A.out + A.line_off[kk] : nullptr;
    const int lf = ndig(flag), lp = sdig(pos1), lm = ndig(mapq), lpn = sdig(pnext1), lt = sdig(tlen);
    // QNAME FLAG RNAME POS MAPQ
    uint64_t x = lq + 1;
    const uint64_t xf = x, xr = xf + lf + 1, xp = xr + lrn + 1, xm = xp + lp + 1;
    x = xm + lm + 1;
    if (W) {
        warp_map(o, r + 36, lq, Ident());
        for (uint32_t j = lane; j < lrn; j += 32) o[xr + j] = rn[j];
        if (lane == 0) { o[lq] = '\t'; put_dec(o + xf, flag, lf); o[xf + lf] = '\t'; }
        else if (lane == 1) { o[xr + lrn] = '\t'; put_dec(o + xp, pos1, lp); o[xp + lp] = '\t'; }
        else if (lane == 2) { put_dec(o + xm, mapq, lm); o[xm + lm] = '\t'; }
    }
    // CIGAR: "*" for no operations, else <len><op> per operation, 32 operations per step
    const uint8_t* cw = r + 36 + l_name;
    if (ncig == 0) { if (W && lane == 0) o[x] = '*'; x++; }
    bool bad_op = false;
    for (uint32_t c0 = 0; c0 < ncig; c0 += 32) {
        const uint32_t i = c0 + lane;
        uint32_t w = 0; int len = 0;
        if (i < ncig) { w = rd32(cw + 4ull * i); len = ndig(w >> 4) + 1; bad_op |= (w & 15u) > 8u; }
        const int incl = warp_incl(len), tot = __shfl_sync(FULL_MASK, incl, 31);
        if (W && i < ncig) { put_dec(o + x + incl - len, w >> 4, len - 1); o[x + incl - 1] = tbl[16 + min(w & 15u, 8u)]; }
        x += tot;
    }
    if (M == FM_MEASURE && bad_op) atomicOr(A.small, FE_CIGAR_OP);
    // RNEXT PNEXT TLEN
    const uint64_t xx = x + 1, xpn = xx + lrx + 1, xt = xpn + lpn + 1;
    x = xt + lt + 1;
    if (W) {
        for (uint32_t j = lane; j < lrx; j += 32) o[xx + j] = rx[j];
        if (lane == 0) { o[xx - 1] = '\t'; o[xx + lrx] = '\t'; }
        else if (lane == 1) { put_dec(o + xpn, pnext1, lpn); o[xpn + lpn] = '\t'; }
        else if (lane == 2) { put_dec(o + xt, tlen, lt); o[xt + lt] = '\t'; }
    }
    // SEQ (nibble -> "=ACMGRSVTWYHKDBN"; l_seq 0 gives an empty field) and QUAL (+ 33)
    const uint8_t* sq = cw + 4ull * ncig;
    const uint64_t ls = (L + 1) >> 1;
    if (W) {
        for (uint64_t j = lane; j < ls; j += 32) {
            const uint8_t b = sq[j];
            o[x + 2 * j] = tbl[b >> 4];
            if (2 * j + 1 < L) o[x + 2 * j + 1] = tbl[b & 15];
        }
        if (lane == 0) o[x + L] = '\t';
        warp_map(o + x + L + 1, A.qual ? A.qual + A.qoff[k] : sq + ls, L, Phred33());
    }
    x += 2 * L + 1;
    // optional fields in record order: "\tTG:T:value"; every integer type prints as i (parseBam* widens to int64)
    uint64_t t = 36 + l_name + 4ull * ncig + ls + L;
    const uint64_t fb = A.fbase ? A.fbase[kk] : 0;                        // (no float values in the lines: no slots)
    uint64_t fj = 0;                                                      // float values of this line so far
    while (t + 3 <= rec) {
        const uint8_t t0 = r[t], t1 = r[t + 1], ty = r[t + 2];
        const uint64_t fe = tagwalk::field_end(r, t, rec);
        if (A.drop && tagwalk::dropped(A.drop, t0, t1)) { t = fe; continue; }   // no text, no float slot
        t += 3;
        const bool integer = ty == 'c' || ty == 'C' || ty == 's' || ty == 'S' || ty == 'i' || ty == 'I';
        if (W && lane == 0) { o[x] = '\t'; o[x + 1] = t0; o[x + 2] = t1; o[x + 3] = ':'; o[x + 4] = integer ? 'i' : ty; o[x + 5] = ':'; }
        x += 6;
        if (integer) {
            int64_t v; int sz;
            switch (ty) {
                case 'c': v = (int8_t)r[t]; sz = 1; break;
                case 'C': v = r[t]; sz = 1; break;
                case 's': v = (int16_t)rd16(r + t); sz = 2; break;
                case 'S': v = rd16(r + t); sz = 2; break;
                case 'i': v = (int32_t)rd32(r + t); sz = 4; break;
                default: v = rd32(r + t); sz = 4; break;
            }
            const int nd = sdig(v);
            if (W && lane == 0) put_dec(o + x, v, nd);
            x += nd; t += sz;
        } else if (ty == 'A') {
            if (W && lane == 0) o[x] = r[t];
            x += 1; t += 1;
        } else if (ty == 'f') {
            int fl = 0;
            if (lane == 0) fl = float_text<M>(A, fb + fj, rd32(r + t), W ? o + x : nullptr);
            x += __shfl_sync(FULL_MASK, fl, 0); t += 4; fj++;
        } else if (ty == 'Z' || ty == 'H') {                              // H: the stored hex digits in lower case (AppendUint(b, 16))
            const uint64_t n = fe - 1 - t;
            if (W) { if (ty == 'Z') warp_map(o + x, r + t, n, Ident()); else warp_map(o + x, r + t, n, Lower()); }
            x += n; t = fe;
        } else if (ty == 'B') {                                           // subtype, then ","value per element over the warp
            const uint8_t sub = r[t];
            const uint32_t cnt = rd32(r + t + 1);
            t += 5;
            if (W && lane == 0) o[x] = sub;
            x += 1;
            const int es = tagwalk::elem_size(sub);
            for (uint32_t e0 = 0; e0 < cnt; e0 += 32) {
                const uint32_t e = e0 + lane;
                int len = 0; int64_t v = 0;
                const uint8_t* q = r + t + (uint64_t)es * e;
                uint8_t* oe = nullptr;
                if (e < cnt) {
                    switch (sub) {
                        case 'c': v = (int8_t)q[0]; break;
                        case 'C': v = q[0]; break;
                        case 's': v = (int16_t)rd16(q); break;
                        case 'S': v = rd16(q); break;
                        case 'i': v = (int32_t)rd32(q); break;
                        default: v = rd32(q); break;
                    }
                    len = 1 + (sub == 'f' ? (M == FM_EMIT ? (int)(A.foff[fb + fj + e + 1] - A.foff[fb + fj + e]) : 0) : sdig(v));
                }
                const int incl = warp_incl(len), tot = __shfl_sync(FULL_MASK, incl, 31);
                if (e < cnt) {
                    if (W) { oe = o + x + incl - len; oe[0] = ','; }
                    if (sub == 'f') float_text<M>(A, fb + fj + e, (uint32_t)v, W ? oe + 1 : nullptr);
                    else if (W) put_dec(oe + 1, v, len - 1);
                }
                x += tot;
            }
            if (sub == 'f') fj += cnt;
            t = fe;
        } else break;                                                     // (the ingest accepted no other type)
    }
    x += 1;
    if (W && lane == 0) o[x - 1] = '\n';
    if (M == FM_MEASURE && lane == 0) {
        const bool big = x + (uint64_t)gofloat::MAX_LEN * fj >= (1ull << 32);
        A.len[kk] = big ? 0u : (uint32_t)x; A.nf[kk] = (uint32_t)fj;
        if (big) atomicOr(A.small, FE_LINE_LIMIT);
        if (fj) atomicAdd(A.small + 1, (unsigned long long)fj);
    }
}

template <int M> __global__ void __launch_bounds__(256) sam_out_kernel(FmtArgs A) {
    __shared__ uint8_t tbl[32];                                           // [0, 16): SEQ nibble -> base, [16, 25): CIGAR op -> "MIDNSHP=X"
    if (threadIdx.x < 16) tbl[threadIdx.x] = (uint8_t)"=ACMGRSVTWYHKDBN"[threadIdx.x];
    else if (threadIdx.x < 25) tbl[threadIdx.x] = (uint8_t)"MIDNSHP=X"[threadIdx.x - 16];
    __syncthreads();
    const uint64_t kk = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (kk >= A.n) return;
    format_line<M>(A, kk, tbl);
}

// line length += the texts of its float values (slots fbase[kk] .. fbase[kk] + nf[kk])
__global__ void __launch_bounds__(256) sam_out_flen_kernel(uint64_t n, const uint64_t* __restrict__ fbase, const uint32_t* __restrict__ nf, const uint64_t* __restrict__ foff, uint32_t* __restrict__ len) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) len[i] += (uint32_t)(foff[fbase[i] + nf[i]] - foff[fbase[i]]);
}

// @SQ names and their canon (first index with the same name), uploaded once per context
int sam_out_tables(elp_ctx* c) {
    if (c->sam_out) return E_OK;
    SamOutState* S = new SamOutState();
    c->sam_out = S;
    std::vector<uint8_t> names; std::vector<uint32_t> off(1, 0); std::vector<int32_t> canon(c->n_contigs + 1, -1);
    std::map<std::string, int32_t> first;
    for (int i = 0; i < c->n_contigs; i++) {
        const std::string& s = c->contig_names[i];
        names.insert(names.end(), s.begin(), s.end()); off.push_back((uint32_t)names.size());
        canon[i] = first.emplace(s, i).first->second;
    }
    auto star = first.find("*");
    if (star != first.end()) canon[c->n_contigs] = star->second;
    CUDA_TRY(c, cudaMalloc(&S->d_names, std::max<size_t>(names.size(), 1)));
    CUDA_TRY(c, cudaMalloc(&S->d_name_off, off.size() * 4));
    CUDA_TRY(c, cudaMalloc(&S->d_canon, canon.size() * 4));
    CUDA_TRY(c, cudaMalloc(&S->d_small, 16));
    CUDA_TRY(c, cudaMemcpy(S->d_names, names.data(), names.size(), cudaMemcpyHostToDevice));
    CUDA_TRY(c, cudaMemcpy(S->d_name_off, off.data(), off.size() * 4, cudaMemcpyHostToDevice));
    CUDA_TRY(c, cudaMemcpy(S->d_canon, canon.data(), canon.size() * 4, cudaMemcpyHostToDevice));
    return E_OK;
}

// the refusals of elp_fetch_sam and elp_fetch_sam_bytes (no device work but the record filters' selection); *sel: that selection or null
int sam_out_check(elp_ctx* c, uint64_t first, uint64_t n, const uint32_t** sel) {
    if (!c->sorted) return c->fail(E_STATE, "elp_fetch_sam before elp_sort_markdup");
    if (c->bam_reads != c->n) return c->fail(E_STATE, "elp_fetch_sam: not every read of this context came in through elp_append_bam or elp_append_sam");
    if (c->n_cleaned) return c->fail(E_STATE, "elp_fetch_sam: elp_clean_sam rewrote %llu CIGARs; the stored records still carry the old ones (use elp_fetch)", (unsigned long long)c->n_cleaned);
    if (c->n_contigs > 0 && !c->has_contig_names) return c->fail(E_INVAL, "elp_fetch_sam: the context was created without elp_config.contig_names, so RNAME / RNEXT cannot be written");
    if (c->n_sam_lost_names) return c->fail(E_STATE, "elp_fetch_sam: %llu SAM lines of this context have an RNAME or RNEXT that is not an @SQ name (or RNEXT '=' with such an RNAME); their stored records cannot reproduce it (use elp_fetch_bam)", (unsigned long long)c->n_sam_lost_names);
    uint64_t n_out = 0;
    TRY(out_select(c, sel, &n_out));
    if (first + n > n_out) {
        if (*sel) return c->fail(E_INVAL, "elp_fetch_sam: range [%llu,%llu) exceeds the %llu output records that pass the record filters (elp_n_output)", (unsigned long long)first, (unsigned long long)(first + n), (unsigned long long)n_out);
        return c->fail(E_INVAL, "elp_fetch_sam: range [%llu,%llu) exceeds %llu reads", (unsigned long long)first, (unsigned long long)(first + n), (unsigned long long)c->n);
    }
    return E_OK;
}

// measure (and the float step): line lengths scanned into off_stage[0..n], *total bytes; A is left ready for the emit pass
int sam_out_prepare(elp_ctx* c, uint64_t first, uint64_t n, const uint32_t* sel, uint64_t* total, FmtArgs* Aout) {
    TRY(sam_out_tables(c));
    SamOutState& S = *c->sam_out;
    cudaStream_t s = c->stream;
    TRY(grow(c, c->scan_tmp, n + 8, 0)); TRY(grow(c, c->off_stage, n + 2, 0)); TRY(grow(c, S.nf, n + 8, 0));
    FmtArgs A{};
    A.n = n; A.first = first; A.sel = sel; A.drop = c->out_fields ? c->d_out_drop : nullptr; A.perm = c->perm.p; A.all_start = c->bam_all_off.p; A.all = c->bam_all.p;
    A.flag = c->s_flag.p; A.mapq = c->s_mapq.p; A.qoff = c->s_out_off.p; A.qual = c->qual_out_valid ? c->qual_out.p : nullptr;
    A.names = S.d_names; A.name_off = S.d_name_off; A.canon = S.d_canon; A.n_contigs = c->n_contigs;
    A.len = c->scan_tmp.p; A.nf = S.nf.p; A.small = S.d_small;
    CUDA_TRY(c, cudaMemsetAsync(S.d_small, 0, 16, s));
    c->begin("sam_out_measure", (double)c->n_bam * (double)n / (double)std::max<uint64_t>(c->n, 1));
    sam_out_kernel<FM_MEASURE><<<nblk(n * 32, 256), 256, 0, s>>>(A);
    c->end(); LAUNCH_CHECK(c);
    TRY(exclusive_scan_u32_to_u64(c, c->scan_tmp.p, c->off_stage.p, n));
    unsigned long long small[2];
    CUDA_TRY(c, cudaMemcpyAsync(small, S.d_small, 16, cudaMemcpyDeviceToHost, s));
    CUDA_TRY(c, cudaMemcpyAsync(total, c->off_stage.p + n, 8, cudaMemcpyDeviceToHost, s));
    CUDA_TRY(c, cudaStreamSynchronize(s));
    if (small[0] & FE_CIGAR_OP) return c->fail(E_BAM, "elp_fetch_sam: a CIGAR operation code above 8 (cigarOps of the reference has 9 entries, sam/bam-files.go:356-362)");
    if (small[0] & FE_LINE_LIMIT) return c->fail(E_LIMIT, "elp_fetch_sam: a SAM line of 2^32 bytes or more");
    const uint64_t nfl = small[1];
    if (nfl) {   // float values: bits listed on the device, formatted on the host (Go's shortest 'g'), texts uploaded
        TRY(grow(c, S.fbase, n + 2, 0)); TRY(grow(c, S.fbits, nfl + 1, 0)); TRY(grow(c, S.foff, nfl + 2, 0));
        TRY(exclusive_scan_u32_to_u64(c, S.nf.p, S.fbase.p, n));
        A.fbase = S.fbase.p; A.fbits = S.fbits.p;
        c->begin("sam_out_float", (double)c->n_bam * (double)n / (double)std::max<uint64_t>(c->n, 1) + 4.0 * (double)nfl);
        sam_out_kernel<FM_LIST><<<nblk(n * 32, 256), 256, 0, s>>>(A);
        c->end(); LAUNCH_CHECK(c);
        std::vector<uint32_t> bits(nfl);
        CUDA_TRY(c, cudaMemcpyAsync(bits.data(), S.fbits.p, nfl * 4, cudaMemcpyDeviceToHost, s));
        CUDA_TRY(c, cudaStreamSynchronize(s));
        std::vector<char> txt(nfl * gofloat::MAX_LEN); std::vector<uint8_t> tl(nfl);
        const int threads = nfl >= (1u << 16) ? (int)std::min(16u, std::max(1u, std::thread::hardware_concurrency())) : 1;
        pool_for(nfl, threads, [&](size_t i) { tl[i] = (uint8_t)gofloat::format_f32(bits[i], &txt[i * gofloat::MAX_LEN]); });
        std::vector<uint64_t> foff(nfl + 1, 0);
        for (uint64_t i = 0; i < nfl; i++) foff[i + 1] = foff[i] + tl[i];
        std::vector<uint8_t> packed(foff[nfl]);
        for (uint64_t i = 0; i < nfl; i++) std::memcpy(&packed[foff[i]], &txt[i * gofloat::MAX_LEN], tl[i]);
        TRY(grow(c, S.ftext, foff[nfl] + 1, 0));
        CUDA_TRY(c, cudaMemcpyAsync(S.ftext.p, packed.data(), foff[nfl], cudaMemcpyHostToDevice, s));
        CUDA_TRY(c, cudaMemcpyAsync(S.foff.p, foff.data(), (nfl + 1) * 8, cudaMemcpyHostToDevice, s));
        A.ftext = S.ftext.p; A.foff = S.foff.p;
        c->begin("sam_out_float", 20.0 * (double)n);
        sam_out_flen_kernel<<<nblk(n, 256), 256, 0, s>>>(n, S.fbase.p, S.nf.p, S.foff.p, c->scan_tmp.p);
        c->end(); LAUNCH_CHECK(c);
        TRY(exclusive_scan_u32_to_u64(c, c->scan_tmp.p, c->off_stage.p, n));
        CUDA_TRY(c, cudaMemcpyAsync(total, c->off_stage.p + n, 8, cudaMemcpyDeviceToHost, s));
        CUDA_TRY(c, cudaStreamSynchronize(s));   // (packed / foff are pageable host memory)
    }
    A.line_off = c->off_stage.p;
    *Aout = A;
    return E_OK;
}

}  // namespace

extern "C" uint64_t elp_fetch_sam_bytes(elp_ctx* c, uint64_t first, uint64_t n) {
    if (!c || n == 0) return 0;
    cudaSetDevice(c->device);
    const uint32_t* sel = nullptr;
    if (sam_out_check(c, first, n, &sel)) return 0;
    uint64_t total = 0; FmtArgs A;
    if (sam_out_prepare(c, first, n, sel, &total, &A)) return 0;
    return total;
}

extern "C" int elp_fetch_sam(elp_ctx* c, uint64_t first, uint64_t n, char* out, uint64_t capacity, uint64_t* line_off) {
    if (!c || (!out && n)) return ELP_EINVAL;
    cudaSetDevice(c->device);
    const uint32_t* sel = nullptr;
    TRY(sam_out_check(c, first, n, &sel));
    if (n == 0) { if (line_off) line_off[0] = 0; return ELP_OK; }
    uint64_t total = 0; FmtArgs A;
    TRY(sam_out_prepare(c, first, n, sel, &total, &A));
    if (total > capacity) return c->fail(E_INVAL, "elp_fetch_sam: output buffer too small (%llu > %llu)", (unsigned long long)total, (unsigned long long)capacity);
    TRY(grow(c, c->bam_raw, total + 64, 0));                              // staging of the text
    A.out = c->bam_raw.p;
    c->begin("sam_out_emit", (double)c->n_bam * (double)n / (double)std::max<uint64_t>(c->n, 1) + (double)total);
    sam_out_kernel<FM_EMIT><<<nblk(n * 32, 256), 256, 0, c->stream>>>(A);
    c->end(); LAUNCH_CHECK(c);
    CUDA_TRY(c, cudaMemcpyAsync(out, c->bam_raw.p, total, cudaMemcpyDeviceToHost, c->stream));
    if (line_off) CUDA_TRY(c, cudaMemcpyAsync(line_off, c->off_stage.p, (n + 1) * 8, cudaMemcpyDeviceToHost, c->stream));
    CUDA_TRY(c, cudaStreamSynchronize(c->stream));
    return ELP_OK;
}
