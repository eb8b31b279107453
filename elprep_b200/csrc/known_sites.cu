// known_sites.cu -- --known-sites on the device: .elsites files read, parsed, sorted and flattened into the known-sites table
// (elp_load_known_sites).
//
// The reference loads every file with intervals.FromElsitesFile (intervals/intervals.go:199-254), appends the intervals of each
// chromosome (NewBaseRecalibrator, filters/bqsr.go:424-443), then sorts (ParallelSortByStart) and flattens (ParallelFlatten) each.
//   host           checks the header and streams the rest of each file through two page-locked chunks: the upload of chunk k+1 runs
//                  while the kernels of chunk k do; the bytes after the last '\n' of a chunk are carried into the next one
//   sites_lines    the line finder of elp_append_sam (text_parse.cuh)
//   sites_parse    one thread per line, a warp over 32 consecutive lines: the three fields, strconv.ParseInt, the chromosome name (each
//                  run of equal names in a warp is looked up once: files are grouped by chromosome); then one (contig, start, end) per
//                  @SQ line with that name, at its scanned offset
//   sites_sort     the onesweep radix sort of contig << 32 | (start ^ 2^31), the end as payload
//   sites_flatten  one prefix max over contig << 32 | (end ^ 2^31): interval i opens a group iff it is the first of its contig or its start
//                  lies above every earlier end of its contig; the group heads are compacted and each group keeps the max of its ends
// A VCF in the list (plain or BGZF, see vcf.cuh) gives the intervals of intervals.FromVcfFile (intervals/intervals.go:306-338):
//   host           the header, parsed as ParseHeader does (BGZF: its leading blocks inflated with zlib); then the data lines go through
//                  the two chunks as reference_load.cu streams FASTA (plain text uploaded, BGZF blocks inflated by bgzf_inflate), the
//                  partial line at a chunk's end carried on the device
//   sites_lines    the same line finder
//   vcf_parse      a warp per 32 lines (vcf.cuh) into the arrays sites_parse fills; sites_sort, sites_flatten and the install follow as
//                  for .elsites lines, over the intervals of every file in list order
// Nothing is installed before every file was read and every line accepted; the new table is one allocation (ContigTable::block).
#include <algorithm>
#include <cerrno>
#include <cstdio>
#include <cstring>
#include <vector>
#include <zlib.h>
#include "ctx.h"
#include "text_parse.cuh"
#include "file_stage.cuh"
#include "bgzf_scan.hpp"
#include "vcf.cuh"
#include "../../include/elprep_b200.h"

namespace {

const char SITES_HEADER[] = "# elsites format version 1.0\n";   // intervals.ElsitesHeader (intervals/intervals.go:176)
constexpr uint64_t SITES_HEADER_LEN = sizeof(SITES_HEADER) - 1;
constexpr uint64_t SITES_MAX_LINE = 65536;                     // bufio.MaxScanTokenSize: a longer line stops the reference's scanner
constexpr uint64_t SITES_CHUNK_DEFAULT = 32ull << 20;
constexpr uint64_t VCF_FRONT = VCF_MAX_LINE;                   // device bytes ahead of a VCF chunk's text: room for the carried partial line
constexpr uint64_t BGZF_MAX_BLOCK = 65536;

}  // namespace

// page-locked and device staging, reused by every call on the context
struct SitesStage {
    FileStage f;                                                 // the two chunks (file_stage.cuh); a carried partial line sits in front of the file bytes
    FileStage v;                                                 // the chunks of VCF files: VCF_FRONT device bytes ahead of each chunk's text
    DBuf<uint8_t> tb[2];                                         // inflated BGZF VCF text, VCF_FRONT bytes in
    DBuf<unsigned long long> d_small;                            // [0] first error (line << 8 | SitesErr or VcfErr), [1] unmatched lines, [2] QUAL band count
    HBuf<unsigned long long> h_small;                            // [0, 1] copies, [2] '\n' count, [3] intervals, [4] virtual line end, [5, 8) VCF words
};

void free_state(SitesStage* S) { delete S; }

namespace {

// why a line fails; the smallest (line << 8 | code) of a file is reported
enum SitesErr : uint32_t { KS_FIELDS = 1, KS_START, KS_END, KS_LONG };
const char* sites_err_text(uint32_t e) {
    switch (e) {
        case KS_FIELDS: return "invalid sites line (no chromosome before the first tab, or no second tab)";
        case KS_START: return "start: strconv.ParseInt(s, 10, 32) fails";
        case KS_END: return "end: strconv.ParseInt(s, 10, 32) fails";
        case KS_LONG: return "line of 65536 bytes or more (bufio.Scanner: token too long)";
        default: return "?";
    }
}

// ---- sites_parse ----
struct SitesArgs {
    const uint8_t* text; const uint64_t* ls; uint64_t n_lines;
    uint64_t line0;                                  // line number (header = 0) of the chunk's first line within its file
    NameDict dict;
    int32_t* ent; int32_t* start; int32_t* end;      // per accepted line: name entry (-1: unknown), start, end
    uint32_t* emit;                                  // per line: intervals it contributes (one per @SQ line with its name)
    unsigned long long* small;
};

// FromElsitesFile's loop body for one line (intervals.go:221-247), after bufio.ScanLines dropped the '\n' and one '\r' before it
__global__ void __launch_bounds__(256) sites_parse_kernel(SitesArgs A) {
    const unsigned lane = threadIdx.x & 31;
    const uint64_t k = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const bool live = k < A.n_lines;
    uint64_t s0 = 0, nn = 0;                         // the line's start and its name's length
    uint32_t err = 0;
    int64_t st = 0, en = 0;
    if (live) {
        s0 = A.ls[k];
        const uint64_t raw = A.ls[k + 1] - 1 - s0;
        const uint8_t* p = A.text + s0;
        uint64_t n = raw;
        if (n && p[n - 1] == '\r') n--;
        if (raw >= SITES_MAX_LINE) err = KS_LONG;
        else {
            uint64_t i = 0;
            while (i < n && p[i] != '\t') i++;
            uint64_t j = i + 1;
            while (j < n && p[j] != '\t') j++;
            if (i == 0 || i >= n || j >= n) err = KS_FIELDS;
            else if (!parse_dec(p + i + 1, j - i - 1, true, INT32_MIN, INT32_MAX, &st)) err = KS_START;
            else if (!parse_dec(p + j + 1, n - j - 1, true, INT32_MIN, INT32_MAX, &en)) err = KS_END;
            nn = i;
        }
    }
    // the name: a line whose name equals the previous lane's takes that lane's entry; the first line of each run looks it up
    const bool named = live && !err;
    const uint64_t ps0 = __shfl_up_sync(FULL_MASK, s0, 1), pnn = __shfl_up_sync(FULL_MASK, nn, 1);
    const bool pnamed = __shfl_up_sync(FULL_MASK, (int)named, 1) != 0;
    bool lead = named;
    if (named && lane > 0 && pnamed && pnn == nn) {
        const uint8_t* p = A.text + s0; const uint8_t* q = A.text + ps0;
        uint64_t j = 0;
        while (j < nn && p[j] == q[j]) j++;
        lead = j < nn;
    }
    int e = lead ? name_entry(A.dict, A.text + s0, nn) : -1;
    const unsigned below = __ballot_sync(FULL_MASK, lead) & (0xffffffffu >> (31 - lane));
    const int e_lead = __shfl_sync(FULL_MASK, e, below ? 31 - __clz(below) : (int)lane);
    if (named && !lead) e = e_lead;
    const uint32_t m = named && e >= 0 ? A.dict.all_off[e + 1] - A.dict.all_off[e] : 0;
    if (live) {
        A.emit[k] = m;
        if (named) { A.ent[k] = e; A.start[k] = (int32_t)st; A.end[k] = (int32_t)en; }
        else atomicMin(A.small, ((unsigned long long)(A.line0 + k) << 8) | err);
    }
    const unsigned um = __ballot_sync(FULL_MASK, named && m == 0);   // valid lines on a chromosome that is no @SQ SN ("*" included)
    if (lane == 0 && um) atomicAdd(A.small + 1, (unsigned long long)__popc(um));
}

// the intervals of the accepted lines, at their scanned offsets: key contig << 32 | (start ^ 2^31), payload end
__global__ void __launch_bounds__(256) sites_emit_kernel(uint64_t n, const int32_t* __restrict__ ent, const int32_t* __restrict__ start, const int32_t* __restrict__ end,
                                                          const uint32_t* __restrict__ emit, const uint64_t* __restrict__ off, NameDict D,
                                                          uint64_t* __restrict__ keys, uint32_t* __restrict__ vals) {
    const uint64_t k = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= n) return;
    const uint32_t m = emit[k];
    if (!m) return;
    const uint64_t o = off[k];
    const int32_t* ids = D.all + D.all_off[ent[k]];
    const uint32_t lo = (uint32_t)start[k] ^ 0x80000000u, v = (uint32_t)end[k];
    for (uint32_t j = 0; j < m; j++) { keys[o + j] = ((uint64_t)(uint32_t)ids[j] << 32) | lo; vals[o + j] = v; }
}

// ---- sites_flatten ----
// Over the sorted intervals, v_i = contig_i << 32 | (end_i ^ 2^31).  Contigs never decrease, so the max of v over the intervals before i
// carries contig_i exactly when i is not the first of its contig, and then its low word is the largest earlier end of the contig.
// Flatten (intervals.go:101-117) extends the open group while start <= its end; a closed group ended below the start of the group after
// it, so "start_i > every earlier end of the contig" is exactly "start_i > the end of the open group": i opens a group.
constexpr int FL_T = 256, FL_ITEMS = 8, FL_TILE = FL_T * FL_ITEMS;

__device__ __forceinline__ uint64_t fl_val(uint64_t key, uint32_t end) { return (key & 0xffffffff00000000ull) | (end ^ 0x80000000u); }

__device__ __forceinline__ uint64_t block_max(uint64_t m, uint64_t* sh) {   // every thread gets the max over the block
    for (int o = 16; o; o >>= 1) m = max(m, (uint64_t)__shfl_xor_sync(FULL_MASK, m, o));
    if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = m;
    __syncthreads();
    m = 0;
    for (int w = 0; w < FL_T / 32; w++) m = max(m, sh[w]);
    return m;
}

__global__ void __launch_bounds__(FL_T) sites_tile_max_kernel(const uint64_t* __restrict__ keys, const uint32_t* __restrict__ ends, uint64_t n, uint64_t* __restrict__ tmax) {
    __shared__ uint64_t sh[FL_T / 32];
    const uint64_t t0 = (uint64_t)blockIdx.x * FL_TILE;
    uint64_t m = 0;
#pragma unroll
    for (int j = 0; j < FL_ITEMS; j++) { const uint64_t i = t0 + (uint64_t)j * FL_T + threadIdx.x; if (i < n) m = max(m, fl_val(keys[i], ends[i])); }
    m = block_max(m, sh);
    if (threadIdx.x == 0) tmax[blockIdx.x] = m;
}

// tmax[t] <- the max over the tiles before t (0 for tile 0), in one CTA
__global__ void __launch_bounds__(1024) sites_tile_scan_kernel(uint64_t* __restrict__ tmax, uint64_t tiles) {
    __shared__ uint64_t wsum[32];
    __shared__ uint64_t carry;
    const unsigned lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (threadIdx.x == 0) carry = 0;
    __syncthreads();
    for (uint64_t base = 0; base < tiles; base += 1024) {
        const uint64_t i = base + threadIdx.x;
        const uint64_t v = i < tiles ? tmax[i] : 0;
        uint64_t x = v;
        for (int o = 1; o < 32; o <<= 1) { const uint64_t y = __shfl_up_sync(FULL_MASK, x, o); if (lane >= (unsigned)o) x = max(x, y); }
        if (lane == 31) wsum[warp] = x;
        __syncthreads();
        if (warp == 0) {
            uint64_t w = wsum[lane];
            for (int o = 1; o < 32; o <<= 1) { const uint64_t y = __shfl_up_sync(FULL_MASK, w, o); if (lane >= (unsigned)o) w = max(w, y); }
            wsum[lane] = w;
        }
        __syncthreads();
        uint64_t ex = __shfl_up_sync(FULL_MASK, x, 1);
        if (lane == 0) ex = 0;
        if (warp) ex = max(ex, wsum[warp - 1]);
        const uint64_t c0 = carry, total = wsum[31];
        __syncthreads();
        if (i < tiles) tmax[i] = max(c0, ex);
        if (threadIdx.x == 0) carry = max(c0, total);
        __syncthreads();
    }
}

// head[i] = 1 iff sorted interval i opens a group; tpre: the exclusive tile maxima of sites_tile_scan_kernel
__global__ void __launch_bounds__(FL_T) sites_head_kernel(const uint64_t* __restrict__ keys, const uint32_t* __restrict__ ends, uint64_t n,
                                                          const uint64_t* __restrict__ tpre, uint32_t* __restrict__ head) {
    __shared__ uint64_t wsum[FL_T / 32];
    const unsigned lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const uint64_t i0 = (uint64_t)blockIdx.x * FL_TILE + (uint64_t)threadIdx.x * FL_ITEMS;
    uint64_t kk[FL_ITEMS], v[FL_ITEMS], m = 0;
#pragma unroll
    for (int j = 0; j < FL_ITEMS; j++) {
        const uint64_t i = i0 + j;
        kk[j] = i < n ? keys[i] : 0;
        v[j] = i < n ? fl_val(kk[j], ends[i]) : 0;
        m = max(m, v[j]);
    }
    uint64_t x = m;   // exclusive max over the threads before this one in the tile
    for (int o = 1; o < 32; o <<= 1) { const uint64_t y = __shfl_up_sync(FULL_MASK, x, o); if (lane >= (unsigned)o) x = max(x, y); }
    if (lane == 31) wsum[warp] = x;
    __syncthreads();
    uint64_t run = __shfl_up_sync(FULL_MASK, x, 1);
    if (lane == 0) run = 0;
    for (unsigned w = 0; w < warp; w++) run = max(run, wsum[w]);
    run = max(run, tpre[blockIdx.x]);
#pragma unroll
    for (int j = 0; j < FL_ITEMS; j++) {
        const uint64_t i = i0 + j;
        if (i >= n) break;
        const int32_t s = (int32_t)((uint32_t)kk[j] ^ 0x80000000u), e = (int32_t)((uint32_t)run ^ 0x80000000u);
        head[i] = i == 0 || (run >> 32) != (kk[j] >> 32) || s > e;
        run = max(run, v[j]);
    }
}

// group g = gid[i] + head[i] - 1: its head writes the start, every member raises the end (biased, so that unsigned max is signed max);
// first[contig] = the contig's first group
__global__ void __launch_bounds__(256) sites_compact_kernel(const uint64_t* __restrict__ keys, const uint32_t* __restrict__ ends, uint64_t n, const uint32_t* __restrict__ head,
                                                             const uint64_t* __restrict__ gid, int32_t* __restrict__ out, uint64_t* __restrict__ first) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint64_t key = keys[i];
    const uint32_t h = head[i];
    const uint64_t g = gid[i] + h - 1;
    if (h) out[2 * g] = (int32_t)((uint32_t)key ^ 0x80000000u);
    atomicMax(reinterpret_cast<unsigned*>(out + 2 * g + 1), ends[i] ^ 0x80000000u);
    if (i == 0 || (keys[i - 1] >> 32) != (key >> 32)) first[key >> 32] = g;
}

__global__ void __launch_bounds__(256) sites_unbias_kernel(uint64_t n_groups, int32_t* __restrict__ out) {
    const uint64_t g = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (g < n_groups) out[2 * g + 1] = (int32_t)((uint32_t)out[2 * g + 1] ^ 0x80000000u);
}

// ---- host side ----
struct SitesScratch {   // per call; freed on return
    DBuf<uint32_t> cnt, emit, vals_a, vals_b, head; DBuf<uint64_t> cnt_off, ls, emit_off, keys_a, keys_b, tmax, gid, first;
    DBuf<int32_t> ent, start, end;
    DBuf<uint64_t> band_line, band_at;                           // VCF: QUAL values next to the overflow bound
    DBuf<uint8_t> inames, itype; DBuf<uint32_t> ioff; DBuf<int32_t> inum;   // VCF: the declared INFO IDs
};

int sites_stage_init(elp_ctx* c) {
    if (!c->sites) c->sites.reset(new SitesStage());
    SitesStage& S = *c->sites;
    const uint64_t want = c->sites_chunk ? c->sites_chunk : SITES_CHUNK_DEFAULT, cap = want + SITES_MAX_LINE;
    TRY(stage_init(c, S.f, want, cap, stage_padded(cap), "elp_load_known_sites"));
    CUDA_TRY(c, S.d_small.fit(4)); CUDA_TRY(c, S.h_small.fit(16));
    return name_dict_upload(c);
}

int upload(elp_ctx* c, SitesStage& S, const LineChunk& ch) { return stage_upload(c, S.f, ch.b, ch.m, 0); }

// '\n' count of the chunk into h_small[2] (read after the next synchronisation)
int count_lines(elp_ctx* c, SitesStage& S, SitesScratch& X, const LineChunk& ch) {
    const uint64_t n_chunks = (ch.m + SAM_CHUNK - 1) / SAM_CHUNK;
    TRY(grow(c, X.cnt, n_chunks + 8, 0)); TRY(grow(c, X.cnt_off, n_chunks + 2, 0));
    CUDA_TRY(c, cudaStreamWaitEvent(c->stream, S.f.up[ch.b], 0));
    c->begin("sites_lines", (double)ch.m);
    sam_count_kernel<<<nblk(n_chunks, 256), 256, 0, c->stream>>>(S.f.d[ch.b].p, n_chunks, X.cnt.p);
    c->end(); LAUNCH_CHECK(c);
    TRY(exclusive_scan_u32_to_u64(c, X.cnt.p, X.cnt_off.p, n_chunks));
    CUDA_TRY(c, cudaMemcpyAsync(S.h_small.p + 2, X.cnt_off.p + n_chunks, 8, cudaMemcpyDeviceToHost, c->stream));
    return E_OK;
}

// the chunk's lines: line starts, parse and the scan of the interval counts are enqueued; *n_lines is the chunk's line count
int parse_launch(elp_ctx* c, SitesStage& S, SitesScratch& X, const LineChunk& ch, uint64_t line0, uint64_t* n_lines) {
    cudaStream_t s = c->stream;
    CUDA_TRY(c, cudaStreamSynchronize(s));
    const uint64_t n_nl = S.h_small.p[2], n_chunks = (ch.m + SAM_CHUNK - 1) / SAM_CHUNK;
    const bool open_end = S.f.h[ch.b].p[ch.m - 1] != '\n';
    const uint64_t nl = n_nl + (open_end ? 1 : 0);
    TRY(grow(c, X.ls, nl + 2, 0)); TRY(grow(c, X.ent, nl + 8, 0)); TRY(grow(c, X.start, nl + 8, 0)); TRY(grow(c, X.end, nl + 8, 0));
    TRY(grow(c, X.emit, nl + 8, 0)); TRY(grow(c, X.emit_off, nl + 2, 0));
    CUDA_TRY(c, cudaMemsetAsync(X.ls.p, 0, 8, s));
    c->begin("sites_lines", (double)ch.m + 8.0 * (double)n_nl);
    sam_lines_kernel<<<nblk(n_chunks, 256), 256, 0, s>>>(S.f.d[ch.b].p, n_chunks, X.cnt_off.p, X.ls.p);
    c->end(); LAUNCH_CHECK(c);
    if (open_end) { S.h_small.p[4] = ch.m + 1; CUDA_TRY(c, cudaMemcpyAsync(X.ls.p + nl, S.h_small.p + 4, 8, cudaMemcpyHostToDevice, s)); }   // a virtual '\n' past the text
    SitesArgs A{};
    A.text = S.f.d[ch.b].p; A.ls = X.ls.p; A.n_lines = nl; A.line0 = line0; A.dict = c->names.view();
    A.ent = X.ent.p; A.start = X.start.p; A.end = X.end.p; A.emit = X.emit.p; A.small = S.d_small.p;
    c->begin("sites_parse", (double)ch.m + 8.0 * (double)(nl + 1) + 16.0 * (double)nl);
    sites_parse_kernel<<<nblk(nl, 256), 256, 0, s>>>(A);
    c->end(); LAUNCH_CHECK(c);
    TRY(exclusive_scan_u32_to_u64(c, X.emit.p, X.emit_off.p, nl));
    CUDA_TRY(c, cudaMemcpyAsync(S.h_small.p, S.d_small.p, 16, cudaMemcpyDeviceToHost, s));
    CUDA_TRY(c, cudaMemcpyAsync(S.h_small.p + 3, X.emit_off.p + nl, 8, cudaMemcpyDeviceToHost, s));
    *n_lines = nl;
    return E_OK;
}

// the parse's verdict, then the chunk's intervals appended at keys_a / vals_a + *total
int parse_finish(elp_ctx* c, SitesStage& S, SitesScratch& X, const LineChunk& ch, int file, const char* path, uint64_t nl, uint64_t* total) {
    cudaStream_t s = c->stream;
    CUDA_TRY(c, cudaStreamSynchronize(s));
    if (S.h_small.p[0] != ~0ull)
        return c->fail(E_SITES, "elp_load_known_sites: %s (file %d), line %llu (0-based, header = line 0): %s", path, file, (unsigned long long)(S.h_small.p[0] >> 8),
                       sites_err_text((uint32_t)(S.h_small.p[0] & 0xff)));
    const uint64_t add = S.h_small.p[3], t0 = *total;
    if (t0 + add >= (1ull << 30)) return c->fail(E_LIMIT, "elp_load_known_sites: 2^30 or more intervals in total (the limit of the device sort)");
    if (t0 + add + 4 > X.keys_a.cap) { const size_t want = std::max<size_t>(t0 + add + 4, 2 * X.keys_a.cap); TRY(grow(c, X.keys_a, want, t0)); TRY(grow(c, X.vals_a, want, t0)); }
    c->begin("sites_parse", 24.0 * (double)nl + 12.0 * (double)add);
    sites_emit_kernel<<<nblk(nl, 256), 256, 0, s>>>(nl, X.ent.p, X.start.p, X.end.p, X.emit.p, X.emit_off.p, c->names.view(), X.keys_a.p + t0, X.vals_a.p + t0);
    c->end(); LAUNCH_CHECK(c);
    CUDA_TRY(c, cudaEventRecord(S.f.used[ch.b], s));
    *total = t0 + add;
    return E_OK;
}

// ---- VCF files ----
int vcf_fail(elp_ctx* c, const char* path, int file, uint64_t line, const char* why) {
    return c->fail(E_VCF, "elp_load_known_sites: %s (file %d), line %llu (1-based, header lines counted): %s", path, file, (unsigned long long)line, why);
}
int read_fail(elp_ctx* c, const char* path) { return c->fail(E_INVAL, "elp_load_known_sites: cannot read %s: %s", path, strerror(errno)); }

struct VcfState {     // carried from chunk to chunk
    uint64_t line0 = 1;                                      // the 1-based number of the next chunk's first line
    const uint8_t* carry = nullptr; uint64_t carry_n = 0;    // the partial line at the end of the last chunk (device)
};

// the QUAL values in the band next to the overflow bound, decided with strtod: the smallest chunk line whose value overflows, or ~0
int vcf_band(elp_ctx* c, SitesScratch& X, const uint8_t* t, uint64_t n_band, uint64_t* bad) {
    std::vector<uint64_t> ln(n_band), at(n_band);
    CUDA_TRY(c, cudaMemcpy(ln.data(), X.band_line.p, n_band * 8, cudaMemcpyDeviceToHost));
    CUDA_TRY(c, cudaMemcpy(at.data(), X.band_at.p, n_band * 8, cudaMemcpyDeviceToHost));
    std::vector<uint64_t> order(n_band);
    for (uint64_t i = 0; i < n_band; i++) order[i] = i;
    std::sort(order.begin(), order.end(), [&](uint64_t a, uint64_t b) { return ln[a] < ln[b]; });
    std::vector<uint8_t> q;
    *bad = ~0ull;
    for (uint64_t i : order) {
        q.resize(at[i] & 0xffff);
        CUDA_TRY(c, cudaMemcpy(q.data(), t + (at[i] >> 16), q.size(), cudaMemcpyDeviceToHost));
        if (go_float_overflows(q.data(), q.size())) { *bad = ln[i]; return E_OK; }
    }
    return E_OK;
}

// one chunk of VCF text: nnew bytes at buf + VCF_FRONT (zero bytes behind them), of which the first `skip` still belong to the header,
// behind the carried partial line; its intervals are appended at keys_a / vals_a + *total.  `overlap` runs on the host while the line
// count runs.
template <class F>
int vcf_chunk(elp_ctx* c, SitesStage& S, SitesScratch& X, VcfState& St, const VcfInfoTab& info, uint8_t* buf, uint64_t skip, uint64_t nnew, bool last,
              int file, const char* path, cudaEvent_t release_prev, uint64_t* total, F&& overlap) {
    cudaStream_t s = c->stream;
    unsigned long long* hw = S.h_small.p;
    const uint64_t nc = St.carry_n, a = (VCF_FRONT - nc) & ~(uint64_t)(SAM_CHUNK - 1), front = VCF_FRONT - nc + skip - a, end = VCF_FRONT + nnew - a;
    uint8_t* t = buf + a;
    if (nc) CUDA_TRY(c, cudaMemcpyAsync(buf + VCF_FRONT - nc, St.carry, nc, cudaMemcpyDeviceToDevice, s));
    if (VCF_FRONT - nc - a) CUDA_TRY(c, cudaMemsetAsync(t, 0, VCF_FRONT - nc - a, s));   // (no '\n' in front of the first line)
    if (skip) CUDA_TRY(c, cudaMemsetAsync(buf + VCF_FRONT, 0, skip, s));                  // (nor in the header's bytes)
    if (release_prev) CUDA_TRY(c, cudaEventRecord(release_prev, s));
    St.carry = nullptr; St.carry_n = 0;
    if (end == front) return overlap();
    const uint64_t n_chunks = (end + SAM_CHUNK - 1) / SAM_CHUNK;
    TRY(grow(c, X.cnt, n_chunks + 8, 0)); TRY(grow(c, X.cnt_off, n_chunks + 2, 0));
    c->begin("sites_lines", (double)(end - front));
    sam_count_kernel<<<nblk(n_chunks, 256), 256, 0, s>>>(t, n_chunks, X.cnt.p);
    c->end(); LAUNCH_CHECK(c);
    TRY(exclusive_scan_u32_to_u64(c, X.cnt.p, X.cnt_off.p, n_chunks));
    CUDA_TRY(c, cudaMemcpyAsync(hw + 2, X.cnt_off.p + n_chunks, 8, cudaMemcpyDeviceToHost, s));
    TRY(overlap());
    CUDA_TRY(c, cudaStreamSynchronize(s));
    const uint64_t n_nl = hw[2];
    TRY(grow(c, X.ls, n_nl + 2, 0));
    hw[7] = front;
    CUDA_TRY(c, cudaMemcpyAsync(X.ls.p, hw + 7, 8, cudaMemcpyHostToDevice, s));
    c->begin("sites_lines", (double)(end - front) + 8.0 * (double)n_nl);
    sam_lines_kernel<<<nblk(n_chunks, 256), 256, 0, s>>>(t, n_chunks, X.cnt_off.p, X.ls.p);
    c->end(); LAUNCH_CHECK(c);
    CUDA_TRY(c, cudaMemcpyAsync(hw + 6, X.ls.p + n_nl, 8, cudaMemcpyDeviceToHost, s));
    CUDA_TRY(c, cudaStreamSynchronize(s));
    const uint64_t m = hw[6];   // the end of the whole lines
    uint64_t nl = n_nl;
    if (last && m < end) { hw[4] = end + 1; nl++; CUDA_TRY(c, cudaMemcpyAsync(X.ls.p + nl, hw + 4, 8, cudaMemcpyHostToDevice, s)); }   // a virtual '\n'
    if (!last) { St.carry = t + m; St.carry_n = end - m; }
    if (nl) {
        TRY(grow(c, X.ent, nl + 8, 0)); TRY(grow(c, X.start, nl + 8, 0)); TRY(grow(c, X.end, nl + 8, 0)); TRY(grow(c, X.emit, nl + 8, 0));
        TRY(grow(c, X.emit_off, nl + 2, 0)); TRY(grow(c, X.band_line, nl + 1, 0)); TRY(grow(c, X.band_at, nl + 1, 0));
        CUDA_TRY(c, cudaMemsetAsync(S.d_small.p + 2, 0, 8, s));
        VcfArgs A{};
        A.t = t; A.ls = X.ls.p; A.n_lines = nl; A.line0 = St.line0; A.dict = c->names.view(); A.info = info;
        A.ent = X.ent.p; A.start = X.start.p; A.end = X.end.p; A.emit = X.emit.p; A.small = S.d_small.p;
        A.band_line = X.band_line.p; A.band_at = X.band_at.p; A.n_band = S.d_small.p + 2;
        const uint64_t groups = (nl + 31) / 32;
        const unsigned grid = (unsigned)std::min<uint64_t>((groups + VP_T / 32 - 1) / (VP_T / 32), 132 * 16);
        c->begin("vcf_parse", (double)(std::max(m, end) - front) + 8.0 * (double)(nl + 1) + 16.0 * (double)nl);
        vcf_parse_kernel<<<grid, VP_T, 0, s>>>(A);
        c->end(); LAUNCH_CHECK(c);
        TRY(exclusive_scan_u32_to_u64(c, X.emit.p, X.emit_off.p, nl));
        CUDA_TRY(c, cudaMemcpyAsync(hw + 8, S.d_small.p, 24, cudaMemcpyDeviceToHost, s));
        CUDA_TRY(c, cudaMemcpyAsync(hw + 3, X.emit_off.p + nl, 8, cudaMemcpyDeviceToHost, s));
        CUDA_TRY(c, cudaStreamSynchronize(s));
        unsigned long long err = hw[8];
        if (hw[10]) {
            uint64_t bad = ~0ull;
            TRY(vcf_band(c, X, t, hw[10], &bad));
            if (bad != ~0ull && St.line0 + bad <= (err >> 8)) err = ((St.line0 + bad) << 8) | VL_QUAL_RANGE;   // QUAL precedes FILTER and INFO
        }
        if (err != ~0ull) return vcf_fail(c, path, file, err >> 8, vcf_err_text((uint32_t)(err & 0xff)));
        const uint64_t add = hw[3], t0 = *total;
        if (t0 + add >= (1ull << 30)) return c->fail(E_LIMIT, "elp_load_known_sites: 2^30 or more intervals in total (the limit of the device sort)");
        if (t0 + add + 4 > X.keys_a.cap) { const size_t want = std::max<size_t>(t0 + add + 4, 2 * X.keys_a.cap); TRY(grow(c, X.keys_a, want, t0)); TRY(grow(c, X.vals_a, want, t0)); }
        c->begin("sites_parse", 24.0 * (double)nl + 12.0 * (double)add);
        sites_emit_kernel<<<nblk(nl, 256), 256, 0, s>>>(nl, X.ent.p, X.start.p, X.end.p, X.emit.p, X.emit_off.p, c->names.view(), X.keys_a.p + t0, X.vals_a.p + t0);
        c->end(); LAUNCH_CHECK(c);
        *total = t0 + add;
        St.line0 += nl;
    }
    if (St.carry_n >= VCF_MAX_LINE) return vcf_fail(c, path, file, St.line0, vcf_err_text(VL_LONG));
    return E_OK;
}

// the leading BGZF blocks of a file, inflated on the host one at a time for the header (HReader's byte source)
struct BgzfHead {
    elp_ctx* c; FILE* f; const char* path;
    std::vector<uint8_t> cz; uint64_t cz_at = 0, out = 0;   // compressed bytes not yet inflated, their file offset; bytes inflated
    std::vector<BgzfBlock> blocks;                          // in_off: file offset, out_off, isize
    int operator()(std::vector<uint8_t>& buf) {
        for (;;) {
            std::vector<BgzfBlock> bl; uint64_t tot = 0, used = 0;
            if (scan_blocks(cz.data(), cz.size(), bl, &tot, &used, 1))
                return c->fail(E_BGZF, "elp_load_known_sites: %s, file offset %llu: malformed BGZF block header (gzip magic, FEXTRA, BC subfield, block size or ISIZE)", path, (unsigned long long)cz_at);
            if (!bl.empty()) {
                BgzfBlock b = bl[0];
                const size_t o = buf.size();
                buf.resize(o + b.isize);
                bool ok = true;
                if (b.isize) {
                    z_stream zs; memset(&zs, 0, sizeof zs);
                    ok = inflateInit2(&zs, -15) == Z_OK;
                    if (ok) {
                        zs.next_in = cz.data() + b.cdata_off; zs.avail_in = (uInt)b.cdata_len; zs.next_out = buf.data() + o; zs.avail_out = b.isize;
                        ok = inflate(&zs, Z_FINISH) == Z_STREAM_END && zs.total_out == b.isize;
                        inflateEnd(&zs);
                    }
                }
                if (!ok || (uint32_t)crc32(crc32(0L, Z_NULL, 0), buf.data() + o, b.isize) != b.crc)
                    return c->fail(E_BGZF, "elp_load_known_sites: %s, BGZF block at file offset %llu: bad DEFLATE data or CRC32", path, (unsigned long long)cz_at);
                b.in_off = cz_at; b.out_off = out;
                blocks.push_back(b);
                out += b.isize;
                cz.erase(cz.begin(), cz.begin() + used); cz_at += used;
                if (b.isize) return 1;
                continue;
            }
            uint8_t tmp[1 << 16];
            const size_t got = fread(tmp, 1, sizeof tmp, f);
            if (!got) {
                if (ferror(f)) return read_fail(c, path);
                if (!cz.empty()) return c->fail(E_BGZF, "elp_load_known_sites: %s, file offset %llu: the file ends inside a BGZF block", path, (unsigned long long)cz_at);
                return 0;
            }
            cz.insert(cz.end(), tmp, tmp + got);
        }
    }
};

struct PlainHead {
    elp_ctx* c; FILE* f; const char* path;
    int operator()(std::vector<uint8_t>& buf) {
        const size_t o = buf.size();
        buf.resize(o + (1 << 16));
        const size_t got = fread(buf.data() + o, 1, 1 << 16, f);
        buf.resize(o + got);
        if (!got && ferror(f)) return read_fail(c, path);
        return got ? 1 : 0;
    }
};

// the declared INFO IDs to the device (the first of equal IDs, as SmallMap.Get finds it)
int vcf_info_upload(elp_ctx* c, SitesScratch& X, const VcfHeader& h, VcfInfoTab* T) {
    std::vector<uint8_t> names, type; std::vector<uint32_t> off(1, 0); std::vector<int32_t> num;
    std::vector<std::string> seen;
    for (const VcfInfo& fi : h.infos) {
        if (std::find(seen.begin(), seen.end(), fi.id) != seen.end()) continue;
        seen.push_back(fi.id);
        names.insert(names.end(), fi.id.begin(), fi.id.end()); off.push_back((uint32_t)names.size()); type.push_back(fi.type); num.push_back(fi.number);
    }
    TRY(grow(c, X.inames, names.size() + 1, 0)); TRY(grow(c, X.ioff, off.size(), 0)); TRY(grow(c, X.itype, type.size() + 1, 0)); TRY(grow(c, X.inum, num.size() + 1, 0));
    if (!names.empty()) CUDA_TRY(c, cudaMemcpy(X.inames.p, names.data(), names.size(), cudaMemcpyHostToDevice));
    CUDA_TRY(c, cudaMemcpy(X.ioff.p, off.data(), off.size() * 4, cudaMemcpyHostToDevice));
    if (!type.empty()) CUDA_TRY(c, cudaMemcpy(X.itype.p, type.data(), type.size(), cudaMemcpyHostToDevice));
    if (!num.empty()) CUDA_TRY(c, cudaMemcpy(X.inum.p, num.data(), num.size() * 4, cudaMemcpyHostToDevice));
    *T = VcfInfoTab{X.inames.p, X.ioff.p, X.itype.p, X.inum.p, (int)type.size()};
    return E_OK;
}

// plain VCF text after the header: chunk k+1 is read and uploaded while the line count of chunk k runs
int vcf_plain(elp_ctx* c, SitesStage& S, SitesScratch& X, VcfState& St, const VcfInfoTab& info, FILE* f, int file, const char* path, uint64_t* total) {
    FileStage& V = S.v;
    const uint64_t chunk = V.chunk;
    auto fill = [&](int b, uint64_t* got, bool* last) -> int {
        TRY(stage_wait_host(c, V, b));
        *got = fread(V.h[b].p, 1, chunk, f);
        if (*got < chunk && ferror(f)) return read_fail(c, path);
        *last = *got < chunk;
        return stage_upload(c, V, b, *got, VCF_FRONT);
    };
    int b = 0; uint64_t got = 0; bool last = false;
    TRY(fill(b, &got, &last));
    for (;;) {
        uint64_t got2 = 0; bool last2 = true;
        CUDA_TRY(c, cudaStreamWaitEvent(c->stream, V.up[b], 0));
        if (!got) CUDA_TRY(c, cudaMemsetAsync(V.d[b].p + VCF_FRONT, 0, SAM_CHUNK, c->stream));
        TRY(vcf_chunk(c, S, X, St, info, V.d[b].p, 0, got, last, file, path, V.used[b ^ 1], total, [&]() { return last ? E_OK : fill(b ^ 1, &got2, &last2); }));
        if (last) break;
        b ^= 1; got = got2; last = last2;   // (vcf_chunk of the next chunk records used[b ^ 1] behind its copy of the carried line)
    }
    return E_OK;
}

// BGZF VCF from file offset `at` (a block start), the first `skip` inflated bytes being header: the whole blocks of each chunk inflated
// on the device, an incomplete last block carried to the next chunk on the host (as reference_load.cu reads BGZF FASTA)
int vcf_bgzf(elp_ctx* c, SitesStage& S, SitesScratch& X, VcfState& St, const VcfInfoTab& info, FILE* f, int file, const char* path, uint64_t at, uint64_t skip, uint64_t* total) {
    FileStage& V = S.v;
    const uint64_t chunk = V.chunk;
    std::vector<uint8_t> cz;
    std::vector<BgzfBlock> blocks;
    bool eof_block = false;
    int b = 0;
    for (;;) {
        uint8_t* h = V.h[0].p;
        const uint64_t nc = cz.size();
        if (nc) memcpy(h, cz.data(), nc);
        const size_t got = fread(h + nc, 1, chunk, f);
        if (got < chunk && ferror(f)) return read_fail(c, path);
        const bool last = got < chunk;
        const uint64_t n = nc + got;
        uint64_t tot = 0, used = 0;
        blocks.clear();
        if (scan_blocks(h, n, blocks, &tot, &used)) {
            const uint64_t bad = blocks.empty() ? 0 : blocks.back().cdata_off + blocks.back().cdata_len + BGZF_TRL;
            return c->fail(E_BGZF, "elp_load_known_sites: %s, file offset %llu: malformed BGZF block header (gzip magic, FEXTRA, BC subfield, block size or ISIZE)", path,
                           (unsigned long long)(at + bad));
        }
        if (last && used < n)
            return c->fail(E_BGZF, "elp_load_known_sites: %s, file offset %llu: the file ends inside a BGZF block (%llu bytes left)", path, (unsigned long long)(at + used),
                           (unsigned long long)(n - used));
        if (!blocks.empty()) {
            const BgzfBlock& lb = blocks.back();
            eof_block = lb.cdata_len == 2 && h[lb.cdata_off] == 3 && h[lb.cdata_off + 1] == 0 && lb.crc == 0 && lb.isize == 0;   // bgzf-files.go:111-115
        }
        if (last && !eof_block) return c->fail(E_BGZF, "elp_load_known_sites: %s, file offset %llu: invalid BGZF file: does not end in proper EOF marker", path, (unsigned long long)(at + used));
        if (!blocks.empty() || last) {
            TRY(grow(c, S.tb[b], VCF_FRONT + stage_padded(tot), 0));
            if (!blocks.empty()) {
                char who[1200];
                snprintf(who, sizeof who, "elp_load_known_sites: %s, BGZF blocks from file offset %llu", path, (unsigned long long)at);
                TRY(bgzf_inflate_run(c, who, h, used, blocks, tot, S.tb[b].p + VCF_FRONT));
            }
            CUDA_TRY(c, cudaMemsetAsync(S.tb[b].p + VCF_FRONT + tot, 0, stage_padded(tot) - tot, c->stream));
            TRY(vcf_chunk(c, S, X, St, info, S.tb[b].p, std::min(skip, tot), tot, last, file, path, nullptr, total, []() { return E_OK; }));
            skip = 0;
            b ^= 1;
        }
        cz.assign(h + used, h + n);
        at += used;
        if (last) return E_OK;
    }
}

// one VCF file: the header on the host, then every data line through the device, appended behind *total
int load_vcf(elp_ctx* c, SitesStage& S, SitesScratch& X, int file, const char* path, FILE* f, bool bgzf, uint64_t* total) {
    const uint64_t want = c->sites_chunk ? c->sites_chunk : SITES_CHUNK_DEFAULT;
    TRY(stage_init(c, S.v, want, want + BGZF_MAX_BLOCK, VCF_FRONT + stage_padded(want), "elp_load_known_sites"));
    VcfHeader h;
    uint64_t bad_line = 0; const char* why = nullptr;
    uint64_t at = 0, skip = 0;
    if (bgzf) {
        BgzfHead src{c, f, path};
        const int rc = vcf_header(src, &h, &bad_line, &why);
        if (rc == E_VCF) return vcf_fail(c, path, file, bad_line, why);
        TRY(rc);
        at = src.cz_at;   // the data start in the block that holds byte h.bytes, or in the first block after it (an empty one included)
        for (const BgzfBlock& b : src.blocks)
            if (b.out_off + b.isize > h.bytes || (b.isize == 0 && b.out_off >= h.bytes)) { at = b.in_off; skip = h.bytes - b.out_off; break; }
    } else {
        PlainHead src{c, f, path};
        const int rc = vcf_header(src, &h, &bad_line, &why);
        if (rc == E_VCF) return vcf_fail(c, path, file, bad_line, why);
        TRY(rc);
        at = h.bytes;
    }
    if (fseeko(f, (off_t)at, SEEK_SET) != 0) return read_fail(c, path);
    VcfInfoTab info{};
    TRY(vcf_info_upload(c, X, h, &info));
    VcfState St;
    St.line0 = h.lines + 1;
    return bgzf ? vcf_bgzf(c, S, X, St, info, f, file, path, at, skip, total) : vcf_plain(c, S, X, St, info, f, file, path, total);
}

// one file: the header on the host, then every line through the device, appended behind *total.  The format comes from the content:
// the .elsites header, a first byte 0x1f (BGZF VCF, as vcf.Open sniffs it, vcf-files.go:1285-1312), or "##fileformat=VCFv4." (plain VCF)
int load_file(elp_ctx* c, SitesStage& S, SitesScratch& X, int file, const char* path, uint64_t* total) {
    FILE* f = fopen(path, "rb");
    if (!f) return c->fail(E_INVAL, "elp_load_known_sites: cannot open %s: %s", path, strerror(errno));
    struct Closer { FILE* f; ~Closer() { fclose(f); } } closer{f};
    char hd[SITES_HEADER_LEN];   // bufio.Reader.ReadString('\n') must return exactly ElsitesHeader (intervals.go:204-210)
    const size_t got = fread(hd, 1, SITES_HEADER_LEN, f);
    if (got < SITES_HEADER_LEN && ferror(f)) return c->fail(E_INVAL, "elp_load_known_sites: cannot read %s: %s", path, strerror(errno));
    const bool elsites = got == SITES_HEADER_LEN && memcmp(hd, SITES_HEADER, SITES_HEADER_LEN) == 0;
    if (!elsites && got >= 1 && (uint8_t)hd[0] == 0x1f) return fseeko(f, 0, SEEK_SET) ? read_fail(c, path) : load_vcf(c, S, X, file, path, f, true, total);
    if (!elsites && got >= VCF_PREFIX_LEN && memcmp(hd, VCF_PREFIX, VCF_PREFIX_LEN) == 0)
        return fseeko(f, 0, SEEK_SET) ? read_fail(c, path) : load_vcf(c, S, X, file, path, f, false, total);
    if (!elsites)
        return c->fail(E_SITES, "elp_load_known_sites: %s (file %d), line 0 (0-based, header = line 0): not a .elsites file - the first line is not \"# elsites format version 1.0\"", path, file);
    std::vector<uint8_t> carry;
    uint64_t line0 = 1;
    LineChunk cur;
    TRY(stage_read_lines(c, S.f, f, path, "elp_load_known_sites", SITES_MAX_LINE, carry, 0, &cur));
    TRY(upload(c, S, cur));
    for (;;) {
        uint64_t nl = 0;
        if (cur.m) { TRY(count_lines(c, S, X, cur)); TRY(parse_launch(c, S, X, cur, line0, &nl)); }
        const bool more = !cur.last && !cur.long_tail;
        LineChunk nxt;
        if (more) { TRY(stage_read_lines(c, S.f, f, path, "elp_load_known_sites", SITES_MAX_LINE, carry, cur.b ^ 1, &nxt)); TRY(upload(c, S, nxt)); }   // overlaps the kernels of cur
        if (cur.m) TRY(parse_finish(c, S, X, cur, file, path, nl, total));
        line0 += nl;
        if (cur.long_tail) return c->fail(E_SITES, "elp_load_known_sites: %s (file %d), line %llu (0-based, header = line 0): %s", path, file, (unsigned long long)line0, sites_err_text(KS_LONG));
        if (!more) return E_OK;
        cur = nxt;
    }
}

// sorted intervals -> flattened groups in one allocation (*block, *n_groups pairs); first[contig] = its first group or ~0
int flatten(elp_ctx* c, SitesScratch& X, const uint64_t* keys, const uint32_t* ends, uint64_t n, DBuf<int32_t>* block, uint64_t* n_groups, std::vector<uint64_t>& first) {
    cudaStream_t s = c->stream;
    const int nc = c->n_contigs;
    const uint64_t tiles = (n + FL_TILE - 1) / FL_TILE;
    TRY(grow(c, X.tmax, tiles + 1, 0)); TRY(grow(c, X.head, n + 4, 0)); TRY(grow(c, X.gid, n + 2, 0)); TRY(grow(c, X.first, nc + 1, 0));
    c->begin("sites_flatten", 12.0 * (double)n + 8.0 * (double)tiles);
    sites_tile_max_kernel<<<(unsigned)tiles, FL_T, 0, s>>>(keys, ends, n, X.tmax.p);
    c->end(); LAUNCH_CHECK(c);
    c->begin("sites_flatten", 16.0 * (double)tiles);
    sites_tile_scan_kernel<<<1, 1024, 0, s>>>(X.tmax.p, tiles);
    c->end(); LAUNCH_CHECK(c);
    c->begin("sites_flatten", 16.0 * (double)n + 8.0 * (double)tiles);
    sites_head_kernel<<<(unsigned)tiles, FL_T, 0, s>>>(keys, ends, n, X.tmax.p, X.head.p);
    c->end(); LAUNCH_CHECK(c);
    TRY(exclusive_scan_u32_to_u64(c, X.head.p, X.gid.p, n));
    uint64_t G = 0;
    CUDA_TRY(c, cudaMemcpyAsync(&G, X.gid.p + n, 8, cudaMemcpyDeviceToHost, s));
    CUDA_TRY(c, cudaStreamSynchronize(s));
    DBuf<int32_t> out;
    cudaError_t e = out.fit(2 * G);
    if (e != cudaSuccess) { cudaGetLastError(); return c->fail(e == cudaErrorMemoryAllocation ? E_NOMEM : E_CUDA, "device allocation of %llu bytes failed", (unsigned long long)(G * 8)); }
    int rc = E_OK;
    auto step = [&](cudaError_t x) { if (rc == E_OK && x != cudaSuccess) rc = c->fail(E_CUDA, "elp_load_known_sites: %s", cudaGetErrorString(x)); };
    step(cudaMemsetAsync(out.p, 0, G * 8, s));
    step(cudaMemsetAsync(X.first.p, 0xff, (size_t)nc * 8, s));
    c->begin("sites_flatten", 24.0 * (double)n + 8.0 * (double)G);
    sites_compact_kernel<<<nblk(n, 256), 256, 0, s>>>(keys, ends, n, X.head.p, X.gid.p, out.p, X.first.p);
    c->end(); step(cudaGetLastError());
    c->begin("sites_flatten", 8.0 * (double)G);
    sites_unbias_kernel<<<nblk(G, 256), 256, 0, s>>>(G, out.p);
    c->end(); step(cudaGetLastError());
    first.assign(nc, ~0ull);
    if (nc) step(cudaMemcpyAsync(first.data(), X.first.p, (size_t)nc * 8, cudaMemcpyDeviceToHost, s));
    step(cudaStreamSynchronize(s));
    if (rc) return rc;
    *block = std::move(out); *n_groups = G;
    return E_OK;
}

}  // namespace

extern "C" int elp_load_known_sites(elp_ctx* c, const char* const* paths, int32_t n_paths, uint64_t* n_unmatched) {
    if (!c) return ELP_EINVAL;
    cudaSetDevice(c->device);
    if (n_paths < 0 || (n_paths && !paths)) return c->fail(E_INVAL, "elp_load_known_sites: %d paths at %p", n_paths, (const void*)paths);
    for (int i = 0; i < n_paths; i++) if (!paths[i]) return c->fail(E_INVAL, "elp_load_known_sites: path %d is null", i);
    if (c->n_contigs > 0 && !c->has_contig_names)
        return c->fail(E_INVAL, "elp_load_known_sites: the context was created without elp_config.contig_names, so chromosome names cannot be resolved");
    const int nc = c->n_contigs;
    DBuf<int32_t> block; uint64_t G = 0, unmatched = 0;
    std::vector<uint64_t> first(nc, ~0ull);
    if (n_paths) {
        TRY(sites_stage_init(c));
        SitesStage& S = *c->sites;
        struct Drain { SitesStage& S; ~Drain() { cudaStreamSynchronize(S.f.copy); if (S.v.copy) cudaStreamSynchronize(S.v.copy); } } drain{S};   // no upload outlives the call
        SitesScratch X;
        CUDA_TRY(c, cudaMemsetAsync(S.d_small.p, 0xff, 8, c->stream));
        CUDA_TRY(c, cudaMemsetAsync(S.d_small.p + 1, 0, 8, c->stream));
        uint64_t total = 0;
        for (int i = 0; i < n_paths; i++) TRY(load_file(c, S, X, i, paths[i], &total));
        CUDA_TRY(c, cudaMemcpyAsync(S.h_small.p + 1, S.d_small.p + 1, 8, cudaMemcpyDeviceToHost, c->stream));
        CUDA_TRY(c, cudaStreamSynchronize(c->stream));
        unmatched = S.h_small.p[1];
        if (total) {
            TRY(grow(c, X.keys_b, total + 4, 0)); TRY(grow(c, X.vals_b, total + 4, 0));
            int bits = 32;
            for (uint32_t v = (uint32_t)nc; v; v >>= 1) bits++;
            // sites_sort spans the radix passes (which also report under radix_*_sites); it is recorded once the sort is enqueued
            cudaEvent_t ea = nullptr;
            if (c->profile) { ea = c->get_event(); cudaEventRecord(ea, c->stream); }
            bool in_b = false;
            TRY(radix_sort_u64(c, X.keys_a.p, X.keys_b.p, X.vals_a.p, X.vals_b.p, total, bits, &in_b, "sites"));
            if (c->profile) {
                PendingEvent pe; pe.name = "sites_sort"; pe.a = ea; pe.b = c->get_event();
                pe.alg_bytes = (double)rs::make_plan(bits).n_passes * 2.0 * 12.0 * (double)total;
                cudaEventRecord(pe.b, c->stream);
                c->pending.push_back(pe);
            }
            TRY(flatten(c, X, in_b ? X.keys_b.p : X.keys_a.p, in_b ? X.vals_b.p : X.vals_a.p, total, &block, &G, first));
        }
    }
    // install: every contig's list is replaced (contigs appear in increasing order, so a contig's groups end at the next one's first)
    std::vector<int32_t*> d(nc, nullptr); std::vector<uint64_t> cnt(nc, 0);
    uint64_t next = G;
    for (int i = nc - 1; i >= 0; i--)
        if (first[i] != ~0ull) { d[i] = block.p + 2 * first[i]; cnt[i] = next - first[i]; next = first[i]; }
    c->known_sites.install(std::move(block), std::move(d), std::move(cnt));
    if (n_unmatched) *n_unmatched = unmatched;
    return ELP_OK;
}

extern "C" int64_t elp_known_sites_get(elp_ctx* c, int32_t contig, int32_t* se, uint64_t cap) {
    if (!c) return -1;
    cudaSetDevice(c->device);
    if (contig < 0 || contig >= c->n_contigs) { c->fail(E_INVAL, "elp_known_sites_get: contig %d out of range", contig); return -1; }
    const RegionTable& t = c->known_sites;
    const uint64_t n = t.n[contig];
    const uint64_t k = std::min(n, cap);
    if (se && k) {
        if (cudaMemcpyAsync(se, t.d[contig], k * 8, cudaMemcpyDeviceToHost, c->stream) != cudaSuccess || cudaStreamSynchronize(c->stream) != cudaSuccess) {
            c->fail(E_CUDA, "elp_known_sites_get: %s", cudaGetErrorString(cudaGetLastError()));
            return -1;
        }
    }
    return (int64_t)n;
}

extern "C" int elp_debug_set_sites_chunk(elp_ctx* c, uint64_t bytes) {
    if (!c) return ELP_EINVAL;
    if (bytes > (1ull << 32)) return c->fail(E_INVAL, "elp_debug_set_sites_chunk: %llu bytes (at most 2^32)", (unsigned long long)bytes);
    c->sites_chunk = bytes;   // the staging is reallocated by the next load
    return ELP_OK;
}
