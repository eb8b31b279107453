// bgzf_inflate.cu -- a BGZF-compressed BAM file straight into a context (elp_append_bgzf; SURVEY.md §8f row 2, utils/bgzf/bgzf-files.go:95-127,164-221).
//
// Per call: the host finds the whole BGZF blocks (bgzf_scan.hpp; an incomplete trailing block is carried to the next call), uploads the
// compressed bytes and a table of (cdata_off, cdata_len, out_off, isize, crc) once, and the device does the rest:
//   bgzf_inflate   one warp per block: the DEFLATE decoder of inflate.cuh (tables in shared memory, warp-uniform symbol decode, warp-wide
//                  copies) straight into bam_raw, behind the bytes carried from the last call
//   bgzf_crc       one warp per block: per-lane CRC-32 of a 1/32 slice, folded with the x^(2^k) shift table
//   bam_header     one thread, until the BAM header is complete: its length and the reference list, which the host checks against elp_config
//   bam_frame      the record boundaries (below), then bam_ingest_core as for elp_append_bam
// The bytes of a record that the call does not complete stay at the front of bam_raw for the next call.
//
// Framing.  The block_size chain is inherently serial, so the bytes are cut into SEG-byte segments and each segment guesses its first
// record start with a plausibility test (a speed heuristic only: it never decides the result) and walks the chain from the guess to the
// first start at or past its end (its exit).  Segment 0 starts at the true start.  Segments whose guess differs from their predecessor's
// exit are walked again from that exit (bam_frame_fix_kernel); rounds repeat until every segment agrees with its predecessor.  Then every
// segment is right by induction (a segment whose guess equals the exit of a right predecessor is right), so the result is the serial walk.
// Each round makes at least one more segment right; in practice one round repairs every wrong guess.  A record longer than a segment
// passes through: the segment's exit is its entry.
#include <algorithm>
#include <cstring>
#include "ctx.h"
#include "bgzf_scan.hpp"
#include "inflate.cuh"
#include "../../include/elprep_b200.h"

namespace {

__device__ __forceinline__ uint32_t drd32(const uint8_t* p) { return (uint32_t)p[0] | ((uint32_t)p[1] << 8) | ((uint32_t)p[2] << 16) | ((uint32_t)p[3] << 24); }
__device__ __forceinline__ uint32_t drd16(const uint8_t* p) { return (uint32_t)p[0] | ((uint32_t)p[1] << 8); }

struct BlockDesc { uint64_t cdata_off, out_off; uint32_t cdata_len, isize, crc, pad; };

struct WarpTeam {
    static constexpr unsigned size = 32;
    unsigned lane;
    __device__ void sync() const { __syncwarp(); }
};

constexpr int INF_WARPS = 4;
__global__ void __launch_bounds__(INF_WARPS * 32) bgzf_inflate_kernel(const uint8_t* __restrict__ in, const BlockDesc* __restrict__ tab, uint64_t nb, uint8_t* __restrict__ out,
                                                                      uint32_t* __restrict__ status) {
    __shared__ dfl::Tables T[INF_WARPS];
    const unsigned w = threadIdx.x >> 5;
    const uint64_t b = (uint64_t)blockIdx.x * INF_WARPS + w;
    if (b >= nb) return;
    const BlockDesc d = tab[b];
    uint32_t st = dfl::OK;
    if (d.isize) st = dfl::inflate_stream(WarpTeam{threadIdx.x & 31}, T[w], in + d.cdata_off, d.cdata_len, out + d.out_off, d.isize);   // (an empty block is not decoded, as elp_bgzf_inflate)
    if ((threadIdx.x & 31) == 0) status[b] = st;
}

struct X2n { uint32_t v[32]; };
__global__ void __launch_bounds__(256) bgzf_crc_kernel(const BlockDesc* __restrict__ tab, uint64_t nb, const uint8_t* __restrict__ out, uint32_t* __restrict__ status, X2n x2n) {
    __shared__ uint32_t ctab[256];
    ctab[threadIdx.x] = dfl::crc_table_entry(threadIdx.x);
    __syncthreads();
    const unsigned lane = threadIdx.x & 31;
    const uint64_t b = (uint64_t)blockIdx.x * 8 + (threadIdx.x >> 5);
    if (b >= nb || status[b]) return;
    const BlockDesc d = tab[b];
    const uint32_t v = dfl::warp_crc(ctab, x2n.v, out + d.out_off, d.isize, lane);
    if (lane == 0 && v != d.crc) status[b] = dfl::E_CRC;
}

// the BAM header at b[0, n) (sam/bam-files.go ParseHeader): r[0] = 0 complete, 1 more bytes needed, 2 malformed; r[1] = its length;
// r[2] = offset of n_ref
__global__ void bam_header_walk_kernel(const uint8_t* __restrict__ b, uint64_t n, uint64_t* __restrict__ r) {
    if (threadIdx.x || blockIdx.x) return;
    const uint8_t magic[4] = {'B', 'A', 'M', 1};
    r[0] = 1;
    for (uint64_t i = 0; i < 4 && i < n; i++) if (b[i] != magic[i]) { r[0] = 2; return; }
    if (n < 8) return;
    const int32_t l_text = (int32_t)drd32(b + 4);
    if (l_text < 0) { r[0] = 2; return; }
    uint64_t x = 8ull + (uint64_t)l_text;
    if (x + 4 > n) return;
    const int32_t n_ref = (int32_t)drd32(b + x);
    if (n_ref < 0) { r[0] = 2; return; }
    r[2] = x; x += 4;
    for (int32_t k = 0; k < n_ref; k++) {
        if (x + 4 > n) return;
        const int32_t l_name = (int32_t)drd32(b + x);
        if (l_name < 0) { r[0] = 2; return; }
        x += 8ull + (uint64_t)l_name;
        if (x > n) return;
    }
    r[1] = x; r[0] = 0;
}

// ---- framing ----
constexpr uint64_t SEG = 4096;
struct Frame { const uint8_t* b; uint64_t n, nseg; int32_t n_ref; };
__device__ __forceinline__ uint64_t seg_end(const Frame& F, uint64_t s) { return min((s + 1) * SEG, F.n); }
// first chain position at or past the end of segment s, walking from g (stops at a position whose block_size lies past the bytes)
__device__ uint64_t frame_walk(const Frame& F, uint64_t s, uint64_t g) {
    const uint64_t e = seg_end(F, s);
    uint64_t p = g;
    while (p < e && p + 4 <= F.n) p += 4ull + drd32(F.b + p);
    return p;
}
// could a record start at p?  block_size >= 32, l_read_name >= 1 with its NUL, refID and next_refID in [-1, n_ref), l_seq >= 0, the
// variable lengths within block_size.  Only decides how many rounds the framing takes, never where records start.
__device__ bool plausible(const Frame& F, uint64_t p) {
    if (p + 36 > F.n) return false;
    const uint8_t* r = F.b + p;
    const uint32_t bs = drd32(r);
    const int32_t refid = (int32_t)drd32(r + 4), nref = (int32_t)drd32(r + 24), l_seq = (int32_t)drd32(r + 20);
    const uint32_t l_name = r[12], n_cig = drd16(r + 16);
    if (bs < 32 || l_name < 1 || l_seq < 0 || refid < -1 || refid >= F.n_ref || nref < -1 || nref >= F.n_ref) return false;
    if (32ull + l_name + 4ull * n_cig + ((uint64_t)l_seq + 1) / 2 + (uint64_t)l_seq > bs) return false;
    return p + 36 + l_name > F.n || r[36 + l_name - 1] == 0;
}
__global__ void __launch_bounds__(256) bam_frame_guess_kernel(Frame F, uint64_t* __restrict__ g, uint64_t* __restrict__ x) {
    const uint64_t s = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= F.nseg) return;
    const uint64_t e = seg_end(F, s);
    uint64_t guess = s ? e : 0;                                 // no plausible start: the segment's entry lies at or past its end
    if (s) for (uint64_t p = s * SEG; p < e; p++) {
        uint64_t q = p; int k = 0;                              // the record at p and the next two in its chain (or the end of the bytes)
        while (k < 3 && q + 36 <= F.n && plausible(F, q)) { q += 4ull + drd32(F.b + q); k++; }
        if (k == 3 || (k > 0 && q + 36 > F.n)) { guess = p; break; }
    }
    g[s] = guess; x[s] = frame_walk(F, s, guess);
}
// a repair round (g1, x1 start as copies of g0, x0): a chase starts at every segment that disagrees with a predecessor which agrees with its
// own predecessor, walks it from that predecessor's exit and goes on into the next segments until its exit equals the next guess or it
// reaches the start of another chase (so chases write disjoint segments).  The first disagreeing segment always starts one from a right
// entry, so every round extends the right prefix; isolated wrong guesses are all repaired in one round.
__device__ __forceinline__ bool chase_start(const uint64_t* g, const uint64_t* x, uint64_t u) { return g[u] != x[u - 1] && (u == 1 || g[u - 1] == x[u - 2]); }
__global__ void __launch_bounds__(256) bam_frame_fix_kernel(Frame F, const uint64_t* __restrict__ g0, const uint64_t* __restrict__ x0, uint64_t* __restrict__ g1, uint64_t* __restrict__ x1,
                                                            uint32_t* __restrict__ changed) {
    const uint64_t s = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (s == 0 || s >= F.nseg || !chase_start(g0, x0, s)) return;
    *changed = 1;
    uint64_t e = x0[s - 1];
    for (uint64_t u = s;;) {
        const uint64_t xe = frame_walk(F, u, e);
        g1[u] = e; x1[u] = xe;
        if (++u >= F.nseg || g0[u] == xe || chase_start(g0, x0, u)) break;
        e = xe;
    }
}
// the chain positions of segment s (from its right entry): counted, then written
template <bool EMIT>
__global__ void __launch_bounds__(256) bam_frame_emit_kernel(Frame F, const uint64_t* __restrict__ g, uint32_t* __restrict__ cnt, const uint64_t* __restrict__ off, uint64_t* __restrict__ out) {
    const uint64_t s = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= F.nseg) return;
    const uint64_t st = s * SEG, e = seg_end(F, s);
    uint64_t p = g[s], k = 0;
    while (p < e) {
        if (p >= st) { if (EMIT) out[off[s] + k] = p; k++; }
        if (p + 4 > F.n) break;
        p += 4ull + drd32(F.b + p);
    }
    if (!EMIT) cnt[s] = (uint32_t)k;
}
__global__ void set_u64_kernel(uint64_t* p, uint64_t v) { *p = v; }

}  // namespace

struct BgzfStream {
    std::vector<uint8_t> carry;              // host: the incomplete trailing BGZF block of the last call
    bool poisoned = false, header_done = false, last_eof = false;
    uint64_t tail = 0;                       // device: bytes at the front of bam_raw that no complete record covers yet (header or record)
    DBuf<uint8_t> in, spare, dbg_out;        // compressed bytes; second record buffer (swapped with bam_raw); elp_debug_inflate's output
    DBuf<BlockDesc> tab;
    DBuf<uint32_t> status, seg_cnt;
    DBuf<uint64_t> seg;                      // framing: guess and exit of every segment, two generations
    DBuf<uint64_t> d_small;                  // [4] header walk result
    X2n x2n;
};

void bgzf_stream_reset(elp_ctx* c) {
    c->bgzf_open = false;
    if (!c->bgzf) return;
    BgzfStream& S = *c->bgzf;
    S.carry.clear(); S.poisoned = S.header_done = S.last_eof = false; S.tail = 0;
}

void free_state(BgzfStream* S) { delete S; }

static int bgzf_state(elp_ctx* c) {
    if (c->bgzf) return E_OK;
    c->bgzf.reset(new BgzfStream());
    dfl::x2n_table(c->bgzf->x2n.v);
    CUDA_TRY(c, c->bgzf->d_small.fit(4));
    return E_OK;
}

// upload the blocks' compressed bytes (parts: host runs whose concatenation the offsets of `blocks` index) and inflate them to out;
// ELP_EBGZF naming the first bad block
static int inflate_blocks(elp_ctx* c, const char* who, const std::vector<std::pair<const uint8_t*, uint64_t>>& parts, const std::vector<BgzfBlock>& blocks, uint64_t total, uint8_t* out) {
    BgzfStream& S = *c->bgzf;
    cudaStream_t s = c->stream;
    const uint64_t nb = blocks.size();
    uint64_t n_in = 0;
    for (auto& p : parts) n_in += p.second;
    TRY(grow(c, S.in, n_in + 16, 0)); TRY(grow(c, S.tab, nb + 1, 0)); TRY(grow(c, S.status, nb + 1, 0));
    std::vector<BlockDesc> tab(nb);
    for (uint64_t i = 0; i < nb; i++) tab[i] = BlockDesc{blocks[i].cdata_off, blocks[i].out_off, (uint32_t)blocks[i].cdata_len, blocks[i].isize, blocks[i].crc, 0};
    uint64_t at = 0;
    for (auto& p : parts) { if (p.second) CUDA_TRY(c, cudaMemcpyAsync(S.in.p + at, p.first, p.second, cudaMemcpyHostToDevice, s)); at += p.second; }
    CUDA_TRY(c, cudaMemcpyAsync(S.tab.p, tab.data(), nb * sizeof(BlockDesc), cudaMemcpyHostToDevice, s));
    c->begin("bgzf_inflate", (double)n_in + (double)total);
    bgzf_inflate_kernel<<<nblk(nb, INF_WARPS), INF_WARPS * 32, 0, s>>>(S.in.p, S.tab.p, nb, out, S.status.p);
    c->end(); LAUNCH_CHECK(c);
    c->begin("bgzf_crc", (double)total);
    bgzf_crc_kernel<<<nblk(nb, 8), 256, 0, s>>>(S.tab.p, nb, out, S.status.p, S.x2n);
    c->end(); LAUNCH_CHECK(c);
    std::vector<uint32_t> st(nb);
    CUDA_TRY(c, cudaMemcpyAsync(st.data(), S.status.p, nb * 4, cudaMemcpyDeviceToHost, s));
    CUDA_TRY(c, cudaStreamSynchronize(s));   // (tab is pageable and goes out of scope)
    for (uint64_t i = 0; i < nb; i++)
        if (st[i]) return c->fail(E_BGZF, "%s: BGZF block %llu of the call (its DEFLATE data at compressed byte %llu of the uploaded run): %s", who, (unsigned long long)i,
                                  (unsigned long long)blocks[i].cdata_off, dfl::status_text(st[i]));
    return E_OK;
}

int bgzf_inflate_run(elp_ctx* c, const char* who, const uint8_t* in, uint64_t n_in, const std::vector<BgzfBlock>& blocks, uint64_t total, uint8_t* out) {
    TRY(bgzf_state(c));
    return inflate_blocks(c, who, {{in, n_in}}, blocks, total, out);
}

// the reference list of a complete header at bam_raw[0, hdr) against elp_config, or against the input dictionary of elp_set_input_dictionary
// while it is set: n_ref, every l_ref and (when given) every name
static int check_header(elp_ctx* c, uint64_t ref_at, uint64_t hdr) {
    std::vector<uint8_t> h(hdr - ref_at);
    CUDA_TRY(c, cudaMemcpyAsync(h.data(), c->bam_raw.p + ref_at, h.size(), cudaMemcpyDeviceToHost, c->stream));
    CUDA_TRY(c, cudaStreamSynchronize(c->stream));
    const int32_t n_ref = (int32_t)rd32(h.data());
    if (!c->inputs.empty()) {   // elp_add_input: the selected input's @SQ
        const elp_ctx::InputDict& d = c->inputs[c->cur_input];
        if (n_ref != (int32_t)d.len.size()) return c->fail(E_INVAL, "elp_append_bgzf: the BAM header has %d reference sequences, the selected input (elp_select_input %d) has %zu", n_ref, c->cur_input, d.len.size());
        uint64_t x = 4;
        for (int32_t k = 0; k < n_ref; k++) {
            const uint32_t l_name = rd32(h.data() + x);
            const char* name = reinterpret_cast<const char*>(h.data() + x + 4);
            const int32_t l_ref = (int32_t)rd32(h.data() + x + 4 + l_name);
            const std::string nm(name, l_name ? strnlen(name, l_name) : 0);
            if (l_ref != d.len[k] || nm != d.names[k])
                return c->fail(E_INVAL, "elp_append_bgzf: reference %d of the BAM header is '%s' of length %d, the selected input (elp_select_input %d) says '%s' of length %d",
                               k, nm.c_str(), l_ref, c->cur_input, d.names[k].c_str(), d.len[k]);
            x += 8ull + l_name;
        }
        return E_OK;
    }
    if (c->dict_mode) {
        if (n_ref != c->n_in) return c->fail(E_INVAL, "elp_append_bgzf: the BAM header has %d reference sequences, the input dictionary (elp_set_input_dictionary) has %d", n_ref, c->n_in);
        uint64_t x = 4;
        for (int32_t k = 0; k < n_ref; k++) {
            const uint32_t l_name = rd32(h.data() + x);
            const char* name = reinterpret_cast<const char*>(h.data() + x + 4);
            const int32_t l_ref = (int32_t)rd32(h.data() + x + 4 + l_name);
            const std::string nm(name, l_name ? strnlen(name, l_name) : 0);
            if (l_ref != c->in_len[k] || nm != c->in_tab[k])
                return c->fail(E_INVAL, "elp_append_bgzf: reference %d of the BAM header is '%s' of length %d, the input dictionary (elp_set_input_dictionary) says '%s' of length %d",
                               k, nm.c_str(), l_ref, c->in_tab[k].c_str(), c->in_len[k]);
            x += 8ull + l_name;
        }
        return E_OK;
    }
    if (n_ref != c->n_contigs) return c->fail(E_INVAL, "elp_append_bgzf: the BAM header has %d reference sequences, elp_config has %d contigs", n_ref, c->n_contigs);
    uint64_t x = 4;
    for (int32_t k = 0; k < n_ref; k++) {
        const uint32_t l_name = rd32(h.data() + x);
        const char* name = reinterpret_cast<const char*>(h.data() + x + 4);
        const int32_t l_ref = (int32_t)rd32(h.data() + x + 4 + l_name);
        if (l_ref != c->contig_len[k]) return c->fail(E_INVAL, "elp_append_bgzf: reference %d of the BAM header has length %d, elp_config says %d", k, l_ref, c->contig_len[k]);
        const std::string nm(name, l_name ? strnlen(name, l_name) : 0);
        if (c->has_contig_names && nm != c->contig_names[k])
            return c->fail(E_INVAL, "elp_append_bgzf: reference %d of the BAM header is '%s', elp_config says '%s'", k, nm.c_str(), c->contig_names[k].c_str());
        x += 8ull + l_name;
    }
    return E_OK;
}

// record boundaries of bam_raw[0, n): bam_off[0..*nrec] (bam_off[*nrec] = *used, the bytes the complete records take)
static int frame_records(elp_ctx* c, uint64_t n, uint64_t* nrec, uint64_t* used) {
    *nrec = 0; *used = 0;
    if (n == 0) return E_OK;
    BgzfStream& S = *c->bgzf;
    cudaStream_t s = c->stream;
    const uint64_t nseg = (n + SEG - 1) / SEG;
    TRY(grow(c, S.seg, 4 * nseg + 4, 0)); TRY(grow(c, S.seg_cnt, nseg + 8, 0)); TRY(grow(c, c->off_stage, nseg + 2, 0));
    const Frame F{c->bam_raw.p, n, nseg, c->inputs.empty() ? ingest_ref_bound(c, false) : relabel_ref_bound(c)};
    uint64_t *g0 = S.seg.p, *x0 = g0 + nseg, *g1 = x0 + nseg, *x1 = g1 + nseg;   // generation 0 and 1: guesses, then exits
    uint32_t* changed = reinterpret_cast<uint32_t*>(S.d_small.p);
    c->begin("bam_frame", (double)n);
    bam_frame_guess_kernel<<<nblk(nseg, 256), 256, 0, s>>>(F, g0, x0);
    c->end(); LAUNCH_CHECK(c);
    for (uint32_t ch = 1; ch;) {
        CUDA_TRY(c, cudaMemsetAsync(changed, 0, 4, s));
        CUDA_TRY(c, cudaMemcpyAsync(g1, g0, 2 * nseg * 8, cudaMemcpyDeviceToDevice, s));   // (g1, x1 follow g0, x0 in the same layout)
        c->begin("bam_frame", 0);
        bam_frame_fix_kernel<<<nblk(nseg, 256), 256, 0, s>>>(F, g0, x0, g1, x1, changed);
        c->end(); LAUNCH_CHECK(c);
        CUDA_TRY(c, cudaMemcpyAsync(&ch, changed, 4, cudaMemcpyDeviceToHost, s));
        CUDA_TRY(c, cudaStreamSynchronize(s));
        std::swap(g0, g1); std::swap(x0, x1);
    }
    c->begin("bam_frame", 0);
    bam_frame_emit_kernel<false><<<nblk(nseg, 256), 256, 0, s>>>(F, g0, S.seg_cnt.p, nullptr, nullptr);
    c->end(); LAUNCH_CHECK(c);
    TRY(exclusive_scan_u32_to_u64(c, S.seg_cnt.p, c->off_stage.p, nseg));
    uint64_t m = 0, x_last = 0;
    CUDA_TRY(c, cudaMemcpyAsync(&m, c->off_stage.p + nseg, 8, cudaMemcpyDeviceToHost, s));
    CUDA_TRY(c, cudaMemcpyAsync(&x_last, x0 + nseg - 1, 8, cudaMemcpyDeviceToHost, s));
    CUDA_TRY(c, cudaStreamSynchronize(s));
    TRY(grow(c, c->bam_off, m + 2, 0));
    c->begin("bam_frame", 0);
    bam_frame_emit_kernel<true><<<nblk(nseg, 256), 256, 0, s>>>(F, g0, nullptr, c->off_stage.p, c->bam_off.p);
    c->end(); LAUNCH_CHECK(c);
    if (x_last == n) {                                           // the last record ends exactly at n
        set_u64_kernel<<<1, 1, 0, s>>>(c->bam_off.p + m, n); c->launches++; LAUNCH_CHECK(c);
        *nrec = m; *used = n;
    } else {                                                     // the last position starts a record the bytes do not complete
        CUDA_TRY(c, cudaMemcpyAsync(used, c->bam_off.p + m - 1, 8, cudaMemcpyDeviceToHost, s));
        CUDA_TRY(c, cudaStreamSynchronize(s));
        *nrec = m - 1;
    }
    return E_OK;
}

// bam_raw[from, to) -> the front of the spare buffer, which then becomes bam_raw
static int move_to_front(elp_ctx* c, uint64_t from, uint64_t to) {
    BgzfStream& S = *c->bgzf;
    TRY(grow(c, S.spare, to - from + 64, 0));
    if (to > from) CUDA_TRY(c, cudaMemcpyAsync(S.spare.p, c->bam_raw.p + from, to - from, cudaMemcpyDeviceToDevice, c->stream));
    std::swap(c->bam_raw, S.spare);
    return E_OK;
}

static int append_bgzf(elp_ctx* c, const uint8_t* data, uint64_t n) {
    BgzfStream& S = *c->bgzf;
    // whole blocks: the carried block completed from the front of data, then the blocks of the rest; an incomplete trailing block is carried
    std::vector<BgzfBlock> blocks; uint64_t total = 0, k = 0, pre_used = 0;
    std::vector<uint8_t> pre;
    if (!S.carry.empty()) {
        pre = S.carry;
        pre.insert(pre.end(), data, data + std::min<uint64_t>(n, 65536 + 64));
        TRY(scan_blocks(pre.data(), pre.size(), blocks, &total, &pre_used, 1) ? c->fail(E_BGZF, "elp_append_bgzf: malformed BGZF block header") : E_OK);
        if (blocks.empty()) { S.carry = pre; return E_OK; }       // (n < 64 KiB: all of data went into the carry)
        k = pre_used - S.carry.size();
    }
    uint64_t used = 0;
    const size_t n_pre = blocks.size();
    if (scan_blocks(data + k, n - k, blocks, &total, &used)) return c->fail(E_BGZF, "elp_append_bgzf: malformed BGZF block header");
    for (size_t i = n_pre; i < blocks.size(); i++) { blocks[i].cdata_off += pre_used; blocks[i].in_off += pre_used; }
    S.carry.assign(data + k + used, data + n);
    if (blocks.empty()) return E_OK;
    const BgzfBlock& lb = blocks.back();
    const uint8_t* lc = lb.cdata_off < pre_used ? pre.data() + lb.cdata_off : data + k + (lb.cdata_off - pre_used);
    S.last_eof = lb.cdata_len == 2 && lc[0] == 3 && lc[1] == 0 && lb.crc == 0 && lb.isize == 0;   // bgzf-files.go:111-115
    // inflate behind the carried bytes
    const uint64_t t0 = S.tail, avail = t0 + total;
    TRY(grow(c, c->bam_raw, avail + 64, t0));
    TRY(inflate_blocks(c, "elp_append_bgzf", {{pre.data(), pre_used}, {data + k, used}}, blocks, total, c->bam_raw.p + t0));
    S.tail = avail;
    uint64_t start = 0;
    if (!S.header_done) {
        uint64_t r[3] = {0, 0, 0};
        c->begin("bam_header", (double)avail);
        bam_header_walk_kernel<<<1, 32, 0, c->stream>>>(c->bam_raw.p, avail, S.d_small.p);
        c->end(); LAUNCH_CHECK(c);
        CUDA_TRY(c, cudaMemcpyAsync(r, S.d_small.p, 24, cudaMemcpyDeviceToHost, c->stream));
        CUDA_TRY(c, cudaStreamSynchronize(c->stream));
        if (r[0] == 2) return c->fail(E_BAM, "elp_append_bgzf: not a BAM file (magic or header lengths)");
        if (r[0] == 1) return E_OK;                                // the header continues in a later call
        TRY(check_header(c, r[2], r[1]));
        S.header_done = true;
        start = r[1];
    }
    if (start) { TRY(move_to_front(c, start, avail)); S.tail = avail - start; }
    const uint64_t nb = S.tail;
    uint64_t nrec = 0, used_rec = 0;
    TRY(frame_records(c, nb, &nrec, &used_rec));
    if (nrec) {
        if (c->n + nrec >= (1ull << 32)) return c->fail(E_LIMIT, "more than 2^32-1 reads in one context");
        TRY(bam_ingest_core(c, used_rec, nrec));
    }
    if (used_rec) { TRY(move_to_front(c, used_rec, nb)); S.tail = nb - used_rec; }
    return E_OK;
}

extern "C" int elp_append_bgzf(elp_ctx* c, const uint8_t* data, uint64_t n_bytes) {
    if (!c || (!data && n_bytes)) return ELP_EINVAL;
    cudaSetDevice(c->device);
    std::lock_guard<std::mutex> lk(c->append_mu);
    if (c->sorted) return c->fail(E_STATE, "elp_append_bgzf after elp_sort_markdup (call elp_reset first)");
    TRY(bgzf_state(c));
    if (!c->bgzf_open) TRY(relabel_check_selected(c, "elp_append_bgzf"));
    if (c->bgzf->poisoned) return c->fail(E_STATE, "elp_append_bgzf: an earlier call of this file failed (call elp_reset first)");
    c->bgzf_open = true;
    const int rc = append_bgzf(c, data, n_bytes);
    if (rc) c->bgzf->poisoned = true;
    return rc;
}

extern "C" int elp_append_bgzf_end(elp_ctx* c) {
    if (!c) return ELP_EINVAL;
    cudaSetDevice(c->device);
    std::lock_guard<std::mutex> lk(c->append_mu);
    if (!c->bgzf_open || !c->bgzf) return c->fail(E_STATE, "elp_append_bgzf_end without an open file");
    BgzfStream& S = *c->bgzf;
    if (S.poisoned) return c->fail(E_STATE, "elp_append_bgzf_end: an earlier call of this file failed (call elp_reset first)");
    int rc = E_OK;
    if (!S.carry.empty()) rc = c->fail(E_BGZF, "elp_append_bgzf_end: the file ends inside a BGZF block (%zu bytes left)", S.carry.size());
    else if (!S.last_eof) rc = c->fail(E_BGZF, "invalid BGZF file: does not end in proper EOF marker");
    else if (!S.header_done) rc = c->fail(E_BAM, "elp_append_bgzf_end: the file ends inside the BAM header");
    else if (S.tail) rc = c->fail(E_BAM, "elp_append_bgzf_end: the file ends inside an alignment record (%llu bytes left)", (unsigned long long)S.tail);
    if (rc) { S.poisoned = true; return rc; }
    bgzf_stream_reset(c);
    return ELP_OK;
}

extern "C" int elp_debug_inflate(elp_ctx* c, const uint8_t* data, uint64_t n, uint8_t* out, uint64_t capacity, uint64_t* out_n) {
    if (!c || (!data && n) || !out_n) return ELP_EINVAL;
    cudaSetDevice(c->device);
    std::lock_guard<std::mutex> lk(c->append_mu);
    TRY(bgzf_state(c));
    std::vector<BgzfBlock> blocks; uint64_t total = 0;
    if (scan_blocks(data, n, blocks, &total)) return c->fail(E_BGZF, "elp_debug_inflate: malformed BGZF block header");
    if (total > capacity || (!out && total)) return c->fail(E_INVAL, "elp_debug_inflate: output buffer too small (%llu > %llu)", (unsigned long long)total, (unsigned long long)capacity);
    BgzfStream& S = *c->bgzf;
    TRY(grow(c, S.dbg_out, total + 64, 0));
    if (!blocks.empty()) TRY(inflate_blocks(c, "elp_debug_inflate", {{data, n}}, blocks, total, S.dbg_out.p));
    if (total) {
        CUDA_TRY(c, cudaMemcpyAsync(out, S.dbg_out.p, total, cudaMemcpyDeviceToHost, c->stream));
        CUDA_TRY(c, cudaStreamSynchronize(c->stream));
    }
    *out_n = total;
    return ELP_OK;
}
