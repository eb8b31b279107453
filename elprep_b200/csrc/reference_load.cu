// reference_load.cu -- --reference on the device: an .elfasta file, or a FASTA file (plain or BGZF-compressed), read into the one-hot
// reference of every contig (elp_load_reference).
//
// The format is decided from the content: ElfastaMagic 31 FA 57 A1 (fasta/fasta-files.go:237) is an .elfasta, a first byte 0x1f is BGZF
// (bgzf.IsGzip, utils.HandleBGZF), anything else is FASTA text.
// FASTA follows ParseFasta(path, nil, false, false) and contigFromHeader (fasta-files.go:75-89,159-229), chunk by chunk:
//   host            plain text goes through the two page-locked chunks of file_stage.cuh, the upload of chunk k+1 overlapping the kernels
//                   of chunk k; BGZF goes through the same chunks as whole blocks (bgzf_scan.hpp, a partial block carried on the host) and
//                   is inflated by the kernels behind elp_append_bgzf (bgzf_inflate, bgzf_crc).  Either way the new text lands FA_FRONT
//                   bytes into a device buffer, and the partial line at the end of the previous chunk is copied on the device right in
//                   front of it.  The host never reads a base.
//   fasta_lines     the line finder of text_parse.cuh
//   fasta_classify  one thread per line: empty, header or sequence; the 65536-byte limit; the empty-line rule (a sequence line right after
//                   an empty line is refused; whether the last line of a chunk was empty is carried in a device word); the first non-empty
//                   line of the file; a header's name
//   fasta_scatter   one warp per line: a sequence line's bytes to the raw sequence buffer at the exclusive scan of the line lengths, a
//                   header's name, line and raw offset to the header list (copied to the host: a few thousand at most)
//   ref_pack        after the last chunk, the sequence of each name that is an @SQ SN, from the raw buffer through ref_pack_hot_kernel
// .elfasta follows OpenElfasta (fasta-files.go:286-336): the offset table is read and checked on the host; only the byte ranges of names
// that are an @SQ SN are read, through the same chunks, and ref_pack_span_kernel packs each chunk at its base offset in the contig.
// Nothing is installed before the whole file was accepted; the new references are one allocation (ContigTable::block of elp_ctx::ref).
#include <algorithm>
#include <cerrno>
#include <cstdio>
#include <cstring>
#include <map>
#include <string>
#include <sys/stat.h>
#include <vector>
#include "ctx.h"
#include "text_parse.cuh"
#include "file_stage.cuh"
#include "bgzf_scan.hpp"
#include "refhot.cuh"
#include "../../include/elprep_b200.h"

namespace {

constexpr uint64_t FA_MAX_LINE = 65536;          // bufio.MaxScanTokenSize: a longer line stops the reference's scanner
constexpr uint64_t FA_FRONT = FA_MAX_LINE;       // device bytes ahead of each chunk's text: room for the carried partial line
constexpr uint64_t REF_CHUNK_DEFAULT = 32ull << 20;
constexpr uint64_t BGZF_MAX_BLOCK = 65536;
const uint8_t ELFASTA_MAGIC[4] = {0x31, 0xFA, 0x57, 0xA1};
constexpr int VARINT_FIELD = 10;                 // binary.MaxVarintLen64


// why a FASTA file is refused; the smallest (line << 8 | code) is reported (1-based lines)
enum FaErr : uint32_t { FA_FIRST = 1, FA_LONG, FA_EMPTY };
const char* fa_err_text(uint32_t e) {
    switch (e) {
        case FA_FIRST: return "invalid fasta file - missing first header";
        case FA_LONG: return "line of 65536 bytes or more (bufio.Scanner: token too long)";
        case FA_EMPTY: return "invalid fasta file - empty line";
        default: return "?";
    }
}
// device words of one load: the smallest error, the first non-empty line (line << 1 | not a header), and two slots of "the line before
// the chunk is empty" (the file start counts as one)
enum { W_ERR = 0, W_FIRST = 1, W_PREV = 2, W_N = 4 };

__device__ __forceinline__ bool graphic(uint8_t b) { return b >= '!' && b <= '~'; }

// bufio.ScanLines' token of line k: its bytes before '\n' (*raw), minus one '\r' before it
__device__ __forceinline__ uint64_t token_len(const uint8_t* t, const uint64_t* ls, uint64_t k, uint64_t* raw) {
    const uint64_t s0 = ls[k], r = ls[k + 1] - 1 - s0;
    *raw = r;
    return r && t[s0 + r - 1] == '\r' ? r - 1 : r;
}

// ---- fasta_classify ----
struct FaArgs {
    const uint8_t* t; const uint64_t* ls; uint64_t n_lines, line0;   // line0: the 1-based number of line 0
    const unsigned long long* prev_in; unsigned long long* prev_out;
    uint32_t* seqlen; uint32_t* hdr; uint32_t* namelen; uint32_t* namest;
    unsigned long long* w;
};

// ParseFasta's loop body for one line (fasta-files.go:176-226)
__global__ void __launch_bounds__(256) fasta_classify_kernel(FaArgs A) {
    const uint64_t k = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= A.n_lines) return;
    uint64_t raw, praw;
    const uint64_t n = token_len(A.t, A.ls, k, &raw), line = A.line0 + k;
    const uint8_t* p = A.t + A.ls[k];
    const bool prev_empty = k ? token_len(A.t, A.ls, k - 1, &praw) == 0 : *A.prev_in != 0;
    uint32_t sl = 0, h = 0, nl = 0, ns = 0;
    if (raw >= FA_MAX_LINE) atomicMin(A.w + W_ERR, ((unsigned long long)line << 8) | FA_LONG);
    else if (n) {
        const bool header = p[0] == '>';
        if (prev_empty) atomicMin(A.w + W_FIRST, ((unsigned long long)line << 1) | (header ? 0u : 1u));   // only such a line can be the first
        if (!header) {
            sl = (uint32_t)n;
            if (prev_empty) atomicMin(A.w + W_ERR, ((unsigned long long)line << 8) | FA_EMPTY);
        } else {   // contigFromHeader (fasta-files.go:75-89); with no byte in '!'..'~', Go slices the one byte past the token
            h = 1;
            uint64_t i = 1;
            while (i < n && !graphic(p[i])) i++;
            uint64_t j = i + 1;
            while (j < n && graphic(p[j])) j++;
            ns = (uint32_t)i; nl = (uint32_t)(j - i);
        }
    }
    if (k == A.n_lines - 1) *A.prev_out = raw < FA_MAX_LINE && n == 0;
    A.seqlen[k] = sl; A.hdr[k] = h; A.namelen[k] = nl; A.namest[k] = ns;
}

// ---- fasta_scatter ----
struct FaScatter {
    const uint8_t* t; const uint64_t* ls; uint64_t n_lines, line0;
    const uint32_t* seqlen; const uint32_t* namelen; const uint32_t* namest;
    const uint64_t* seq_off; const uint64_t* hdr_off; const uint64_t* name_off;   // exclusive scans of seqlen, hdr, namelen
    uint8_t* raw; uint64_t raw_base;
    uint64_t* hdr_line; uint64_t* hdr_raw; uint64_t* hdr_name; uint8_t* names;
};

__global__ void __launch_bounds__(256) fasta_scatter_kernel(FaScatter A) {
    const unsigned lane = threadIdx.x & 31;
    const uint64_t nw = (uint64_t)gridDim.x * (blockDim.x >> 5);
    for (uint64_t k = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; k < A.n_lines; k += nw) {
        const uint8_t* p = A.t + A.ls[k];
        const uint32_t sl = A.seqlen[k];
        if (sl) {
            uint8_t* d = A.raw + A.raw_base + A.seq_off[k];
            for (uint32_t j = lane; j < sl; j += 32) d[j] = p[j];
        } else if (const uint32_t nl = A.namelen[k]) {
            const uint64_t h = A.hdr_off[k], no = A.name_off[k];
            if (lane == 0) { A.hdr_line[h] = A.line0 + k; A.hdr_raw[h] = A.raw_base + A.seq_off[k]; A.hdr_name[h] = no; }
            const uint8_t* q = p + A.namest[k];
            for (uint32_t j = lane; j < nl; j += 32) A.names[no + j] = q[j];
        }
    }
}

// ---- host side ----
struct RefScratch {   // per call; freed on return
    DBuf<uint32_t> cnt, seqlen, hdr, namelen, namest;
    DBuf<uint64_t> cnt_off, ls, seq_off, hdr_off, name_off, hdr_line, hdr_raw, hdr_name;
    DBuf<uint8_t> raw, names, tb[2];
    DBuf<unsigned long long> d_w;
    HBuf<unsigned long long> h_w;   // [0, 8) readbacks, [8, 16) uploads
    FileStage S;                    // last: destroyed first, so its uploads have landed before the buffers above are freed
};

struct Seq { std::string name; uint64_t line, raw, len; };   // one header of the file and its sequence in the raw buffer

struct FaState {      // carried from chunk to chunk
    uint64_t line0 = 1;                                      // the 1-based number of the next chunk's first line
    uint64_t raw_total = 0;                                  // sequence bytes so far
    unsigned long long first = ~0ull;                        // the W_FIRST word after the last chunk
    int prev = 0;                                            // the W_PREV slot the next chunk reads
    const uint8_t* carry = nullptr; uint64_t carry_n = 0;    // the partial line at the end of the last chunk (device)
    std::vector<Seq> seqs;
};

// one chunk of text: nnew bytes at buf + FA_FRONT (zero bytes behind them), behind the carried partial line; `overlap` runs on the host
// while the line count runs
template <class F>
int fasta_chunk(elp_ctx* c, RefScratch& X, FaState& St, uint8_t* buf, uint64_t nnew, bool last, const char* path, cudaEvent_t release_prev, F&& overlap) {
    cudaStream_t s = c->stream;
    unsigned long long* hw = X.h_w.p;
    const uint64_t nc = St.carry_n, a = (FA_FRONT - nc) & ~(uint64_t)(SAM_CHUNK - 1), front = FA_FRONT - nc - a, end = FA_FRONT + nnew - a;
    uint8_t* t = buf + a;
    if (nc) CUDA_TRY(c, cudaMemcpyAsync(buf + FA_FRONT - nc, St.carry, nc, cudaMemcpyDeviceToDevice, s));
    if (front) CUDA_TRY(c, cudaMemsetAsync(t, 0, front, s));   // (no '\n' in front of the first line)
    if (release_prev) CUDA_TRY(c, cudaEventRecord(release_prev, s));
    St.carry = nullptr; St.carry_n = 0;
    if (end == front) return overlap();
    const uint64_t n_chunks = (end + SAM_CHUNK - 1) / SAM_CHUNK;
    TRY(grow(c, X.cnt, n_chunks + 8, 0)); TRY(grow(c, X.cnt_off, n_chunks + 2, 0));
    c->begin("fasta_lines", (double)(end - front));
    sam_count_kernel<<<nblk(n_chunks, 256), 256, 0, s>>>(t, n_chunks, X.cnt.p);
    c->end(); LAUNCH_CHECK(c);
    TRY(exclusive_scan_u32_to_u64(c, X.cnt.p, X.cnt_off.p, n_chunks));
    CUDA_TRY(c, cudaMemcpyAsync(hw, X.cnt_off.p + n_chunks, 8, cudaMemcpyDeviceToHost, s));
    TRY(overlap());
    CUDA_TRY(c, cudaStreamSynchronize(s));
    const uint64_t n_nl = hw[0];
    TRY(grow(c, X.ls, n_nl + 2, 0));
    hw[8] = front;
    CUDA_TRY(c, cudaMemcpyAsync(X.ls.p, hw + 8, 8, cudaMemcpyHostToDevice, s));
    c->begin("fasta_lines", (double)(end - front) + 8.0 * (double)n_nl);
    sam_lines_kernel<<<nblk(n_chunks, 256), 256, 0, s>>>(t, n_chunks, X.cnt_off.p, X.ls.p);
    c->end(); LAUNCH_CHECK(c);
    CUDA_TRY(c, cudaMemcpyAsync(hw + 1, X.ls.p + n_nl, 8, cudaMemcpyDeviceToHost, s));
    CUDA_TRY(c, cudaStreamSynchronize(s));
    const uint64_t m = hw[1];   // the end of the whole lines
    uint64_t nl = n_nl;
    if (last && m < end) { hw[9] = end + 1; nl++; CUDA_TRY(c, cudaMemcpyAsync(X.ls.p + nl, hw + 9, 8, cudaMemcpyHostToDevice, s)); }   // a virtual '\n'
    if (!last) { St.carry = t + m; St.carry_n = end - m; }
    if (nl) {
        TRY(grow(c, X.seqlen, nl + 8, 0)); TRY(grow(c, X.hdr, nl + 8, 0)); TRY(grow(c, X.namelen, nl + 8, 0)); TRY(grow(c, X.namest, nl + 8, 0));
        TRY(grow(c, X.seq_off, nl + 2, 0)); TRY(grow(c, X.hdr_off, nl + 2, 0)); TRY(grow(c, X.name_off, nl + 2, 0));
        FaArgs A{};
        A.t = t; A.ls = X.ls.p; A.n_lines = nl; A.line0 = St.line0;
        A.prev_in = X.d_w.p + W_PREV + St.prev; A.prev_out = X.d_w.p + W_PREV + (St.prev ^ 1);
        A.seqlen = X.seqlen.p; A.hdr = X.hdr.p; A.namelen = X.namelen.p; A.namest = X.namest.p; A.w = X.d_w.p;
        c->begin("fasta_classify", (double)(m - front) + 8.0 * (double)(nl + 1) + 16.0 * (double)nl);
        fasta_classify_kernel<<<nblk(nl, 256), 256, 0, s>>>(A);
        c->end(); LAUNCH_CHECK(c);
        TRY(exclusive_scan_u32_to_u64(c, X.seqlen.p, X.seq_off.p, nl));
        TRY(exclusive_scan_u32_to_u64(c, X.hdr.p, X.hdr_off.p, nl));
        TRY(exclusive_scan_u32_to_u64(c, X.namelen.p, X.name_off.p, nl));
        CUDA_TRY(c, cudaMemcpyAsync(hw + 2, X.seq_off.p + nl, 8, cudaMemcpyDeviceToHost, s));
        CUDA_TRY(c, cudaMemcpyAsync(hw + 3, X.hdr_off.p + nl, 8, cudaMemcpyDeviceToHost, s));
        CUDA_TRY(c, cudaMemcpyAsync(hw + 4, X.name_off.p + nl, 8, cudaMemcpyDeviceToHost, s));
        CUDA_TRY(c, cudaMemcpyAsync(hw + 5, X.d_w.p, 16, cudaMemcpyDeviceToHost, s));
        CUDA_TRY(c, cudaStreamSynchronize(s));
        St.prev ^= 1;
        St.first = hw[6];
        unsigned long long err = hw[5];
        if (St.first != ~0ull && (St.first & 1)) err = std::min(err, ((St.first >> 1) << 8) | FA_FIRST);
        if (err != ~0ull) return c->fail(E_FASTA, "elp_load_reference: %s, line %llu: %s", path, err >> 8, fa_err_text((uint32_t)(err & 0xff)));
        const uint64_t nseq = hw[2], nh = hw[3], nname = hw[4], r0 = St.raw_total;
        if (r0 + nseq + 64 > X.raw.cap) TRY(grow(c, X.raw, std::max<size_t>(r0 + nseq + 64, 2 * X.raw.cap), r0));
        TRY(grow(c, X.hdr_line, nh + 1, 0)); TRY(grow(c, X.hdr_raw, nh + 1, 0)); TRY(grow(c, X.hdr_name, nh + 1, 0)); TRY(grow(c, X.names, nname + 1, 0));
        FaScatter B{};
        B.t = t; B.ls = X.ls.p; B.n_lines = nl; B.line0 = St.line0;
        B.seqlen = X.seqlen.p; B.namelen = X.namelen.p; B.namest = X.namest.p;
        B.seq_off = X.seq_off.p; B.hdr_off = X.hdr_off.p; B.name_off = X.name_off.p;
        B.raw = X.raw.p; B.raw_base = r0; B.hdr_line = X.hdr_line.p; B.hdr_raw = X.hdr_raw.p; B.hdr_name = X.hdr_name.p; B.names = X.names.p;
        c->begin("fasta_scatter", 2.0 * (double)(m - front) + 28.0 * (double)nl);
        fasta_scatter_kernel<<<(unsigned)std::min<uint64_t>(nblk(nl, 8), 132 * 32), 256, 0, s>>>(B);
        c->end(); LAUNCH_CHECK(c);
        if (nh) {
            std::vector<uint64_t> hl(nh), hr(nh), hn(nh); std::vector<char> nm(nname);
            CUDA_TRY(c, cudaMemcpyAsync(hl.data(), X.hdr_line.p, nh * 8, cudaMemcpyDeviceToHost, s));
            CUDA_TRY(c, cudaMemcpyAsync(hr.data(), X.hdr_raw.p, nh * 8, cudaMemcpyDeviceToHost, s));
            CUDA_TRY(c, cudaMemcpyAsync(hn.data(), X.hdr_name.p, nh * 8, cudaMemcpyDeviceToHost, s));
            CUDA_TRY(c, cudaMemcpyAsync(nm.data(), X.names.p, nname, cudaMemcpyDeviceToHost, s));
            CUDA_TRY(c, cudaStreamSynchronize(s));
            for (uint64_t i = 0; i < nh; i++) St.seqs.push_back(Seq{std::string(nm.data() + hn[i], (i + 1 < nh ? hn[i + 1] : nname) - hn[i]), hl[i], hr[i], 0});
        }
        St.raw_total = r0 + nseq;
        St.line0 += nl;
    }
    if (St.carry_n >= FA_MAX_LINE) return c->fail(E_FASTA, "elp_load_reference: %s, line %llu: %s", path, (unsigned long long)St.line0, fa_err_text(FA_LONG));
    return E_OK;
}

int read_fail(elp_ctx* c, const char* path) { return c->fail(E_INVAL, "elp_load_reference: cannot read %s: %s", path, strerror(errno)); }

// plain FASTA text: chunk k+1 is read and uploaded while the line count of chunk k runs
int load_fasta_plain(elp_ctx* c, RefScratch& X, FaState& St, FILE* f, const char* path, uint64_t size, uint64_t chunk) {
    FileStage& S = X.S;
    TRY(stage_init(c, S, chunk, chunk, FA_FRONT + stage_padded(chunk), "elp_load_reference"));
    TRY(grow(c, X.raw, size + 64, 0));   // the sequence bytes are at most the file's bytes
    auto fill = [&](int b, uint64_t* got, bool* last) -> int {
        TRY(stage_wait_host(c, S, b));
        *got = fread(S.h[b].p, 1, chunk, f);
        if (*got < chunk && ferror(f)) return read_fail(c, path);
        *last = *got < chunk;
        return stage_upload(c, S, b, *got, FA_FRONT);
    };
    int b = 0; uint64_t got = 0; bool last = false;
    TRY(fill(b, &got, &last));
    for (;;) {
        uint64_t got2 = 0; bool last2 = true;
        CUDA_TRY(c, cudaStreamWaitEvent(c->stream, S.up[b], 0));
        if (!got) CUDA_TRY(c, cudaMemsetAsync(S.d[b].p + FA_FRONT, 0, SAM_CHUNK, c->stream));
        TRY(fasta_chunk(c, X, St, S.d[b].p, got, last, path, S.used[b ^ 1], [&]() { return last ? E_OK : fill(b ^ 1, &got2, &last2); }));
        if (last) break;
        b ^= 1; got = got2; last = last2;   // (fasta_chunk of the next chunk records used[b ^ 1] behind its copy of the carried line)
    }
    return E_OK;
}

// BGZF FASTA: the whole blocks of each chunk inflated on the device, an incomplete last block carried to the next chunk on the host
int load_fasta_bgzf(elp_ctx* c, RefScratch& X, FaState& St, FILE* f, const char* path, uint64_t chunk) {
    FileStage& S = X.S;
    TRY(stage_init(c, S, chunk, chunk + BGZF_MAX_BLOCK, SAM_CHUNK, "elp_load_reference"));
    std::vector<uint8_t> cz;
    std::vector<BgzfBlock> blocks;
    uint64_t at = 0;   // file offset of h[0][0]
    bool eof_block = false;
    int b = 0;
    for (;;) {
        uint8_t* h = S.h[0].p;
        const uint64_t nc = cz.size();
        if (nc) memcpy(h, cz.data(), nc);
        const size_t got = fread(h + nc, 1, chunk, f);
        if (got < chunk && ferror(f)) return read_fail(c, path);
        const bool last = got < chunk;
        const uint64_t n = nc + got;
        uint64_t total = 0, used = 0;
        blocks.clear();
        if (scan_blocks(h, n, blocks, &total, &used)) {
            const uint64_t bad = blocks.empty() ? 0 : blocks.back().cdata_off + blocks.back().cdata_len + BGZF_TRL;
            return c->fail(E_BGZF, "elp_load_reference: %s, file offset %llu: malformed BGZF block header (gzip magic, FEXTRA, BC subfield, block size or ISIZE)", path,
                           (unsigned long long)(at + bad));
        }
        if (last && used < n)
            return c->fail(E_BGZF, "elp_load_reference: %s, file offset %llu: the file ends inside a BGZF block (%llu bytes left)", path, (unsigned long long)(at + used),
                           (unsigned long long)(n - used));
        if (!blocks.empty()) {
            const BgzfBlock& lb = blocks.back();
            eof_block = lb.cdata_len == 2 && h[lb.cdata_off] == 3 && h[lb.cdata_off + 1] == 0 && lb.crc == 0 && lb.isize == 0;   // bgzf-files.go:111-115
        }
        if (last && !eof_block) return c->fail(E_BGZF, "elp_load_reference: %s, file offset %llu: invalid BGZF file: does not end in proper EOF marker", path, (unsigned long long)(at + used));
        if (!blocks.empty() || last) {
            TRY(grow(c, X.tb[b], FA_FRONT + stage_padded(total), 0));
            if (!blocks.empty()) {
                char who[1200];
                snprintf(who, sizeof who, "elp_load_reference: %s, BGZF blocks from file offset %llu", path, (unsigned long long)at);
                TRY(bgzf_inflate_run(c, who, h, used, blocks, total, X.tb[b].p + FA_FRONT));
            }
            CUDA_TRY(c, cudaMemsetAsync(X.tb[b].p + FA_FRONT + total, 0, stage_padded(total) - total, c->stream));
            TRY(fasta_chunk(c, X, St, X.tb[b].p, total, last, path, nullptr, []() { return E_OK; }));
            b ^= 1;
        }
        cz.assign(h + used, h + n);
        at += used;
        if (last) return E_OK;
    }
}

// binary.Varint over a 10-byte field: *n <= 0 when it fails (fasta-files.go:313-324)
int64_t go_varint(const uint8_t* p, int* n) {
    uint64_t x = 0; unsigned s = 0;
    *n = 0;
    for (int i = 0; i < VARINT_FIELD; i++) {
        const uint8_t b = p[i];
        if (b < 0x80) {
            if (i == VARINT_FIELD - 1 && b > 1) { *n = -(i + 1); return 0; }
            x |= (uint64_t)b << s;
            *n = i + 1;
            const int64_t v = (int64_t)(x >> 1);
            return (x & 1) ? ~v : v;
        }
        x |= (uint64_t)(b & 0x7f) << s;
        s += 7;
    }
    return 0;
}

struct Span { uint64_t off, len; };

// OpenElfasta's table walk: name -> byte range, the last of equal names winning; every entry is checked
int elfasta_table(elp_ctx* c, FILE* f, const char* path, uint64_t size, std::map<std::string, Span>& out) {
    std::vector<uint8_t> d;
    auto have = [&](uint64_t i) -> int {   // 1: byte i is in d; 0: it lies past the end of the file; < 0: read error
        while (d.size() <= i) {
            if (d.size() >= size) return 0;
            const uint64_t k = std::min<uint64_t>(size - d.size(), 1 << 16), o = d.size();
            d.resize(o + k);
            if (fread(d.data() + o, 1, k, f) != k) return -1;
        }
        return 1;
    };
    auto bad = [&](uint64_t at, const char* why) { return c->fail(E_FASTA, "elp_load_reference: %s, .elfasta byte offset %llu: %s", path, (unsigned long long)at, why); };
    int r;
    uint64_t i = sizeof ELFASTA_MAGIC;
    for (;;) {
        if ((r = have(i)) <= 0) return r < 0 ? read_fail(c, path) : bad(i, "the offset table runs past the end of the file");
        if (d[i] == '\n') return E_OK;
        const uint64_t start = i;
        for (;; i++) {
            if ((r = have(i)) <= 0) return r < 0 ? read_fail(c, path) : bad(start, "the name of an offset table entry runs past the end of the file");
            if (d[i] == '\t') break;
        }
        std::string name(reinterpret_cast<const char*>(d.data() + start), i - start);
        i++;
        int n = 0;
        if ((r = have(i + VARINT_FIELD - 1)) <= 0) return r < 0 ? read_fail(c, path) : bad(i, "the offset field runs past the end of the file");
        const int64_t off = go_varint(d.data() + i, &n);
        if (n <= 0) return bad(i, "bad number of bytes while parsing offset");
        if ((r = have(i + 2 * VARINT_FIELD - 1)) <= 0) return r < 0 ? read_fail(c, path) : bad(i + VARINT_FIELD, "the size field runs past the end of the file");
        const int64_t sz = go_varint(d.data() + i + VARINT_FIELD, &n);
        if (n <= 0) return bad(i + VARINT_FIELD, "bad number of bytes while parsing size");
        const int64_t hi = (int64_t)((uint64_t)off + (uint64_t)sz);   // data[offset:offset+size] (Go int arithmetic wraps)
        if (off < 0 || hi < off || (uint64_t)hi > size) return bad(i, "the sequence [offset, offset + size) lies outside the file");
        out[name] = Span{(uint64_t)off, (uint64_t)(hi - off)};
        i += 2 * VARINT_FIELD;
    }
}

// the new references: one zeroed allocation, a region per distinct matched name (shared by the @SQ lines with that SN)
struct Install {
    DBuf<uint8_t> block; uint64_t bytes = 0;
    std::vector<uint8_t*> ref; std::vector<uint64_t> len;   // per contig: the payload of its region (nullptr: no sequence) and its length
};
inline uint64_t region_bytes(uint64_t n) { return (n + 1) / 2 + REFHOT_PAD + 64; }

// names -> regions.  lens[name] is the sequence length of every name the file has; *n_unmatched, *n_missing as elp_load_reference;
// region[name] receives the payload pointer (past REFHOT_PAD) of the names some contig uses
// (fasta: a one-byte name outside '!'..'~' is the byte Go read past a header without a name, and matches nothing)
int plan_install(elp_ctx* c, const std::map<std::string, uint64_t>& lens, bool fasta, Install& I, std::map<std::string, uint8_t*>& region,
                 uint64_t* n_unmatched, int32_t* n_missing) {
    const int nc = c->n_contigs;
    std::map<std::string, int> sn;
    for (int i = 0; i < nc; i++) sn[c->contig_names[i]] = i;
    uint64_t um = 0;
    std::map<std::string, uint64_t> at;
    for (auto& kv : lens) {
        const bool nameless = fasta && kv.first.size() == 1 && !(kv.first[0] >= '!' && kv.first[0] <= '~');
        if (nameless || !sn.count(kv.first)) { um++; continue; }
        at[kv.first] = I.bytes;
        I.bytes += region_bytes(kv.second);
    }
    if (I.bytes) {
        cudaError_t e = I.block.fit(I.bytes);
        if (e != cudaSuccess) { cudaGetLastError(); return c->fail(e == cudaErrorMemoryAllocation ? E_NOMEM : E_CUDA, "elp_load_reference: device allocation of %llu bytes failed", (unsigned long long)I.bytes); }
        CUDA_TRY(c, cudaMemsetAsync(I.block.p, 0, I.bytes, c->stream));
    }
    I.ref.assign(nc, nullptr); I.len.assign(nc, 0);
    int32_t miss = 0;
    for (int i = 0; i < nc; i++) {
        auto it = at.find(c->contig_names[i]);
        if (it == at.end()) { miss++; continue; }
        I.ref[i] = I.block.p + it->second + REFHOT_PAD; I.len[i] = lens.at(it->first);
    }
    for (auto& kv : at) region[kv.first] = I.block.p + kv.second + REFHOT_PAD;
    *n_unmatched = um; *n_missing = miss;
    return E_OK;
}

int load_fasta(elp_ctx* c, RefScratch& X, FILE* f, const char* path, bool bgzf, uint64_t size, uint64_t chunk, Install& I, uint64_t* n_unmatched, int32_t* n_missing) {
    FaState St;
    TRY(bgzf ? load_fasta_bgzf(c, X, St, f, path, chunk) : load_fasta_plain(c, X, St, f, path, size, chunk));
    if (St.first == ~0ull) return c->fail(E_FASTA, "elp_load_reference: %s, line %llu: empty fasta file", path, (unsigned long long)St.line0);
    // fasta[contig] = seq (fasta-files.go:192,219): the last of equal names wins
    std::map<std::string, uint64_t> lens, where;
    for (size_t i = 0; i < St.seqs.size(); i++) {
        Seq& q = St.seqs[i];
        q.len = (i + 1 < St.seqs.size() ? St.seqs[i + 1].raw : St.raw_total) - q.raw;
        lens[q.name] = q.len; where[q.name] = q.raw;
    }
    std::map<std::string, uint8_t*> region;
    TRY(plan_install(c, lens, true, I, region, n_unmatched, n_missing));
    for (auto& kv : region) {
        const uint64_t n = lens[kv.first];
        if (!n) continue;
        c->begin("ref_pack", 1.5 * (double)n);
        ref_pack_hot_kernel<<<nblk((n + 1) / 2, 256), 256, 0, c->stream>>>(X.raw.p + where[kv.first], n, kv.second, (n + 1) / 2);
        c->end(); LAUNCH_CHECK(c);
    }
    CUDA_TRY(c, cudaStreamSynchronize(c->stream));
    return E_OK;
}

int load_elfasta(elp_ctx* c, RefScratch& X, FILE* f, const char* path, uint64_t size, uint64_t chunk, Install& I, uint64_t* n_unmatched, int32_t* n_missing) {
    std::map<std::string, Span> tab;
    TRY(elfasta_table(c, f, path, size, tab));
    std::map<std::string, uint64_t> lens;
    for (auto& kv : tab) lens[kv.first] = kv.second.len;
    std::map<std::string, uint8_t*> region;
    TRY(plan_install(c, lens, false, I, region, n_unmatched, n_missing));
    // the matched ranges, in file order, cut into chunks; each chunk is packed at its base offset in its contig
    struct Piece { uint64_t off, len, b0; uint8_t* out; };
    std::vector<Piece> pieces;
    std::vector<std::pair<Span, uint8_t*>> spans;
    for (auto& kv : region) spans.push_back({tab[kv.first], kv.second});
    std::sort(spans.begin(), spans.end(), [](const std::pair<Span, uint8_t*>& x, const std::pair<Span, uint8_t*>& y) { return x.first.off < y.first.off; });
    for (auto& sp : spans)
        for (uint64_t b0 = 0; b0 < sp.first.len; b0 += chunk) pieces.push_back(Piece{sp.first.off + b0, std::min(chunk, sp.first.len - b0), b0, sp.second});
    if (pieces.empty()) return E_OK;
    FileStage& S = X.S;
    TRY(stage_init(c, S, chunk, chunk, stage_padded(chunk), "elp_load_reference"));
    cudaStream_t s = c->stream;
    for (size_t i = 0; i < pieces.size(); i++) {
        const Piece& p = pieces[i];
        const int b = (int)(i & 1);
        TRY(stage_wait_host(c, S, b));   // (the host reads piece i + 1 while piece i uploads and packs)
        if (fseeko(f, (off_t)p.off, SEEK_SET) != 0 || fread(S.h[b].p, 1, p.len, f) != p.len) return read_fail(c, path);
        TRY(stage_upload(c, S, b, p.len, 0));
        CUDA_TRY(c, cudaStreamWaitEvent(s, S.up[b], 0));
        const uint64_t n_out = (p.b0 + p.len + 1) / 2 - p.b0 / 2;
        c->begin("ref_pack", 1.5 * (double)p.len);
        ref_pack_span_kernel<<<nblk(n_out, 256), 256, 0, s>>>(S.d[b].p, p.len, p.b0, p.out);
        c->end(); LAUNCH_CHECK(c);
        CUDA_TRY(c, cudaEventRecord(S.used[b], s));
    }
    CUDA_TRY(c, cudaStreamSynchronize(s));
    return E_OK;
}

}  // namespace

extern "C" int elp_load_reference(elp_ctx* c, const char* path, uint64_t* n_unmatched, int32_t* n_missing) {
    if (!c) return ELP_EINVAL;
    cudaSetDevice(c->device);
    if (!path) return c->fail(E_INVAL, "elp_load_reference: path is null");
    if (c->n_contigs > 0 && !c->has_contig_names)
        return c->fail(E_INVAL, "elp_load_reference: the context was created without elp_config.contig_names, so sequence names cannot be resolved");
    FILE* f = fopen(path, "rb");
    if (!f) return c->fail(E_INVAL, "elp_load_reference: cannot open %s: %s", path, strerror(errno));
    struct Closer { FILE* f; ~Closer() { fclose(f); } } closer{f};
    struct stat sb;
    if (fstat(fileno(f), &sb) != 0) return read_fail(c, path);
    const uint64_t size = (uint64_t)sb.st_size, chunk = c->ref_chunk ? c->ref_chunk : REF_CHUNK_DEFAULT;
    uint8_t magic[4] = {0, 0, 0, 0};
    const size_t got = fread(magic, 1, 4, f);
    if (got < 4 && ferror(f)) return read_fail(c, path);
    if (fseeko(f, 0, SEEK_SET) != 0) return read_fail(c, path);
    RefScratch X;
    CUDA_TRY(c, X.d_w.fit(W_N));
    CUDA_TRY(c, X.h_w.fit(16));
    const unsigned long long w0[W_N] = {~0ull, ~0ull, 1, 0};   // the file start counts as an empty line before line 1
    CUDA_TRY(c, cudaMemcpy(X.d_w.p, w0, sizeof w0, cudaMemcpyHostToDevice));
    Install I;
    uint64_t um = 0; int32_t miss = 0;
    if (got == 4 && memcmp(magic, ELFASTA_MAGIC, 4) == 0) TRY(load_elfasta(c, X, f, path, size, chunk, I, &um, &miss));
    else TRY(load_fasta(c, X, f, path, got > 0 && magic[0] == 0x1f, size, chunk, I, &um, &miss));
    c->ref.install(std::move(I.block), std::move(I.ref), std::move(I.len));   // every contig's reference is replaced
    if (n_unmatched) *n_unmatched = um;
    if (n_missing) *n_missing = miss;
    return ELP_OK;
}

extern "C" int64_t elp_reference_get(elp_ctx* c, int32_t contig, uint8_t* nibbles, uint64_t cap) {
    if (!c) return -1;
    cudaSetDevice(c->device);
    if (contig < 0 || contig >= c->n_contigs) { c->fail(E_INVAL, "elp_reference_get: contig %d out of range", contig); return -1; }
    const uint64_t n = c->ref.n[contig], k = (n + 1) / 2;
    const uint8_t* p = c->ref.d[contig];
    if (nibbles && p && k && cap >= k) {
        if (cudaMemcpyAsync(nibbles, p, k, cudaMemcpyDeviceToHost, c->stream) != cudaSuccess || cudaStreamSynchronize(c->stream) != cudaSuccess) {
            c->fail(E_CUDA, "elp_reference_get: %s", cudaGetErrorString(cudaGetLastError()));
            return -1;
        }
    }
    return (int64_t)n;
}

extern "C" int elp_debug_set_reference_chunk(elp_ctx* c, uint64_t bytes) {
    if (!c) return ELP_EINVAL;
    if (bytes > (1ull << 32)) return c->fail(E_INVAL, "elp_debug_set_reference_chunk: %llu bytes (at most 2^32)", (unsigned long long)bytes);
    c->ref_chunk = bytes;
    return ELP_OK;
}
