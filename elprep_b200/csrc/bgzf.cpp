// bgzf.cpp -- BGZF (de)compression on a host thread pool and the BAM file header walk (SURVEY.md §8f row 2; replaces
// utils/bgzf/bgzf-files.go:95-127 (reader), :324-431 (writer) and the header part of sam/bam-files.go for callers that hold a
// whole BAM file or a run of BGZF blocks in memory).  Host code, no CUDA: BGZF blocks are independent gzip members
// (<= 64 KiB, "BC" extra subfield with the block size, CRC32 + ISIZE trailer), so a first pass finds the block boundaries and
// the output offsets (prefix sum of ISIZE) and a pool of threads inflates / deflates blocks independently with zlib.
// The output of elp_bgzf_inflate, after elp_bam_header_size bytes, is what elp_append_bam takes; elp_fetch_bam output goes
// through elp_bgzf_deflate.  Deflate output is a valid BGZF stream but not byte-identical to Go's compress/flate (different
// encoder); input blocks are 0xff00 bytes (the htslib convention) rather than the reference's 65536, so that incompressible
// data still fits the 16-bit block size.
#include <zlib.h>
#include <atomic>
#include <cstdint>
#include <cstring>
#include <thread>
#include <vector>
#include "../../include/elprep_b200.h"
#include "pool.hpp"

namespace {

constexpr uint64_t BGZF_IN = 0xff00;          // uncompressed bytes per block written
constexpr int BGZF_HDR = 18, BGZF_TRL = 8;

inline uint32_t rd16(const uint8_t* p) { return (uint32_t)p[0] | ((uint32_t)p[1] << 8); }
inline uint32_t rd32(const uint8_t* p) { return (uint32_t)p[0] | ((uint32_t)p[1] << 8) | ((uint32_t)p[2] << 16) | ((uint32_t)p[3] << 24); }
inline void wr16(uint8_t* p, uint32_t v) { p[0] = v & 255; p[1] = (v >> 8) & 255; }
inline void wr32(uint8_t* p, uint32_t v) { p[0] = v & 255; p[1] = (v >> 8) & 255; p[2] = (v >> 16) & 255; p[3] = v >> 24; }

struct Block { uint64_t in_off, cdata_off, cdata_len, out_off; uint32_t isize, crc; };

// block boundaries of a BGZF byte run (utils/bgzf/bgzf-files.go:95-127): gzip member header with FEXTRA, subfield 'B','C',2
int scan_blocks(const uint8_t* d, uint64_t n, std::vector<Block>& blocks, uint64_t* total) {
    uint64_t x = 0, out = 0;
    while (x < n) {
        if (n - x < (uint64_t)BGZF_HDR + BGZF_TRL) return ELP_EBGZF;
        const uint8_t* h = d + x;
        if (h[0] != 31 || h[1] != 139 || h[2] != 8 || !(h[3] & 4)) return ELP_EBGZF;
        const uint32_t xlen = rd16(h + 10);
        if (n - x < 12ull + xlen + BGZF_TRL) return ELP_EBGZF;
        uint32_t bsize = 0; bool found = false;
        for (uint32_t i = 0; i + 4 <= xlen;) {
            const uint8_t* e = h + 12 + i; const uint32_t slen = rd16(e + 2);
            if (e[0] == 66 && e[1] == 67 && slen == 2 && i + 6 <= xlen) { bsize = rd16(e + 4) + 1; found = true; break; }
            i += 4 + slen;
        }
        if (!found) return ELP_EBGZF;                                  // "missing BC extra subfield in BGZF header"
        if (bsize < 12 + xlen + BGZF_TRL || x + bsize > n) return ELP_EBGZF;
        Block b; b.in_off = x; b.cdata_off = x + 12 + xlen; b.cdata_len = bsize - 12 - xlen - BGZF_TRL;
        b.crc = rd32(d + x + bsize - 8); b.isize = rd32(d + x + bsize - 4); b.out_off = out;
        if (b.isize > 65536) return ELP_EBGZF;
        out += b.isize; x += bsize;
        blocks.push_back(b);
    }
    *total = out;
    return ELP_OK;
}

}  // namespace

extern "C" {

int64_t elp_bgzf_inflate_bound(const uint8_t* data, uint64_t n) {
    if (!data && n) return ELP_EINVAL;
    std::vector<Block> blocks; uint64_t total = 0;
    const int rc = scan_blocks(data, n, blocks, &total);
    return rc ? rc : (int64_t)total;
}

int elp_bgzf_inflate(const uint8_t* data, uint64_t n, uint8_t* out, uint64_t capacity, uint64_t* out_n, int n_threads) {
    if ((!data && n) || !out_n) return ELP_EINVAL;
    std::vector<Block> blocks; uint64_t total = 0;
    int rc = scan_blocks(data, n, blocks, &total);
    if (rc) return rc;
    if (total > capacity || (!out && total)) return ELP_EINVAL;
    std::atomic<int> err{0};
    pool_for(blocks.size(), n_threads, [&](size_t i) {
        const Block& b = blocks[i];
        if (b.isize == 0) { if (b.crc != 0) err = 1; return; }
        z_stream zs; std::memset(&zs, 0, sizeof zs);
        if (inflateInit2(&zs, -15) != Z_OK) { err = 1; return; }
        zs.next_in = const_cast<Bytef*>(data + b.cdata_off); zs.avail_in = (uInt)b.cdata_len;
        zs.next_out = out + b.out_off; zs.avail_out = b.isize;
        const int r = inflate(&zs, Z_FINISH);
        const bool ok = r == Z_STREAM_END && zs.total_out == b.isize;
        inflateEnd(&zs);
        if (!ok || (uint32_t)crc32(crc32(0L, Z_NULL, 0), out + b.out_off, b.isize) != b.crc) err = 1;
    });
    if (err) return ELP_EBGZF;
    *out_n = total;
    return ELP_OK;
}

uint64_t elp_bgzf_deflate_bound(uint64_t n) {
    const uint64_t nb = (n + BGZF_IN - 1) / BGZF_IN;
    return nb * (BGZF_IN + 5 + 64 + BGZF_HDR + BGZF_TRL) + 28;
}

int elp_bgzf_deflate(const uint8_t* data, uint64_t n, uint8_t* out, uint64_t capacity, uint64_t* out_n, int level, int n_threads, int write_eof) {
    if ((!data && n) || !out || !out_n) return ELP_EINVAL;
    if (capacity < elp_bgzf_deflate_bound(n)) return ELP_EINVAL;
    const size_t nb = (size_t)((n + BGZF_IN - 1) / BGZF_IN);
    const uint64_t slot = BGZF_IN + 5 + 64 + BGZF_HDR + BGZF_TRL;       // every block is compressed into its own slot, then compacted
    std::vector<uint32_t> sizes(nb);
    std::atomic<int> err{0};
    pool_for(nb, n_threads, [&](size_t i) {
        const uint64_t off = (uint64_t)i * BGZF_IN, len = std::min<uint64_t>(BGZF_IN, n - off);
        uint8_t* o = out + (uint64_t)i * slot;
        static const uint8_t hdr[BGZF_HDR] = {0x1f, 0x8b, 0x08, 0x04, 0, 0, 0, 0, 0x00, 0xff, 0x06, 0x00, 0x42, 0x43, 0x02, 0x00, 0, 0};   // bgzf-files.go:336-340
        std::memcpy(o, hdr, BGZF_HDR);
        uint32_t clen = 0;
        for (int attempt = 0; attempt < 2; attempt++) {                  // second attempt: stored blocks (incompressible input)
            z_stream zs; std::memset(&zs, 0, sizeof zs);
            if (deflateInit2(&zs, attempt ? 0 : level, Z_DEFLATED, -15, 8, Z_DEFAULT_STRATEGY) != Z_OK) { err = 1; return; }
            zs.next_in = const_cast<Bytef*>(data + off); zs.avail_in = (uInt)len;
            zs.next_out = o + BGZF_HDR; zs.avail_out = (uInt)(slot - BGZF_HDR - BGZF_TRL);
            const int r = deflate(&zs, Z_FINISH);
            clen = (uint32_t)zs.total_out;
            deflateEnd(&zs);
            if (r == Z_STREAM_END && BGZF_HDR + clen + BGZF_TRL <= 65536) break;
            if (attempt) { err = 1; return; }
        }
        wr32(o + BGZF_HDR + clen, (uint32_t)crc32(crc32(0L, Z_NULL, 0), data + off, (uInt)len));
        wr32(o + BGZF_HDR + clen + 4, (uint32_t)len);
        sizes[i] = BGZF_HDR + clen + BGZF_TRL;
        wr16(o + 16, sizes[i] - 1);
    });
    if (err) return ELP_EBGZF;
    uint64_t w = 0;
    for (size_t i = 0; i < nb; i++) { if (w != (uint64_t)i * slot) std::memmove(out + w, out + (uint64_t)i * slot, sizes[i]); w += sizes[i]; }
    if (write_eof) {
        static const uint8_t eof[28] = {0x1f, 0x8b, 0x08, 0x04, 0, 0, 0, 0, 0x00, 0xff, 0x06, 0x00, 0x42, 0x43, 0x02, 0x00, 0x1b, 0x00, 0x03, 0x00, 0, 0, 0, 0, 0, 0, 0, 0};
        std::memcpy(out + w, eof, 28); w += 28;
    }
    *out_n = w;
    return ELP_OK;
}

// bytes of the BAM header: magic, l_text, text, n_ref, {l_name, name, l_ref}* (sam/bam-files.go ParseHeader); -1 if malformed / truncated.
// n_ref_out (may be NULL) receives the number of reference sequences: BAM refIDs index them in this order.
int64_t elp_bam_header_size(const uint8_t* bam, uint64_t n, int32_t* n_ref_out) {
    if (!bam || n < 12 || std::memcmp(bam, "BAM\1", 4) != 0) return -1;
    const int32_t l_text = (int32_t)rd32(bam + 4);
    if (l_text < 0 || 8ull + (uint64_t)l_text + 4 > n) return -1;
    uint64_t x = 8ull + (uint64_t)l_text;
    const int32_t n_ref = (int32_t)rd32(bam + x); x += 4;
    if (n_ref < 0) return -1;
    for (int32_t r = 0; r < n_ref; r++) {
        if (x + 4 > n) return -1;
        const int32_t l_name = (int32_t)rd32(bam + x);
        if (l_name < 0 || x + 4 + (uint64_t)l_name + 4 > n) return -1;
        x += 4 + (uint64_t)l_name + 4;
    }
    if (n_ref_out) *n_ref_out = n_ref;
    return (int64_t)x;
}

}  // extern "C"
