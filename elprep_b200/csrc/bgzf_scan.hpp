// bgzf_scan.hpp -- block boundaries of a BGZF byte run (utils/bgzf/bgzf-files.go:95-127): gzip member header with FEXTRA, subfield
// 'B','C',2 giving the block size, CRC32 + ISIZE trailer.  Shared by the host inflate (bgzf.cpp) and the device inflate (bgzf_inflate.cu).
#pragma once
#include <cstdint>
#include <vector>
#include "../../include/elprep_b200.h"

constexpr int BGZF_TRL = 8;

inline uint32_t rd16(const uint8_t* p) { return (uint32_t)p[0] | ((uint32_t)p[1] << 8); }
inline uint32_t rd32(const uint8_t* p) { return (uint32_t)p[0] | ((uint32_t)p[1] << 8) | ((uint32_t)p[2] << 16) | ((uint32_t)p[3] << 24); }

struct BgzfBlock { uint64_t in_off, cdata_off, cdata_len, out_off; uint32_t isize, crc; };

// Appends the blocks of d[0, n) to `blocks` (out_off continues from *total, which receives the sum of ISIZE).  Without `consumed` the
// run must be whole blocks.  With it, the scan stops before an incomplete trailing block (one that more bytes could still complete)
// and *consumed receives the bytes of the whole blocks; at most max_blocks are taken.  ELP_EBGZF for anything malformed.
inline int scan_blocks(const uint8_t* d, uint64_t n, std::vector<BgzfBlock>& blocks, uint64_t* total, uint64_t* consumed = nullptr, size_t max_blocks = SIZE_MAX) {
    constexpr uint64_t HDR = 18;
    uint64_t x = 0, out = *total;
    size_t taken = 0;
    while (x < n && taken < max_blocks) {
        if (n - x < HDR + BGZF_TRL) { if (consumed) break; return ELP_EBGZF; }
        const uint8_t* h = d + x;
        if (h[0] != 31 || h[1] != 139 || h[2] != 8 || !(h[3] & 4)) return ELP_EBGZF;
        const uint32_t xlen = rd16(h + 10);
        if (n - x < 12ull + xlen + BGZF_TRL) { if (consumed) break; return ELP_EBGZF; }
        uint32_t bsize = 0; bool found = false;
        for (uint32_t i = 0; i + 4 <= xlen;) {
            const uint8_t* e = h + 12 + i; const uint32_t slen = rd16(e + 2);
            if (e[0] == 66 && e[1] == 67 && slen == 2 && i + 6 <= xlen) { bsize = rd16(e + 4) + 1; found = true; break; }
            i += 4 + slen;
        }
        if (!found) return ELP_EBGZF;                                  // "missing BC extra subfield in BGZF header"
        if (bsize < 12 + xlen + BGZF_TRL) return ELP_EBGZF;
        if (x + bsize > n) { if (consumed) break; return ELP_EBGZF; }
        BgzfBlock b; b.in_off = x; b.cdata_off = x + 12 + xlen; b.cdata_len = bsize - 12 - xlen - BGZF_TRL;
        b.crc = rd32(d + x + bsize - 8); b.isize = rd32(d + x + bsize - 4); b.out_off = out;
        if (b.isize > 65536) return ELP_EBGZF;
        out += b.isize; x += bsize;
        blocks.push_back(b);
        taken++;
    }
    *total = out;
    if (consumed) *consumed = x;
    return ELP_OK;
}
