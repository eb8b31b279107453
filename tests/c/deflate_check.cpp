// CPU check of the device DEFLATE encoder: elprep_b200/csrc/deflate.cuh, compiled here as host C++ (a team of one lane), over the corpus of
// deflate_corpus.hpp.  Every stream it writes must inflate back to its input with zlib (inflateInit2(-15) + inflate(Z_FINISH): Z_STREAM_END
// with exactly the input's length) and with the project's own decoder (inflate.cuh), every Huffman code it emits must be complete, and every
// stream must fit the stored bound.
// Built with -fsanitize=address,undefined: input and output are heap buffers of exactly the sizes the encoder may touch.
//
//   deflate_check                      the corpus; prints OK
//   deflate_check deflate IN OUT EOF   IN as BGZF (0xff00-byte blocks, the framing of elp_fetch_bgzf; EOF 1: with the EOF marker) into OUT
//   deflate_check size IN              the bytes of the raw DEFLATE streams of IN's 0xff00-byte blocks
//   deflate_check dump DIR             every input of the corpus (deflate_corpus.hpp) as DIR/NNNN.bin, and DIR/names.txt: "NNNN.bin<TAB>name"
//                                      per line; the device test sends them through the device encoder
#include <zlib.h>
#include <algorithm>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <random>
#include <string>
#include <vector>
#include "deflate.cuh"
#include "deflate_corpus.hpp"

static int n_streams = 0, n_stored = 0, failures = 0;
static std::mt19937_64 rng(20261017);
static dfl::EncShared S;
static std::vector<uint16_t> prev_(65536);
static std::vector<uint32_t> match_(65536);

// the encoder's stream of d (n <= 65535), from buffers of exactly the size it may touch
static std::vector<uint8_t> encode(const std::vector<uint8_t>& d) {
    uint8_t* ib = (uint8_t*)std::malloc(d.size() ? d.size() : 1);
    if (!d.empty()) std::memcpy(ib, d.data(), d.size());
    const size_t words = (dfl::stored_bytes((uint32_t)d.size()) + 3) / 4;
    uint32_t* ob = (uint32_t*)std::malloc(words * 4);
    std::memset(ob, 0xa5, words * 4);                                  // (the encoder must not rely on a zeroed buffer)
    const uint32_t n = dfl::deflate_block(dfl::SerialEnc{}, S, dfl::EncScratch{prev_.data(), match_.data()}, ib, (uint32_t)d.size(), ob);
    std::vector<uint8_t> out(reinterpret_cast<uint8_t*>(ob), reinterpret_cast<uint8_t*>(ob) + n);
    std::free(ib); std::free(ob);
    return out;
}

// Kraft sum of a code in units of 2^-15: complete iff it is exactly 2^15
static uint32_t kraft(const uint8_t* len, int n) { uint32_t k = 0; for (int s = 0; s < n; s++) if (len[s]) k += 1u << (15 - len[s]); return k; }

static void check(const std::string& what, const std::vector<uint8_t>& d) {
    n_streams++;
    const std::vector<uint8_t> z = encode(d);
    auto fail = [&](const char* why) { if (failures < 20) std::printf("FAIL %s (n %zu, %zu bytes out): %s\n", what.c_str(), d.size(), z.size(), why); failures++; };
    if (z.size() > dfl::stored_bytes((uint32_t)d.size())) fail("larger than the stored block");
    if (18 + z.size() + 8 > 65536 && d.size() <= 0xff00) fail("BGZF block over 65536 bytes");
    const bool stored = !z.empty() && (z[0] & 7) == 1;
    n_stored += stored;
    if (!stored) {
        if ((z[0] & 7) != 5) fail("neither a final dynamic nor a final stored block");
        const uint32_t one = 1u << 15;
        for (int s = 0; s < dfl::NLIT; s++) if (S.llen[s] > 15) fail("literal/length code over 15 bits");
        for (int s = 0; s < dfl::NDIST; s++) if (S.dlen[s] > 15) fail("distance code over 15 bits");
        for (int s = 0; s < dfl::NCL; s++) if (S.clen[s] > 7) fail("code-length code over 7 bits");
        if (kraft(S.llen, dfl::NLIT) != one) fail("incomplete literal/length code");
        if (kraft(S.dlen, dfl::NDIST) != one) fail("incomplete distance code");
        if (kraft(S.clen, dfl::NCL) != one) fail("incomplete code-length code");
    }
    // zlib
    std::vector<uint8_t> zo(d.size() + 1);
    z_stream zs; std::memset(&zs, 0, sizeof zs);
    inflateInit2(&zs, -15);
    zs.next_in = const_cast<Bytef*>(z.data()); zs.avail_in = (uInt)z.size();
    zs.next_out = zo.data(); zs.avail_out = (uInt)d.size();
    const int r = inflate(&zs, Z_FINISH);
    const bool zok = r == Z_STREAM_END && zs.total_out == d.size() && zs.avail_in == 0 && (d.empty() || std::memcmp(zo.data(), d.data(), d.size()) == 0);
    inflateEnd(&zs);
    if (!zok) fail("zlib does not inflate it back");
    // the project's decoder
    static dfl::Tables T;
    uint8_t* ib = (uint8_t*)std::malloc(z.size());
    uint8_t* ob = (uint8_t*)std::malloc(d.size() ? d.size() : 1);
    std::memcpy(ib, z.data(), z.size());
    const uint32_t st = dfl::inflate_stream(dfl::Serial{}, T, ib, (uint32_t)z.size(), ob, (uint32_t)d.size());
    if (st != dfl::OK || (d.size() && std::memcmp(ob, d.data(), d.size()) != 0)) fail("inflate.cuh does not inflate it back");
    std::free(ib); std::free(ob);
}

// ---- BGZF framing, as bgzf_deflate.cu frames its blocks ----
static const uint8_t BGZF_HDR[18] = {0x1f, 0x8b, 0x08, 0x04, 0, 0, 0, 0, 0x00, 0xff, 0x06, 0x00, 0x42, 0x43, 0x02, 0x00, 0, 0};
static const uint8_t BGZF_EOF[28] = {0x1f, 0x8b, 0x08, 0x04, 0, 0, 0, 0, 0x00, 0xff, 0x06, 0x00, 0x42, 0x43, 0x02, 0x00, 0x1b, 0x00, 0x03, 0x00, 0, 0, 0, 0, 0, 0, 0, 0};
static void put32(std::vector<uint8_t>& v, uint32_t x) { for (int k = 0; k < 4; k++) v.push_back((uint8_t)(x >> (8 * k))); }

static std::vector<uint8_t> read_file(const char* path) {
    FILE* f = std::fopen(path, "rb");
    if (!f) { std::perror(path); std::exit(2); }
    std::vector<uint8_t> v;
    uint8_t buf[1 << 16]; size_t k;
    while ((k = std::fread(buf, 1, sizeof buf, f)) > 0) v.insert(v.end(), buf, buf + k);
    std::fclose(f);
    return v;
}

static void write_file(const char* path, const std::vector<uint8_t>& v) {
    FILE* f = std::fopen(path, "wb");
    if (!f || (!v.empty() && std::fwrite(v.data(), 1, v.size(), f) != v.size()) || std::fclose(f) != 0) { std::perror(path); std::exit(2); }
}

int main(int argc, char** argv) {
    if (argc == 5 && !std::strcmp(argv[1], "deflate")) {
        const auto d = read_file(argv[2]);
        std::vector<uint8_t> out;
        for (size_t off = 0; off < d.size(); off += 0xff00) {
            const std::vector<uint8_t> blk(d.begin() + off, d.begin() + std::min(d.size(), off + 0xff00));
            const auto z = encode(blk);
            const size_t at = out.size();
            out.insert(out.end(), BGZF_HDR, BGZF_HDR + 18);
            const uint32_t bsize = (uint32_t)(18 + z.size() + 8);
            out[at + 16] = (uint8_t)(bsize - 1); out[at + 17] = (uint8_t)((bsize - 1) >> 8);
            out.insert(out.end(), z.begin(), z.end());
            put32(out, (uint32_t)crc32(0, blk.data(), (uInt)blk.size()));
            put32(out, (uint32_t)blk.size());
        }
        if (std::atoi(argv[4])) out.insert(out.end(), BGZF_EOF, BGZF_EOF + 28);
        write_file(argv[3], out);
        return 0;
    }
    if (argc == 3 && !std::strcmp(argv[1], "size")) {
        const auto d = read_file(argv[2]);
        uint64_t total = 0;
        for (size_t off = 0; off < d.size(); off += 0xff00) {
            const std::vector<uint8_t> blk(d.begin() + off, d.begin() + std::min(d.size(), off + 0xff00));
            const auto z = encode(blk);
            check("sample block " + std::to_string(off / 0xff00), blk);
            total += z.size();
        }
        std::printf("%llu\n", (unsigned long long)total);
        return failures ? 1 : 0;
    }
    if (argc == 3 && !std::strcmp(argv[1], "dump")) {
        std::string names;
        int k = 0;
        corpus::for_each_input(rng, [&](corpus::DefKind, const std::string& name, const std::vector<uint8_t>& d) {
            char file[32]; std::snprintf(file, sizeof file, "%04d.bin", k++);
            write_file((std::string(argv[2]) + "/" + file).c_str(), d);
            names += std::string(file) + "\t" + name + "\n";
        });
        write_file((std::string(argv[2]) + "/names.txt").c_str(), std::vector<uint8_t>(names.begin(), names.end()));
        std::printf("%d inputs dumped\n", k);
        return 0;
    }
    corpus::for_each_input(rng, [](corpus::DefKind, const std::string& name, const std::vector<uint8_t>& d) { check(name, d); });
    {   // the random blocks must take the stored path
        for (size_t n : {(size_t)0xff00, (size_t)65535}) {
            const auto z = encode(corpus::random_bytes(rng, n));
            if ((z[0] & 7) != 1 || z.size() != n + 5) { std::printf("FAIL random %zu: not stored\n", n); failures++; }
        }
    }
    {   // the length limit on its own: Fibonacci frequencies (an unlimited code needs nsym - 1 bits), and codes of 0 to 2 symbols
        for (int limit : {7, 15})
            for (int nsym : {2, 3, 10, 16, 17, 19, 25, 30, 44}) {
                if (limit == 7 && nsym > 19) continue;
                for (int shape = 0; shape < 4; shape++) {
                    uint32_t freq[dfl::NLIT] = {0};
                    uint8_t len[dfl::NLIT];
                    uint32_t a = 1, b = 1;
                    for (int s = 0; s < nsym; s++) {
                        const int at = shape == 1 ? nsym - 1 - s : shape == 2 ? (s * 7) % dfl::NLIT : s;
                        freq[at] = shape == 3 ? (s < 2 ? 0u : 5u) : a;
                        const uint32_t c = a + b; a = b; b = c;
                    }
                    const int n = limit == 7 ? dfl::NCL : dfl::NLIT;
                    dfl::build_lengths(dfl::SerialEnc{}, S.u.h, freq, n, limit, len);
                    uint32_t k = 0; int used = 0, bad = 0;
                    for (int s = 0; s < n; s++) { if (len[s]) { k += 1u << (15 - len[s]); used++; } bad += len[s] > limit || (freq[s] && !len[s]); }
                    if (k != (1u << 15) || bad || used < 2) { std::printf("FAIL lengths limit %d nsym %d shape %d: kraft %u, %d bad\n", limit, nsym, shape, k, bad); failures++; }
                }
            }
        for (int m = 0; m < 2; m++) {                                   // no symbol, one symbol (each position): two codes of length 1
            for (int only = 0; only < (m ? dfl::NDIST : 1); only++) {
                uint32_t freq[dfl::NDIST] = {0};
                uint8_t len[dfl::NDIST];
                if (m) freq[only] = 9;
                dfl::build_lengths(dfl::SerialEnc{}, S.u.h, freq, dfl::NDIST, 15, len);
                int ones = 0, other = 0;
                for (int s = 0; s < dfl::NDIST; s++) { ones += len[s] == 1; other += len[s] > 1; }
                if (ones != 2 || other || (m && len[only] != 1)) { std::printf("FAIL padding m %d only %d\n", m, only); failures++; }
            }
        }
    }
    {   // a long run is matches of length 258 at distance 1
        const auto z = encode(std::vector<uint8_t>(0xff00, 'A'));
        if (z.size() > 400) { std::printf("FAIL run: %zu bytes\n", z.size()); failures++; }
    }
    std::printf("%d streams (%d stored), %d failures\n", n_streams, n_stored, failures);
    if (failures) return 1;
    std::printf("OK\n");
    return 0;
}
