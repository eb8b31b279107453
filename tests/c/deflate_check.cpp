// CPU check of the device DEFLATE encoder: elprep_b200/csrc/deflate.cuh, compiled here as host C++ (a team of one lane).  Every stream it
// writes must inflate back to its input with zlib (inflateInit2(-15) + inflate(Z_FINISH): Z_STREAM_END with exactly the input's length) and
// with the project's own decoder (inflate.cuh), every Huffman code it emits must be complete, and every stream must fit the stored bound.
// Built with -fsanitize=address,undefined: input and output are heap buffers of exactly the sizes the encoder may touch.
//
//   deflate_check                      the corpus; prints OK
//   deflate_check deflate IN OUT EOF   IN as BGZF (0xff00-byte blocks, the framing of elp_fetch_bgzf; EOF 1: with the EOF marker) into OUT
//   deflate_check size IN              the bytes of the raw DEFLATE streams of IN's 0xff00-byte blocks
#include <zlib.h>
#include <algorithm>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <random>
#include <string>
#include <vector>
#include "deflate.cuh"

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

// ---- data ----
static std::vector<uint8_t> random_bytes(size_t n) { std::vector<uint8_t> v(n); for (auto& b : v) b = (uint8_t)rng(); return v; }
static std::vector<uint8_t> periodic(size_t n, int k) { auto p = random_bytes(k); std::vector<uint8_t> v(n); for (size_t i = 0; i < n; i++) v[i] = p[i % k]; return v; }
static std::vector<uint8_t> bam_like(size_t n) {
    std::vector<uint8_t> v;
    int i = 0;
    while (v.size() < n) {
        char name[64]; const int ln = std::snprintf(name, sizeof name, "HWI-ST1234:8:1101:%d:%d", 1000 + (int)(rng() % 20000), i++);
        const int lseq = 100 + (int)(rng() % 51);
        const int bs = 32 + ln + 1 + 4 + (lseq + 1) / 2 + lseq + 7;
        auto put32 = [&](uint32_t x) { for (int k = 0; k < 4; k++) v.push_back((uint8_t)(x >> (8 * k))); };
        put32(bs); put32(rng() % 3); put32((uint32_t)(rng() % 1000000)); v.push_back((uint8_t)(ln + 1)); v.push_back(60); v.push_back(0); v.push_back(0);
        v.push_back(1); v.push_back(0); v.push_back(99); v.push_back(0); put32(lseq); put32(0); put32((uint32_t)(rng() % 1000000)); put32(300);
        v.insert(v.end(), name, name + ln); v.push_back(0);
        put32((uint32_t)lseq << 4);
        for (int k = 0; k < (lseq + 1) / 2; k++) v.push_back((uint8_t)(0x11 << (rng() % 4)));
        for (int k = 0; k < lseq; k++) v.push_back((uint8_t)(30 + rng() % 12));
        v.push_back('R'); v.push_back('G'); v.push_back('Z'); v.push_back('r'); v.push_back('g'); v.push_back('1'); v.push_back(0);
    }
    v.resize(n);
    return v;
}
// literals only: no 3-byte string occurs twice (a de Bruijn-like walk over distinct triples)
static std::vector<uint8_t> no_repeats(size_t n) {
    std::vector<uint8_t> v;
    std::vector<uint8_t> seen(1 << 24, 0);
    v.push_back(0); v.push_back(0);
    while (v.size() < n) {
        const size_t m = v.size();
        int b = -1;
        for (int t = 0; t < 256 && b < 0; t++) {
            const int c = (int)((rng() + t) & 255);
            const uint32_t k = (uint32_t)v[m - 2] | (uint32_t)v[m - 1] << 8 | (uint32_t)c << 16;
            if (!seen[k]) { seen[k] = 1; b = c; }
        }
        if (b < 0) break;
        v.push_back((uint8_t)b);
    }
    v.resize(std::min(v.size(), n));
    return v;
}
// Fibonacci symbol frequencies: an unlimited Huffman code would need far more than 15 bits
static std::vector<uint8_t> fibonacci(size_t n, int nsym) {
    std::vector<uint64_t> f(nsym); f[0] = 1; f[1] = 1;
    for (int s = 2; s < nsym; s++) f[s] = f[s - 1] + f[s - 2];
    std::vector<uint8_t> v;
    for (int s = nsym - 1; s >= 0 && v.size() < n; s--) for (uint64_t k = 0; k < f[s] && v.size() < n; k++) v.push_back((uint8_t)(s * 7 + 1));
    for (int s = 0; s < nsym; s++) v.push_back((uint8_t)(s * 7 + 1));   // every symbol at least once
    v.resize(std::min(v.size(), n));
    std::shuffle(v.begin(), v.end(), rng);                              // (scattered: literals, not one long match)
    return v;
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
        FILE* f = std::fopen(argv[3], "wb");
        if (!f || std::fwrite(out.data(), 1, out.size(), f) != out.size()) { std::perror(argv[3]); return 2; }
        std::fclose(f);
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
    std::vector<std::pair<std::string, std::vector<uint8_t>>> data;
    data.push_back({"empty", {}});
    data.push_back({"one byte", {0x42}});
    data.push_back({"two bytes", {0x42, 0x42}});
    data.push_back({"three equal bytes", {7, 7, 7}});
    data.push_back({"bam 0xff00", bam_like(0xff00)});
    data.push_back({"bam 65535", bam_like(65535)});
    for (size_t n : {1, 5, 100, 1000, 4097, 30000}) data.push_back({"bam " + std::to_string(n), bam_like(n)});
    data.push_back({"random 0xff00", random_bytes(0xff00)});
    data.push_back({"random 65535", random_bytes(65535)});
    for (size_t n : {1, 2, 3, 10, 300}) data.push_back({"random " + std::to_string(n), random_bytes(n)});
    data.push_back({"run 0xff00", std::vector<uint8_t>(0xff00, 'A')});
    data.push_back({"run 259", std::vector<uint8_t>(259, 0)});
    data.push_back({"run 65535", std::vector<uint8_t>(65535, 0xff)});
    for (int k = 1; k <= 40; k++) data.push_back({"period " + std::to_string(k), periodic(4000 + 37 * k, k)});
    for (int k : {255, 256, 257, 258, 259, 1000, 4095, 4096, 4097, 32767, 32768}) data.push_back({"period " + std::to_string(k), periodic(0xff00, k)});
    {   // matches at distance exactly 32768, and one byte too far
        auto a = random_bytes(32768); auto b = a; b.insert(b.end(), a.begin(), a.begin() + 0xff00 - 32768); data.push_back({"distance 32768", b});
        auto c = random_bytes(32769); auto e = c; e.insert(e.end(), c.begin(), c.begin() + 0xff00 - 32769); data.push_back({"distance 32769", e});
    }
    data.push_back({"literals only", no_repeats(0xff00)});
    {   // a single literal value, scattered among random bytes and alone
        auto v = random_bytes(20000); for (size_t i = 0; i < v.size(); i += 2) v[i] = 'Q'; data.push_back({"one literal value in random", v});
        std::vector<uint8_t> w(2, 'Z'); data.push_back({"one literal value, 2 bytes", w});
    }
    for (int nsym : {20, 24, 27}) data.push_back({"fibonacci " + std::to_string(nsym), fibonacci(0xff00, nsym)});
    data.push_back({"fibonacci short", fibonacci(4000, 18)});
    for (int t = 0; t < 60; t++) {                                    // mixtures: BAM-like records with random and repeated stretches
        auto v = bam_like(rng() % 0xff01);
        for (int k = 0; k < 4 && !v.empty(); k++) {
            const size_t a = rng() % v.size(), l = std::min<size_t>(v.size() - a, rng() % 3000);
            const int kind = (int)(rng() % 3);
            for (size_t i = 0; i < l; i++) v[a + i] = kind == 0 ? (uint8_t)rng() : kind == 1 ? (uint8_t)'N' : v[a + (i % 7)];
        }
        data.push_back({"mixture " + std::to_string(t), v});
    }
    for (auto& [name, d] : data) check(name, d);
    {   // the random blocks must take the stored path
        for (size_t n : {(size_t)0xff00, (size_t)65535}) {
            const auto z = encode(random_bytes(n));
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
