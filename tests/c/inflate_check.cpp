// CPU check of the device DEFLATE decoder: elprep_b200/csrc/inflate.cuh, compiled here as host C++ (a team of one lane), against zlib
// stream by stream, over the corpus of inflate_corpus.hpp.  For every stream: the same accept / reject decision as inflateInit2(-15) +
// inflate(Z_FINISH) into exactly ISIZE bytes (what elp_bgzf_inflate accepts), and the same bytes on accept.  Built with
// -fsanitize=address,undefined: input and output are heap buffers of exactly n_in and ISIZE bytes, so any read or write out of bounds stops
// the run.
//
//   inflate_check             the corpus and the per-lane CRC-32 fold; prints the counts and OK
//   inflate_check dump FILE   the same checks, and writes to FILE every ZLIB, CRAFTED and EDGE stream and every 4th MUTATED one as records
//                             of: u8 kind, u16 name length, name, u32 isize, u32 status of the team of one, u8 1 if zlib accepts, u32 stream
//                             length, stream bytes (little-endian); the device test sends them through the device decoder
#include <zlib.h>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <random>
#include <string>
#include <vector>
#include "inflate.cuh"
#include "inflate_corpus.hpp"

static int n_streams = 0, n_accept = 0, n_reject = 0, failures = 0;
static std::mt19937_64 rng(12345);

static bool zlib_inflate(const std::vector<uint8_t>& in, uint32_t isize, std::vector<uint8_t>& out) {
    out.assign(isize, 0);
    z_stream zs; std::memset(&zs, 0, sizeof zs);
    if (inflateInit2(&zs, -15) != Z_OK) return false;
    uint8_t dummy = 0;
    zs.next_in = const_cast<Bytef*>(in.empty() ? &dummy : in.data()); zs.avail_in = (uInt)in.size();
    zs.next_out = isize ? out.data() : &dummy; zs.avail_out = isize;
    const int r = inflate(&zs, Z_FINISH);
    const bool ok = r == Z_STREAM_END && zs.total_out == isize;
    inflateEnd(&zs);
    return ok;
}

// the decoder's status on one stream; *zok: zlib's verdict
static uint32_t check(const std::string& what, const std::vector<uint8_t>& in, uint32_t isize, bool* zok_out) {
    n_streams++;
    std::vector<uint8_t> zout;
    const bool zok = zlib_inflate(in, isize, zout);
    uint8_t* ib = (uint8_t*)std::malloc(in.size() ? in.size() : 1);          // exact sizes: ASan catches any overrun
    uint8_t* ob = (uint8_t*)std::malloc(isize ? isize : 1);
    if (!in.empty()) std::memcpy(ib, in.data(), in.size());
    static dfl::Tables T;
    const uint32_t st = dfl::inflate_stream(dfl::Serial{}, T, ib, (uint32_t)in.size(), ob, isize);
    const bool ok = st == dfl::OK;
    if (ok != zok || (ok && isize && std::memcmp(ob, zout.data(), isize) != 0)) {
        if (failures < 20) std::printf("MISMATCH %s: n_in %zu isize %u zlib %s decoder %s (%s)\n", what.c_str(), in.size(), isize, zok ? "accepts" : "rejects",
                                       ok ? "accepts" : "rejects", dfl::status_text(st));
        failures++;
    }
    (ok ? n_accept : n_reject)++;
    std::free(ib); std::free(ob);
    *zok_out = zok;
    return st;
}

static void put(FILE* f, uint64_t v, int bytes) { for (int k = 0; k < bytes; k++) std::fputc((int)(v >> (8 * k)) & 255, f); }

int main(int argc, char** argv) {
    FILE* dump = nullptr;
    if (argc == 3 && !std::strcmp(argv[1], "dump")) {
        dump = std::fopen(argv[2], "wb");
        if (!dump) { std::perror(argv[2]); return 2; }
    } else if (argc != 1) {
        std::fprintf(stderr, "usage: inflate_check [dump FILE]\n");
        return 2;
    }
    int n_mutated = 0, n_dumped = 0;
    corpus::for_each_stream(rng, [&](corpus::InfKind kind, const std::string& name, const std::vector<uint8_t>& in, uint32_t isize) {
        bool zok = false;
        const uint32_t st = check(name, in, isize, &zok);
        if (!dump || (kind == corpus::MUTATED && n_mutated++ % 4)) return;
        put(dump, kind, 1); put(dump, name.size(), 2); std::fwrite(name.data(), 1, name.size(), dump);
        put(dump, isize, 4); put(dump, st, 4); put(dump, zok, 1); put(dump, in.size(), 4);
        if (!in.empty()) std::fwrite(in.data(), 1, in.size(), dump);
        n_dumped++;
    });
    // ---- CRC-32: per-lane chunks folded with the shift table, as bgzf_crc does, against zlib ----
    {
        uint32_t tab[256], x2n[32];
        for (uint32_t i = 0; i < 256; i++) tab[i] = dfl::crc_table_entry(i);
        dfl::x2n_table(x2n);
        auto fold = [&](const std::vector<uint8_t>& d) {
            const size_t n = d.size();
            const uint32_t want = (uint32_t)crc32(0, d.data(), (uInt)n);
            const size_t chunk = (n + 31) / 32;
            uint32_t got = 0;
            for (size_t lane = 0; lane < 32; lane++) {
                const size_t a = std::min(n, lane * chunk), b = std::min(n, a + chunk);
                got ^= dfl::crc_shift(x2n, dfl::crc_bytes(tab, 0, d.data() + a, (uint32_t)(b - a)), n - b);
            }
            if (got != want) { if (failures < 20) std::printf("MISMATCH crc n %zu: %08x vs %08x\n", n, got, want); failures++; }
        };
        for (int t = 0; t < 200; t++) fold(corpus::random_bytes(rng, t < 4 ? (size_t)t : (size_t)(rng() % 65537)));
        for (size_t n = 4; n <= 64; n++) fold(corpus::random_bytes(rng, n));      // lanes left empty by chunk = (n + 31) / 32
        for (size_t n : {1023, 1024, 1025}) fold(corpus::random_bytes(rng, n));
    }
    if (dump && std::fclose(dump) != 0) { std::perror(argv[2]); return 2; }
    std::printf("%d streams (%d accepted, %d rejected), %d mismatches\n", n_streams, n_accept, n_reject, failures);
    if (dump) std::printf("%d streams dumped\n", n_dumped);
    if (failures) return 1;
    std::printf("OK\n");
    return 0;
}
