// inflate_corpus.hpp -- the DEFLATE decoder's corpus: raw streams with the ISIZE they are decoded into, as named cases.  Shared by
// inflate_check.cpp (inflate.cuh as a team of one lane against zlib, and the dump the device test reads) and team_check.cpp (inflate.cuh as
// host teams of many lanes against the team of one).
//
// for_each_stream(emit) calls emit(kind, name, stream, isize) once per stream, always in the same order with the same bytes:
//   ZLIB     zlib's streams: levels 0-9 and its strategies over BAM-like records, random bytes, runs, period-k data, distances up to 32768,
//            sync and full flushes (many blocks per member), and ISIZE one off either way
//   MUTATED  those streams with bit flips, truncations and flips in the header region
//   CRAFTED  hand-built invalid streams: every rejection of the decoder's header comment
//   EDGE     zlib streams of 2..64 and 1023..1025 bytes: the lengths where the CRC-32 lane slices of warp_crc leave lanes empty
#pragma once
#include <zlib.h>
#include <algorithm>
#include <cstring>
#include <random>
#include <string>
#include <vector>
#include "corpus_data.hpp"

namespace corpus {

enum InfKind : uint8_t { ZLIB = 0, MUTATED = 1, CRAFTED = 2, EDGE = 3 };

inline Bytes zdeflate(const Bytes& d, int level, int strategy, int flush_every = 0, int flush_kind = Z_SYNC_FLUSH) {
    z_stream zs; std::memset(&zs, 0, sizeof zs);
    deflateInit2(&zs, level, Z_DEFLATED, -15, 8, strategy);
    Bytes out(deflateBound(&zs, d.size()) + 64 + (flush_every ? 16 * (d.size() / flush_every + 2) : 0));
    uint8_t dummy = 0;
    zs.next_out = out.data(); zs.avail_out = (uInt)out.size();
    size_t x = 0;
    do {
        const size_t step = flush_every ? std::min<size_t>(flush_every, d.size() - x) : d.size() - x;
        zs.next_in = const_cast<Bytef*>(d.empty() ? &dummy : d.data() + x); zs.avail_in = (uInt)step;
        x += step;
        deflate(&zs, x == d.size() ? Z_FINISH : flush_kind);
    } while (x < d.size());
    out.resize(zs.total_out);
    deflateEnd(&zs);
    return out;
}

// ---- hand-built streams ----
struct BitWriter {
    Bytes v; uint64_t acc = 0; int n = 0;
    void put(uint32_t x, int k) { acc |= (uint64_t)x << n; n += k; while (n >= 8) { v.push_back((uint8_t)acc); acc >>= 8; n -= 8; } }
    void put_rev(uint32_t code, int len) { uint32_t r = 0; for (int i = 0; i < len; i++) r |= ((code >> i) & 1u) << (len - 1 - i); put(r, len); }   // Huffman codes go MSB first
    Bytes done() { if (n) { v.push_back((uint8_t)acc); acc = 0; n = 0; } return v; }
};
// fixed-code symbol (RFC 1951 3.2.6)
inline void fixed_sym(BitWriter& w, int s) {
    if (s < 144) w.put_rev(0x30 + s, 8); else if (s < 256) w.put_rev(0x190 + s - 144, 9); else if (s < 280) w.put_rev(s - 256, 7); else w.put_rev(0xc0 + s - 280, 8);
}
// a dynamic block header: HLIT, HDIST, HCLEN, the code-length code lengths in transmission order, then raw (bits, count) pairs
inline Bytes dynamic_header(int hlit, int hdist, int hclen, const std::vector<int>& clens_in_order, const std::vector<std::pair<int, int>>& syms) {
    BitWriter w;
    w.put(1, 1); w.put(2, 2); w.put(hlit - 257, 5); w.put(hdist - 1, 5); w.put(hclen - 4, 4);
    for (int i = 0; i < hclen; i++) w.put(clens_in_order[i], 3);
    for (auto& s : syms) w.put(s.first, s.second);
    for (int i = 0; i < 64; i++) w.put(0, 8);
    return w.done();
}

template <class F>
void crafted(F&& check) {
    const int order[19] = {16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15};
    {   // block type 3
        BitWriter w; w.put(1, 1); w.put(3, 2); w.put(0, 16); check("btype 3", w.done(), 0); check("btype 3 isize 1", BitWriter{}.done(), 1);
    }
    {   // HLIT > 286, HDIST > 30
        std::vector<int> cl(19, 4);
        check("hlit 287", dynamic_header(287, 1, 19, cl, {}), 10);
        check("hlit 288", dynamic_header(288, 1, 19, cl, {}), 10);
        check("hdist 31", dynamic_header(257, 31, 19, cl, {}), 10);
        check("hdist 32", dynamic_header(257, 32, 19, cl, {}), 10);
    }
    {   // code-length code: over-subscribed, incomplete, empty
        std::vector<int> over(19, 1); check("clen over-subscribed", dynamic_header(257, 1, 19, over, {}), 10);
        std::vector<int> inc(19, 0); inc[0] = 2; check("clen incomplete", dynamic_header(257, 1, 19, inc, {}), 10);
        std::vector<int> one(19, 0); one[3] = 1; check("clen single code", dynamic_header(257, 1, 19, one, {}), 10);
        std::vector<int> none(19, 0); check("clen empty", dynamic_header(257, 1, 4, none, {}), 10);
    }
    {   // code-length code with lengths: symbols 0..15 -> 5 bits (16 codes), 16, 17, 18 -> 5 bits: 19 codes of length 5 = incomplete; use
        // 18 of length 5 ... easier: all 19 symbols with lengths making a complete code: 13 of length 4 ... take 16 symbols of length 4
        // (0..15) -- complete -- plus none for 16..18; then "repeat first" needs symbol 16, so: 0..14 length 4 (15 codes) + 16 length 5 + 17 length 5
        std::vector<int> L(19, 0);
        for (int s = 0; s < 15; s++) L[s] = 4;
        L[16] = 5; L[17] = 5;
        std::vector<int> inorder(19); for (int i = 0; i < 19; i++) inorder[i] = L[order[i]];
        // canonical codes: length 4: symbols 0..14 -> codes 0..14; length 5: first = (15) << 1 = 30: 16 -> 30, 17 -> 31
        auto sym = [&](int s) -> std::pair<int, int> { uint32_t code = s < 15 ? (uint32_t)s : (s == 16 ? 30u : 31u); int len = s < 15 ? 4 : 5;
                                                        uint32_t r = 0; for (int i = 0; i < len; i++) r |= ((code >> i) & 1u) << (len - 1 - i); return {(int)r, len}; };
        check("repeat 16 first", dynamic_header(257, 1, 19, inorder, {sym(16), {0, 2}}), 10);
        std::vector<std::pair<int, int>> lots;                 // 17 with 7 repeats (3 bits = 7 -> 10 zeros) x 40 = 400 > 258: repeat past the end
        for (int i = 0; i < 40; i++) { lots.push_back(sym(17)); lots.push_back({7, 3}); }
        check("repeat past end", dynamic_header(257, 1, 19, inorder, lots), 10);
        // all 258 lengths zero: no end-of-block code
        std::vector<std::pair<int, int>> zeros;
        for (int i = 0; i < 25; i++) { zeros.push_back(sym(17)); zeros.push_back({7, 3}); }   // 250 zeros
        for (int i = 0; i < 8; i++) zeros.push_back(sym(0));
        check("no end-of-block", dynamic_header(257, 1, 19, inorder, zeros), 10);
        // literal/length set over-subscribed: 258 lengths of 1
        std::vector<std::pair<int, int>> ones;
        for (int i = 0; i < 258; i++) ones.push_back(sym(1));
        check("lit over-subscribed", dynamic_header(257, 1, 19, inorder, ones), 10);
        // literal/length set incomplete: only 256 with length 2, 'A' with length 2
        std::vector<std::pair<int, int>> inc;
        for (int i = 0; i < 258; i++) inc.push_back(sym(i == 65 || i == 256 ? 2 : 0));
        check("lit incomplete", dynamic_header(257, 1, 19, inorder, inc), 1);
        // a lone code of length 1 (EOB only), distances empty: complete enough for zlib; an empty block
        std::vector<std::pair<int, int>> lone;
        for (int i = 0; i < 258; i++) lone.push_back(sym(i == 256 ? 1 : 0));
        {
            BitWriter w; w.put(1, 1); w.put(2, 2); w.put(0, 5); w.put(0, 5); w.put(15, 4);
            for (int i = 0; i < 19; i++) w.put(inorder[i], 3);
            for (auto& s : lone) w.put(s.first, s.second);
            w.put(0, 1);                                       // EOB = code 0 of length 1
            check("lone code EOB", w.done(), 0);
            BitWriter w2 = BitWriter{}; w2.put(1, 1); w2.put(2, 2); w2.put(0, 5); w2.put(0, 5); w2.put(15, 4);
            for (int i = 0; i < 19; i++) w2.put(inorder[i], 3);
            for (auto& s : lone) w2.put(s.first, s.second);
            w2.put(1, 1);                                      // the unused code of a lone-code set
            check("lone code unused half", w2.done(), 0);
        }
    }
    {   // fixed code: literal/length symbols 286 and 287, distance codes 30 and 31, distance past the block start
        for (int s : {286, 287}) { BitWriter w; w.put(1, 1); w.put(1, 2); fixed_sym(w, 'a'); fixed_sym(w, 'a'); fixed_sym(w, 'a'); fixed_sym(w, s); w.put(0, 5); fixed_sym(w, 256); check("fixed lit 286/287", w.done(), 6); }
        for (int d : {30, 31}) { BitWriter w; w.put(1, 1); w.put(1, 2); fixed_sym(w, 'a'); fixed_sym(w, 257); w.put_rev(d, 5); fixed_sym(w, 256); check("fixed dist 30/31", w.done(), 4); }
        for (int d : {0, 1, 2, 3}) {                           // distance d + 1 after 2 literals: 1 and 2 are fine, 3 and 4 are too far
            BitWriter w; w.put(1, 1); w.put(1, 2); fixed_sym(w, 'a'); fixed_sym(w, 'b'); fixed_sym(w, 257); w.put_rev(d, 5); fixed_sym(w, 256);
            check("fixed distance vs start", w.done(), 5);
        }
        {   // a non-final empty fixed block, then a final stored block
            BitWriter w; w.put(0, 1); w.put(1, 2); fixed_sym(w, 256); w.put(1, 1); w.put(0, 2); auto v = w.done();
            v.push_back(3); v.push_back(0); v.push_back(0xfc); v.push_back(0xff); v.push_back('x'); v.push_back('y'); v.push_back('z');
            check("fixed then stored", v, 3);
            auto bad = v; bad[bad.size() - 4] ^= 1; check("stored nlen", bad, 3);
            auto tr = v; tr.pop_back(); check("stored truncated", tr, 3);
            auto extra = v; extra.push_back(0x55); extra.push_back(0xaa); check("trailing bytes after final block", extra, 3);
        }
    }
}

// every stream of the corpus, drawing the data from rng (the EDGE streams draw from their own generator, so adding them changed nothing
// the caller draws from rng afterwards)
template <class F>
void for_each_stream(std::mt19937_64& rng, F&& emit) {
    auto zlib = [&](const std::string& name, const Bytes& z, uint32_t isize) { emit(ZLIB, name, z, isize); };
    // ---- streams from zlib ----
    const int strategies[] = {Z_DEFAULT_STRATEGY, Z_FILTERED, Z_HUFFMAN_ONLY, Z_RLE, Z_FIXED};
    std::vector<std::pair<std::string, Bytes>> data;
    data.push_back({"bam", bam_like(rng, 0xff00)});
    data.push_back({"bam 65536", bam_like(rng, 65536)});
    data.push_back({"random", random_bytes(rng, 0xff00)});
    data.push_back({"run", run_of(65536, 'A')});
    data.push_back({"empty", {}});
    data.push_back({"one", {0x42}});
    for (int k = 1; k <= 40; k++) data.push_back({"period " + std::to_string(k), periodic(rng, 4000 + 37 * k, k)});
    {   // distances up to 32768: a random 32 KiB prefix repeated
        auto a = random_bytes(rng, 32768); auto b = a; b.insert(b.end(), a.begin(), a.begin() + 32768); data.push_back({"far", b});
        auto c = random_bytes(rng, 30000); Bytes d(65536); for (size_t i = 0; i < d.size(); i++) d[i] = c[i % c.size()]; data.push_back({"period 30000", d});
    }
    for (auto& [name, d] : data) {
        for (int level = 0; level <= 9; level++)
            for (int st : strategies) {
                if ((level == 0 || level == 6 || level == 1 || level == 9) || st == Z_DEFAULT_STRATEGY || d.size() < 8000) {
                    auto z = zdeflate(d, level, st);
                    zlib(name + " level " + std::to_string(level), z, (uint32_t)d.size());
                }
            }
        // many small blocks per member: sync and full flushes (empty stored blocks between them)
        zlib(name + " sync flush", zdeflate(d, 6, Z_DEFAULT_STRATEGY, 997, Z_SYNC_FLUSH), (uint32_t)d.size());
        zlib(name + " full flush", zdeflate(d, 1, Z_DEFAULT_STRATEGY, 4096, Z_FULL_FLUSH), (uint32_t)d.size());
        zlib(name + " stored sync flush", zdeflate(d, 0, Z_DEFAULT_STRATEGY, 100, Z_SYNC_FLUSH), (uint32_t)d.size());
        // output longer / shorter than ISIZE
        if (!d.empty()) { auto z = zdeflate(d, 6, Z_DEFAULT_STRATEGY); zlib("isize - 1", z, (uint32_t)d.size() - 1); zlib("isize + 1", z, (uint32_t)d.size() + 1); }
    }
    zlib("isize 0xff00", zdeflate(bam_like(rng, 0xff00), 6, Z_DEFAULT_STRATEGY), 0xff00);
    // ---- mutated streams: bit flips and truncations ----
    for (auto& [name, d] : data) {
        if (d.size() < 16) continue;
        for (int level : {1, 6, 9}) {
            for (int st : {Z_DEFAULT_STRATEGY, Z_FIXED, Z_HUFFMAN_ONLY}) {
                const auto z = zdeflate(d, level, st);
                for (int t = 0; t < (name.rfind("period", 0) == 0 ? 3 : 40); t++) {
                    auto m = z;
                    const int flips = 1 + (int)(rng() % 3);
                    for (int f = 0; f < flips; f++) { const size_t bit = rng() % (m.size() * 8); m[bit / 8] ^= (uint8_t)(1u << (bit % 8)); }
                    emit(MUTATED, name + " flipped", m, (uint32_t)d.size());
                    auto head = z; head.resize(rng() % z.size());
                    emit(MUTATED, name + " truncated", head, (uint32_t)d.size());
                    auto early = z; early[rng() % std::min<size_t>(early.size(), 64)] ^= (uint8_t)(1u << (rng() % 8));   // the header region
                    emit(MUTATED, name + " header flip", early, (uint32_t)d.size());
                }
            }
        }
    }
    crafted([&](const char* name, const Bytes& s, uint32_t isize) { emit(CRAFTED, std::string(name), s, isize); });
    // ---- team edges: short streams and the CRC-32 lane-slice edges (chunk = (n + 31) / 32 leaves the last lanes empty) ----
    std::mt19937_64 erng(20261018);
    std::vector<size_t> sizes;
    for (size_t n = 2; n <= 64; n++) sizes.push_back(n);
    for (size_t n : {1023, 1024, 1025}) sizes.push_back(n);
    for (size_t n : sizes) {
        emit(EDGE, "edge random " + std::to_string(n), zdeflate(random_bytes(erng, n), 6, Z_DEFAULT_STRATEGY), (uint32_t)n);
        emit(EDGE, "edge period 3 " + std::to_string(n), zdeflate(periodic(erng, n, 3), 9, Z_DEFAULT_STRATEGY), (uint32_t)n);   // (overlapping copies)
    }
}

}  // namespace corpus
