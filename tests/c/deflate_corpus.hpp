// deflate_corpus.hpp -- the DEFLATE encoder's corpus: inputs of at most 65535 bytes, as named cases.  Shared by deflate_check.cpp
// (deflate.cuh as a team of one lane against zlib and inflate.cuh, and the dump the device test reads) and team_check.cpp (deflate.cuh as
// host teams of many lanes against the team of one).
//
// for_each_input(emit) calls emit(kind, name, bytes) once per input, always in the same order with the same bytes:
//   BASE  empty, 1 and 0xff00 bytes, BAM-like records, random bytes, runs, period-k data, distances of exactly 32768 and 32769, literal-only
//         input, a single literal value, Fibonacci histograms, mixtures
//   TEAM_EDGE  inputs at the edges of the team: n in {1, 2, 3, 31, 32, 33, 255..259, 511..513, 0xff00 - 1, 0xff00} (a chain chunk is 32
//         positions, a parse segment of 0xff00 bytes is 255 at 256 lanes) as runs, periods 1-8 and random bytes; 258-byte matches that start
//         at every offset mod 255, so each crosses a segment boundary; and positions whose different 3-byte strings collide in hash3
#pragma once
#include <algorithm>
#include <random>
#include <string>
#include <vector>
#include "corpus_data.hpp"
#include "deflate.cuh"

namespace corpus {

enum DefKind : uint8_t { BASE = 0, TEAM_EDGE = 1 };

// literals only: no 3-byte string occurs twice (a de Bruijn-like walk over distinct triples)
inline Bytes no_repeats(std::mt19937_64& rng, size_t n) {
    Bytes v;
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
inline Bytes fibonacci(std::mt19937_64& rng, size_t n, int nsym) {
    std::vector<uint64_t> f(nsym); f[0] = 1; f[1] = 1;
    for (int s = 2; s < nsym; s++) f[s] = f[s - 1] + f[s - 2];
    Bytes v;
    for (int s = nsym - 1; s >= 0 && v.size() < n; s--) for (uint64_t k = 0; k < f[s] && v.size() < n; k++) v.push_back((uint8_t)(s * 7 + 1));
    for (int s = 0; s < nsym; s++) v.push_back((uint8_t)(s * 7 + 1));   // every symbol at least once
    v.resize(std::min(v.size(), n));
    std::shuffle(v.begin(), v.end(), rng);                              // (scattered: literals, not one long match)
    return v;
}

// every input of the corpus, drawing the data from rng (the TEAM_EDGE inputs draw from their own generator, so adding them changed nothing the
// caller draws from rng afterwards)
template <class F>
void for_each_input(std::mt19937_64& rng, F&& emit) {
    auto base = [&](const std::string& name, const Bytes& d) { emit(BASE, name, d); };
    base("empty", {});
    base("one byte", {0x42});
    base("two bytes", {0x42, 0x42});
    base("three equal bytes", {7, 7, 7});
    base("bam 0xff00", bam_like(rng, 0xff00));
    base("bam 65535", bam_like(rng, 65535));
    for (size_t n : {1, 5, 100, 1000, 4097, 30000}) base("bam " + std::to_string(n), bam_like(rng, n));
    base("random 0xff00", random_bytes(rng, 0xff00));
    base("random 65535", random_bytes(rng, 65535));
    for (size_t n : {1, 2, 3, 10, 300}) base("random " + std::to_string(n), random_bytes(rng, n));
    base("run 0xff00", Bytes(0xff00, 'A'));
    base("run 259", Bytes(259, 0));
    base("run 65535", Bytes(65535, 0xff));
    for (int k = 1; k <= 40; k++) base("period " + std::to_string(k), periodic(rng, 4000 + 37 * k, k));
    for (int k : {255, 256, 257, 258, 259, 1000, 4095, 4096, 4097, 32767, 32768}) base("period " + std::to_string(k), periodic(rng, 0xff00, k));
    {   // matches at distance exactly 32768, and one byte too far
        auto a = random_bytes(rng, 32768); auto b = a; b.insert(b.end(), a.begin(), a.begin() + 0xff00 - 32768); base("distance 32768", b);
        auto c = random_bytes(rng, 32769); auto e = c; e.insert(e.end(), c.begin(), c.begin() + 0xff00 - 32769); base("distance 32769", e);
    }
    base("literals only", no_repeats(rng, 0xff00));
    {   // a single literal value, scattered among random bytes and alone
        auto v = random_bytes(rng, 20000); for (size_t i = 0; i < v.size(); i += 2) v[i] = 'Q'; base("one literal value in random", v);
        Bytes w(2, 'Z'); base("one literal value, 2 bytes", w);
    }
    for (int nsym : {20, 24, 27}) base("fibonacci " + std::to_string(nsym), fibonacci(rng, 0xff00, nsym));
    base("fibonacci short", fibonacci(rng, 4000, 18));
    for (int t = 0; t < 60; t++) {                                    // mixtures: BAM-like records with random and repeated stretches
        auto v = bam_like(rng, rng() % 0xff01);
        for (int k = 0; k < 4 && !v.empty(); k++) {
            const size_t a = rng() % v.size(), l = std::min<size_t>(v.size() - a, rng() % 3000);
            const int kind = (int)(rng() % 3);
            for (size_t i = 0; i < l; i++) v[a + i] = kind == 0 ? (uint8_t)rng() : kind == 1 ? (uint8_t)'N' : v[a + (i % 7)];
        }
        base("mixture " + std::to_string(t), v);
    }
    // ---- team edges ----
    auto edge = [&](const std::string& name, const Bytes& d) { emit(TEAM_EDGE, name, d); };
    std::mt19937_64 erng(20261018);
    for (size_t n : {1, 2, 3, 31, 32, 33, 255, 256, 257, 258, 259, 511, 512, 513, 0xff00 - 1, 0xff00}) {
        const std::string at = " n " + std::to_string(n);
        edge("edge run" + at, Bytes(n, 'C'));
        for (int k = 1; k <= 8; k++) edge("edge period " + std::to_string(k) + at, periodic(erng, n, k));
        edge("edge random" + at, random_bytes(erng, n));
    }
    // 258-byte matches at distance 200 starting at 255 k + r: input j puts one in every third segment k = 3 m + 1 with r = 3 m + j, so the
    // three inputs start one at every r in 0..254.  At r >= 252 the match covers all of segment k + 1, whose parse entry lies past its end.
    for (int j = 0; j < 3; j++) {
        Bytes v = random_bytes(erng, 0xff00);
        for (uint32_t m = 0; m < 85; m++) {
            const uint32_t p = 255 * (3 * m + 1) + 3 * m + (uint32_t)j;
            if (p + dfl::MAX_MATCH + 1 > v.size()) break;
            v[p - 1] = (uint8_t)(v[p - 1 - 200] ^ 0x55);                // the match starts at p, not before
            for (uint32_t i = 0; i < dfl::MAX_MATCH; i++) v[p + i] = v[p + i - 200];
        }
        edge("edge 258-byte matches at segment offsets " + std::to_string(j) + " mod 3", v);
    }
    {   // 96 different 3-byte strings of one hash3 bucket: positions 3 apart share a chain chunk and a hash but not their bytes
        Bytes t;
        const uint8_t seed[3] = {'h', 'a', 's'};
        const uint32_t h = dfl::hash3(seed);
        for (uint32_t k = 0; t.size() < 3 * 96; k++) {
            const uint8_t s[3] = {(uint8_t)k, (uint8_t)(k >> 8), (uint8_t)(k >> 16)};
            if (dfl::hash3(s) == h) t.insert(t.end(), s, s + 3);
        }
        Bytes v;
        while (v.size() < 0xff00) {                                     // the strings in random order, now and then a random byte between
            const size_t i = erng() % 96;
            v.insert(v.end(), t.begin() + 3 * i, t.begin() + 3 * i + 3);
            if (erng() % 4 == 0) v.push_back((uint8_t)erng());
        }
        v.resize(0xff00);
        edge("edge hash3 collisions", v);
        v.resize(3 * 96);
        for (size_t i = 0; i < 3 * 96; i++) v[i] = t[i];
        edge("edge hash3 collisions, each once", v);
    }
}

}  // namespace corpus
