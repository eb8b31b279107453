// corpus_data.hpp -- the byte generators shared by the DEFLATE decoder and encoder corpora (inflate_corpus.hpp, deflate_corpus.hpp).
// Every generator draws from the caller's generator, so a corpus is the same sequence of bytes on every run.
#pragma once
#include <cstdint>
#include <cstdio>
#include <random>
#include <vector>

namespace corpus {

using Bytes = std::vector<uint8_t>;

inline Bytes random_bytes(std::mt19937_64& rng, size_t n) { Bytes v(n); for (auto& b : v) b = (uint8_t)rng(); return v; }
inline Bytes run_of(size_t n, uint8_t c) { return Bytes(n, c); }
inline Bytes periodic(std::mt19937_64& rng, size_t n, int k) { auto p = random_bytes(rng, k); Bytes v(n); for (size_t i = 0; i < n; i++) v[i] = p[i % k]; return v; }
// BAM-like records: fixed fields, a QNAME, CIGAR, SEQ nibbles, QUAL, a few tags
inline Bytes bam_like(std::mt19937_64& rng, size_t n) {
    Bytes v;
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

}  // namespace corpus
