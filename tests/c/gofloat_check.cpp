// Host client of elprep_b200/csrc/gofloat.hpp for tests/test_sam_format.py: reads little-endian float32 bit patterns from the file
// argv[1] and prints gofloat::format_f32 of each, one per line.
#include <cstdio>
#include <vector>
#include "gofloat.hpp"

int main(int argc, char** argv) {
    if (argc != 2) return 2;
    FILE* f = std::fopen(argv[1], "rb");
    if (!f) return 2;
    std::vector<uint32_t> bits;
    uint32_t b;
    while (std::fread(&b, 4, 1, f) == 1) bits.push_back(b);
    std::fclose(f);
    char out[gofloat::MAX_LEN + 1];
    for (uint32_t v : bits) {
        const int n = gofloat::format_f32(v, out);
        out[n] = '\n';
        std::fwrite(out, 1, n + 1, stdout);
    }
    return 0;
}
