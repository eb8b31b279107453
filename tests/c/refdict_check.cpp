// elprep::RenameChromosomes and elprep::ReplaceReferenceSequenceDictionary (include/elprep_b200.hpp) on the header cases of
// tests/test_reference_dictionary_cpu.py.  One case per input line, five tab-separated fields: SO, mode bits (1 rename, 2 replace), the old
// @SQ names, the new dictionary's names (names hex-encoded, comma-separated).  Per case one output line: the SO after the filters, a tab,
// and the @SQ names after them, in the same encoding.
#include <cstdio>
#include <iostream>
#include <sstream>
#include <string>
#include <vector>

#include "elprep_b200.hpp"

static std::string hex(const std::string& s) {
    static const char d[] = "0123456789abcdef";
    std::string o;
    for (unsigned char c : s) { o += d[c >> 4]; o += d[c & 15]; }
    return o;
}

static std::string unhex(const std::string& h) {
    std::string o;
    for (size_t i = 0; i + 1 < h.size(); i += 2) o += (char)std::stoi(h.substr(i, 2), nullptr, 16);
    return o;
}

static std::vector<elprep::Header::SQ> names(const std::string& field) {
    std::vector<elprep::Header::SQ> v;
    if (field.empty()) return v;
    std::stringstream ss(field);
    std::string item;
    while (std::getline(ss, item, ',')) v.push_back({unhex(item), 1});
    return v;
}

int main() {
    std::string ln;
    while (std::getline(std::cin, ln)) {
        std::vector<std::string> f;
        std::stringstream ss(ln);
        std::string item;
        while (std::getline(ss, item, '\t')) f.push_back(item);
        while (f.size() < 4) f.push_back("");
        elprep::Header h;
        h.SO = unhex(f[0]);
        h.sq = names(f[2]);
        const int mode = std::stoi(f[1]);
        if (mode & 1) { const elprep::RenameChromosomes r(h); (void)r; }
        if (mode & 2) { const elprep::ReplaceReferenceSequenceDictionary d(h, names(f[3])); (void)d; }
        std::string out = hex(h.SO) + "\t";
        for (size_t i = 0; i < h.sq.size(); i++) out += (i ? "," : "") + hex(h.sq[i].SN);
        std::printf("%s\n", out.c_str());
    }
    return 0;
}
