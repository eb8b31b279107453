// elprep::ParseHeaderLineFromString (include/elprep_b200.hpp) over the cases of tests/test_replace_read_group_cpu.py: one case per input
// line, hex-encoded; per case one output line, "ok" followed by " <tag hex>=<value hex>" in tag order, or "panic <message hex>".
#include <cstdio>
#include <iostream>
#include <string>

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

int main() {
    std::string ln;
    while (std::getline(std::cin, ln)) {
        try {
            const auto rec = elprep::ParseHeaderLineFromString(unhex(ln));
            std::string out = "ok";
            for (const auto& kv : rec) out += " " + hex(kv.first) + "=" + hex(kv.second);
            std::printf("%s\n", out.c_str());
        } catch (const elprep::Panic& p) {
            std::printf("panic %s\n", hex(p.what()).c_str());
        }
    }
    return 0;
}
