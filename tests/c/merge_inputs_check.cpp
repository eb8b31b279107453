// elprep::MergeInputs (include/elprep_b200.hpp) on the cases of tests/test_merge_inputs_cpu.py.  One case per input line: the suffix, then
// one field per input header, tab-separated.  A header field is "sq;rg;pg": comma-separated entries, each a hex-encoded SN (sq), ID:PP
// (rg, PP "-" for none) or ID (pg).  Per case one output line: "PANIC <hex message>", or the merged sq, rg and pg in the same encoding,
// the @SQ maps ("|"-separated inputs of comma-separated indices) and the RG and PG maps (comma-separated old:new), tab-separated.
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
static std::vector<std::string> split(const std::string& s, char c) {
    std::vector<std::string> v;
    if (s.empty()) return v;
    std::stringstream ss(s);
    std::string item;
    while (std::getline(ss, item, c)) v.push_back(item);
    if (s.back() == c) v.push_back("");
    return v;
}

int main() {
    std::string ln;
    while (std::getline(std::cin, ln)) {
        const std::vector<std::string> f = split(ln, '\t');
        std::vector<elprep::HeaderLines> hs;
        for (size_t k = 1; k < f.size(); k++) {
            std::vector<std::string> p = split(f[k], ';');
            while (p.size() < 3) p.push_back("");
            elprep::HeaderLines h;
            for (auto& e : split(p[0], ',')) h.SQ.push_back({{"SN", unhex(e)}, {"LN", "1"}});
            for (auto& e : split(p[1], ',')) {
                const size_t c = e.find(':');
                elprep::HeaderLines::Record r{{"ID", unhex(e.substr(0, c))}};
                if (e.substr(c + 1) != "-") r["PP"] = unhex(e.substr(c + 1));
                h.RG.push_back(r);
            }
            for (auto& e : split(p[2], ',')) h.PG.push_back({{"ID", unhex(e)}});
            hs.push_back(h);
        }
        try {
            const elprep::MergedInputs m = elprep::MergeInputs(hs, unhex(f[0]));
            std::string o;
            for (size_t i = 0; i < m.header.SQ.size(); i++) o += (i ? "," : "") + hex(m.header.SQ[i].at("SN"));
            o += "\t";
            for (size_t i = 0; i < m.header.RG.size(); i++) {
                auto pp = m.header.RG[i].find("PP");
                o += (i ? "," : "") + hex(m.header.RG[i].at("ID")) + ":" + (pp == m.header.RG[i].end() ? std::string("-") : hex(pp->second));
            }
            o += "\t";
            for (size_t i = 0; i < m.header.PG.size(); i++) o += (i ? "," : "") + hex(m.header.PG[i].at("ID"));
            o += "\t";
            for (size_t k = 0; k < m.sqMaps.size(); k++) {
                o += k ? "|" : "";
                for (size_t i = 0; i < m.sqMaps[k].size(); i++) o += (i ? "," : "") + std::to_string(m.sqMaps[k][i]);
            }
            for (const auto* mp : {&m.rgMap, &m.pgMap}) {
                o += "\t";
                bool first = true;
                for (auto& kv : *mp) { o += (first ? "" : ",") + hex(kv.first) + ":" + hex(kv.second); first = false; }
            }
            std::printf("%s\n", o.c_str());
        } catch (const elprep::Panic& e) {
            std::printf("PANIC %s\n", hex(e.what()).c_str());
        }
    }
    return 0;
}
