// gofloat.hpp -- strconv.AppendFloat(b, float64(v), 'g', -1, 32) of Go's standard library for a float32 v: the text FormatAlignment
// writes for an f field and every B:f element (formatSamTag, sam/sam-files.go:485-546).  Host code, header-only.
//
// Go's 'g' with shortest precision (strconv/ftoa.go): take the shortest decimal d1...dn that reads back as the same float32 (several
// of that length: the one closest to the exact value), with value = 0.d1...dn x 10^dp; print the %e form when dp - 1 < -4 or
// dp - 1 >= 6 (eprec is 6 for shortest), else the %f form; no trailing zeros either way.  NaN -> "NaN", infinities -> "+Inf" / "-Inf",
// zero -> "0" or "-0".  std::to_chars(float) in scientific form without a precision yields exactly that digit string (shortest
// round trip, closest to the value); only the layout is Go's.
#pragma once
#include <charconv>
#include <cstdint>
#include <cstring>

namespace gofloat {

constexpr int MAX_LEN = 16;   // longest text: "-0.000123456789" style %f forms are 15 bytes, "-1.1754944e-38" 14

// writes the text of the float32 with these bits to out (MAX_LEN bytes of room) and returns its length
inline int format_f32(uint32_t bits, char* out) {
    const bool neg = (bits >> 31) != 0;
    const uint32_t mag = bits & 0x7fffffffu;
    if (mag > 0x7f800000u) { std::memcpy(out, "NaN", 3); return 3; }
    if (mag == 0x7f800000u) { std::memcpy(out, neg ? "-Inf" : "+Inf", 4); return 4; }
    int n = 0;
    if (neg) out[n++] = '-';
    if (mag == 0) { out[n++] = '0'; return n; }
    float f;
    std::memcpy(&f, &mag, 4);
    char sci[32];
    const char* end = std::to_chars(sci, sci + sizeof sci, f, std::chars_format::scientific).ptr;   // d[.ddd]e(+|-)XX
    char dig[12];
    int nd = 0;
    const char* p = sci;
    for (; p < end && *p != 'e'; p++) if (*p != '.') dig[nd++] = *p;
    const bool eneg = p + 1 < end && p[1] == '-';
    int x = 0;                                                           // decimal exponent of d1.d2...dn = dp - 1
    for (const char* q = p + 2; q < end; q++) x = x * 10 + (*q - '0');
    if (eneg) x = -x;
    if (x < -4 || x >= 6) {                                              // %e: d1[.d2...dn]e(+|-)XX, at least two exponent digits
        out[n++] = dig[0];
        if (nd > 1) { out[n++] = '.'; for (int i = 1; i < nd; i++) out[n++] = dig[i]; }
        out[n++] = 'e';
        out[n++] = x < 0 ? '-' : '+';
        const int a = x < 0 ? -x : x;                                    // float32: |x| <= 45
        out[n++] = (char)('0' + a / 10);
        out[n++] = (char)('0' + a % 10);
        return n;
    }
    const int dp = x + 1;                                                // %f: integer part zero-padded, "0." and zeros below 1
    if (dp > 0) for (int i = 0; i < dp; i++) out[n++] = i < nd ? dig[i] : '0';
    else out[n++] = '0';
    if (nd > dp) {
        out[n++] = '.';
        for (int i = dp; i < nd; i++) out[n++] = i < 0 ? '0' : dig[i];
    }
    return n;
}

}  // namespace gofloat
