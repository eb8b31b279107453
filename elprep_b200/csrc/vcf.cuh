// vcf.cuh -- VCF known sites (elp_load_known_sites): the header on the host, the data lines in the vcf_parse kernel.
//
// The reference converts a VCF with intervals.FromVcfFile (intervals/intervals.go:306-338): vcf.ParseHeader and NewVariantParser
// (vcf/vcf-files.go:73-305,749-765), then ParseVariant with NSamples = 0 (:600-738,773-782, string-scanner.go) on every line, and the
// interval [Pos, Pos - 1 + len(Ref)] (Variant.End, vcf-types.go:147-161).
//   vcf_header      host: ParseHeader and the parser checks of NewVariantParser, one declaration at a time; the declared INFO IDs with
//                   their type and number go to the device
//   vcf_parse       one warp per 32 consecutive lines.  The warp walks each line in 32-byte windows and ballots the tabs of CHROM .. FILTER
//                   and the first ' ', ':' or tab of INFO, so no thread walks a long line alone; then each lane takes one line and checks
//                   its fields (POS, QUAL, FILTER, INFO keys, CHROM) from those positions
//   go_float        strconv.ParseFloat(s, 64): the syntax (atof.go special, readFloat, underscoreOK) and the decimal or binary exponent of the
//                   value; the narrow band of exponents next to the overflow bound is decided on the host with strtod
#pragma once
#include <cerrno>
#include <cmath>
#include <cstdlib>
#include <cstring>
#include <string>
#include <vector>
#include "ctx.h"
#include "text_parse.cuh"

namespace {

constexpr uint64_t VCF_MAX_LINE = 65536;          // bufio.MaxScanTokenSize: a longer data line stops the reference's scanner
const char VCF_PREFIX[] = "##fileformat=VCFv4.";  // fileFormatVersionLinePrefix (vcf-types.go:32)
constexpr uint64_t VCF_PREFIX_LEN = sizeof(VCF_PREFIX) - 1;

// why a data line is refused: the first failure in ParseVariant's field order, then End(), then the .elsites round trip
enum VcfErr : uint32_t { VL_LONG = 1, VL_TAB, VL_POS, VL_QUAL, VL_QUAL_RANGE, VL_INFO, VL_END, VL_CHROM };
inline const char* vcf_err_text(uint32_t e) {
    switch (e) {
        case VL_LONG: return "line of 65536 bytes or more (bufio.Scanner: token too long)";
        case VL_TAB: return "missing tabulator in VCF data line";
        case VL_POS: return "POS: strconv.ParseInt(s, 10, 32) fails";
        case VL_QUAL: return "QUAL: strconv.ParseFloat(s, 64) fails (syntax)";
        case VL_QUAL_RANGE: return "QUAL: strconv.ParseFloat(s, 64) fails (value out of range)";
        case VL_INFO: return "INFO: a declared key's value fails its parser";
        case VL_END: return "INFO: END key (Variant.End panics on every value type it can have)";
        case VL_CHROM: return "empty CHROM (vcf-to-elsites writes a line its .elsites loader refuses)";
        default: return "?";
    }
}

// INFO types as vcf-types.go:43-48 numbers them
enum VcfType : uint8_t { VT_INVALID = 0, VT_INTEGER, VT_FLOAT, VT_FLAG, VT_CHARACTER, VT_STRING };

// ---- strconv.ParseFloat(s, 64) ----
enum GoFloat : int { GF_BAD = 0, GF_OK, GF_OVERFLOW, GF_BAND };

__host__ __device__ inline uint8_t go_lower(uint8_t c) { return c | ('x' - 'X'); }   // strconv's lower()
__host__ __device__ inline uint8_t ascii_lower(uint8_t c) { return c >= 'A' && c <= 'Z' ? c + ('a' - 'A') : c; }

// commonPrefixLenIgnoreCase(s, prefix)
__host__ __device__ inline uint64_t go_prefix_ci(const uint8_t* s, uint64_t n, const char* pre, uint64_t np) {
    uint64_t k = 0;
    while (k < n && k < np && ascii_lower(s[k]) == (uint8_t)pre[k]) k++;
    return k;
}

// underscoreOK (strconv/atoi.go): underscores only between digits (a base prefix counts as a digit)
__host__ __device__ inline bool go_underscore_ok(const uint8_t* s, uint64_t n) {
    char saw = '^';
    uint64_t i = 0;
    if (n >= 1 && (s[0] == '-' || s[0] == '+')) { s++; n--; }
    bool hex = false;
    if (n >= 2 && s[0] == '0' && (go_lower(s[1]) == 'b' || go_lower(s[1]) == 'o' || go_lower(s[1]) == 'x')) { i = 2; saw = '0'; hex = go_lower(s[1]) == 'x'; }
    for (; i < n; i++) {
        if ((s[i] >= '0' && s[i] <= '9') || (hex && go_lower(s[i]) >= 'a' && go_lower(s[i]) <= 'f')) { saw = '0'; continue; }
        if (s[i] == '_') { if (saw != '0') return false; saw = '_'; continue; }
        if (saw == '_') return false;
        saw = '!';
    }
    return saw != '_';
}

// The syntax of strconv.ParseFloat(s, 64) (atof.go: special, readFloat, the n == len(s) check), and where the value lies against the
// overflow bound 2^1024 - 2^970 (a value at or above it rounds to +-Inf: a range error; underflow is no error).  *x receives the exponent
// X of the value 0.d1d2... * base^X (base 10, or 2 for hex, with X counted in bits from the leading 1) when the class is GF_BAND.
__host__ __device__ inline int go_float(const uint8_t* s, uint64_t n, int64_t* x) {
    if (!n) return GF_BAD;
    {   // special: an optional sign and "inf" / "infinity", or "nan" without a sign, case-insensitive
        uint64_t ns = 0, k = 0;
        const uint8_t c0 = s[0];
        if (c0 == '+' || c0 == '-' || c0 == 'i' || c0 == 'I') {
            ns = (c0 == '+' || c0 == '-') ? 1 : 0;
            k = go_prefix_ci(s + ns, n - ns, "infinity", 8);
            if (k > 3 && k < 8) k = 3;
            if (k == 3 || k == 8) return ns + k == n ? GF_OK : GF_BAD;
        } else if (c0 == 'n' || c0 == 'N') {
            if (go_prefix_ci(s, n, "nan", 3) == 3) return n == 3 ? GF_OK : GF_BAD;
        }
    }
    uint64_t i = 0;
    bool underscores = false;
    if (s[i] == '+' || s[i] == '-') i++;
    bool hex = false;
    uint8_t exp_char = 'e';
    if (i + 2 < n && s[i] == '0' && go_lower(s[i + 1]) == 'x') { hex = true; i += 2; exp_char = 'p'; }
    bool sawdot = false, sawdigits = false;
    int64_t nd = 0, dp = 0;
    uint32_t lead = 0;   // the first non-zero digit
    for (; i < n; i++) {
        const uint8_t c = s[i];
        if (c == '_') { underscores = true; continue; }
        if (c == '.') { if (sawdot) break; sawdot = true; dp = nd; continue; }
        uint32_t d;
        if (c >= '0' && c <= '9') d = c - '0';
        else if (hex && go_lower(c) >= 'a' && go_lower(c) <= 'f') d = go_lower(c) - 'a' + 10;
        else break;
        sawdigits = true;
        if (d == 0 && nd == 0) { dp--; continue; }   // leading zeros
        if (nd == 0) lead = d;
        nd++;
    }
    if (!sawdigits) return GF_BAD;
    if (!sawdot) dp = nd;
    int64_t e = 0, esign = 1;
    if (i < n && go_lower(s[i]) == exp_char) {
        i++;
        if (i >= n) return GF_BAD;
        if (s[i] == '+') i++; else if (s[i] == '-') { i++; esign = -1; }
        if (i >= n || s[i] < '0' || s[i] > '9') return GF_BAD;
        for (; i < n && ((s[i] >= '0' && s[i] <= '9') || s[i] == '_'); i++) {
            if (s[i] == '_') { underscores = true; continue; }
            if (e < 10000) e = e * 10 + (s[i] - '0');
        }
    } else if (hex) return GF_BAD;   // a hex mantissa must have a 'p' exponent
    if (underscores && !go_underscore_ok(s, i)) return GF_BAD;
    if (i != n) return GF_BAD;
    if (nd == 0) return GF_OK;       // zero
    int64_t X;
    if (!hex) {
        X = dp + esign * e;          // value in [10^(X-1), 10^X)
        if (X <= 308) return GF_OK;
        if (X >= 310) return GF_OVERFLOW;
    } else {
        const int L = lead >= 8 ? 4 : lead >= 4 ? 3 : lead >= 2 ? 2 : 1;
        X = 4 * dp + esign * e - 4 + L;   // value in [2^(X-1), 2^X)
        if (X <= 1023) return GF_OK;
        if (X >= 1025) return GF_OVERFLOW;
    }
    *x = X;
    return GF_BAND;
}

// the exact check of a GF_BAND value on the host: the digits of s as 0.M * 10^P (0x0.M p P for hex) with P the exponent strconv
// computes (its saturated exponent included), rounded by strtod; true when it rounds to +-Inf
inline bool go_float_overflows(const uint8_t* s, uint64_t n) {
    uint64_t i = 0;
    std::string t;
    if (s[0] == '+' || s[0] == '-') { if (s[0] == '-') t += '-'; i = 1; }
    bool hex = false;
    if (i + 2 < n && s[i] == '0' && go_lower(s[i + 1]) == 'x') { hex = true; i += 2; }
    t += hex ? "0x0." : "0.";
    int64_t before = 0; bool dot = false;
    for (; i < n; i++) {
        const uint8_t c = s[i];
        if (c == '_') continue;
        if (c == '.') { dot = true; continue; }
        if ((c >= '0' && c <= '9') || (hex && go_lower(c) >= 'a' && go_lower(c) <= 'f')) { t += (char)c; if (!dot) before++; continue; }
        break;
    }
    int64_t e = 0, esign = 1;
    if (i < n) {   // the exponent character
        i++;
        if (s[i] == '+') i++; else if (s[i] == '-') { i++; esign = -1; }
        for (; i < n; i++) { if (s[i] == '_') continue; if (e < 10000) e = e * 10 + (s[i] - '0'); }
    }
    const int64_t P = (hex ? 4 * before : before) + esign * e;
    t += hex ? 'p' : 'e';
    t += std::to_string(P);
    errno = 0;
    const double v = strtod(t.c_str(), nullptr);
    return std::isinf(v);
}

// utf8.DecodeRune on p[0, n) with p[0] >= 0x80: the size of a valid encoding other than U+FFFD, or 0 (RuneError)
__device__ __forceinline__ uint32_t go_rune(const uint8_t* p, uint64_t n) {
    const uint8_t c = p[0];
    uint32_t sz, lo = 0x80, hi = 0xBF, r;
    if (c >= 0xC2 && c <= 0xDF) { sz = 2; r = c & 0x1F; }
    else if (c >= 0xE0 && c <= 0xEF) { sz = 3; r = c & 0x0F; if (c == 0xE0) lo = 0xA0; if (c == 0xED) hi = 0x9F; }
    else if (c >= 0xF0 && c <= 0xF4) { sz = 4; r = c & 0x07; if (c == 0xF0) lo = 0x90; if (c == 0xF4) hi = 0x8F; }
    else return 0;
    if (n < sz) return 0;
    for (uint32_t j = 1; j < sz; j++) {
        const uint8_t b = p[j];
        if (b < (j == 1 ? lo : 0x80) || b > (j == 1 ? hi : 0xBF)) return 0;
        r = (r << 6) | (b & 0x3F);
    }
    return r == 0xFFFD ? 0 : sz;
}

// ---- vcf_parse ----
struct VcfInfoTab {                       // the declared INFO IDs (the first of equal IDs: SmallMap.Get), on the device
    const uint8_t* names; const uint32_t* off; const uint8_t* type; const int32_t* number; int n;
};

struct VcfArgs {
    const uint8_t* t; const uint64_t* ls; uint64_t n_lines;
    uint64_t line0;                       // the 1-based line number of the chunk's first line in its file
    NameDict dict; VcfInfoTab info;
    int32_t* ent; int32_t* start; int32_t* end; uint32_t* emit;
    unsigned long long* small;            // [0] first error (line << 8 | VcfErr), [1] data lines on no @SQ SN
    uint64_t* band_line; uint64_t* band_at; unsigned long long* n_band;   // QUAL near the overflow bound: line, offset << 16 | length
};

constexpr int VP_T = 256, VP_SLOTS = 9;   // per line: tabs 0..6, INFO's first ' ' / ':' / tab, the number of tabs seen (at most 7)

__device__ __forceinline__ uint64_t skip_space(const uint8_t* p, uint64_t n, uint64_t i) { while (i < n && p[i] == ' ') i++; return i; }
__device__ __forceinline__ bool info_end(uint8_t c) { return c == ' ' || c == ',' || c == ';' || c == '\t'; }   // endOfInfoEntry
__device__ __forceinline__ uint64_t until_info_end(const uint8_t* p, uint64_t n, uint64_t i) { while (i < n && !info_end(p[i])) i++; return i; }

// the declared INFO entry named p[a, b), or -1
__device__ int info_decl(const VcfInfoTab& T, const uint8_t* p, uint64_t a, uint64_t b) {
    for (int k = 0; k < T.n; k++) {
        const uint32_t o = T.off[k], len = T.off[k + 1] - o;
        if (len != b - a) continue;
        uint32_t j = 0;
        while (j < len && T.names[o + j] == p[a + j]) j++;
        if (j == len) return k;
    }
    return -1;
}

// doInfo (vcf-files.go:708-725) from index i; d0: the first ' ', ':' or tab at or after i (or n).  0, VL_INFO, or VL_END for a key "END"
__device__ uint32_t info_walk(const VcfInfoTab& T, const uint8_t* p, uint64_t n, uint64_t i, uint64_t d0) {
    bool first = true, has_end = false;
    for (;;) {
        const uint64_t a = skip_space(p, n, i);
        uint64_t b = a;
        if (first && a == i) b = d0;
        else while (b < n && p[b] != ' ' && p[b] != ':' && p[b] != '\t') b++;
        first = false;
        if (b - a == 3 && p[a] == 'E' && p[a + 1] == 'N' && p[a + 2] == 'D') has_end = true;
        i = b;
        const int k = info_decl(T, p, a, b);
        if (k >= 0) {
            const uint8_t ty = T.type[k];
            i = skip_space(p, n, i);
            if (ty != VT_FLAG) {   // make1InfoParser / makeNInfoParser: '=' is checked, not consumed
                if (i >= n || p[i] != '=') return VL_INFO;
                if (ty == VT_INTEGER || ty == VT_FLOAT) return VL_INFO;   // the value read starts with '='
                if (T.number[k] == 1) {
                    i = ty == VT_CHARACTER ? i + 1 : until_info_end(p, n, i);
                    i = skip_space(p, n, i);
                } else {
                    for (;;) {
                        if (ty == VT_CHARACTER) {
                            if (i >= n) return VL_INFO;
                            if (p[i] < 0x80) i++;
                            else { const uint32_t sz = go_rune(p + i, n - i); if (!sz) return VL_INFO; i += sz; }
                        } else i = until_info_end(p, n, i);
                        i = skip_space(p, n, i);
                        if (i >= n || p[i] != ',') break;
                        i++;
                    }
                }
            }
        } else {   // ParseGenericInfo
            i = skip_space(p, n, i);
            if (i < n && p[i] == '=') {
                i = skip_space(p, n, i + 1);
                for (;;) {
                    i = skip_space(p, n, until_info_end(p, n, i));
                    if (i >= n || p[i] != ',') break;
                    i++;
                }
            }
        }
        i = skip_space(p, n, i);
        if (i >= n || p[i] != ':') return has_end ? VL_END : 0;
        i++;
    }
}

__global__ void __launch_bounds__(VP_T) vcf_parse_kernel(VcfArgs A) {
    __shared__ uint32_t sh[VP_T / 32][32 * VP_SLOTS];
    const unsigned lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
    uint32_t* S = sh[wib];
    const uint64_t n_groups = (A.n_lines + 31) / 32, stride = (uint64_t)gridDim.x * (VP_T / 32);
    for (uint64_t g = (uint64_t)blockIdx.x * (VP_T / 32) + wib; g < n_groups; g += stride) {
        const uint64_t k0 = g * 32;
        const uint32_t nl = A.n_lines - k0 < 32 ? (uint32_t)(A.n_lines - k0) : 32u;
        // the warp walks each line: the tabs ending CHROM .. FILTER, then INFO's first ' ', ':' or tab
        for (uint32_t l = 0; l < nl; l++) {
            const uint64_t s0 = A.ls[k0 + l], raw = A.ls[k0 + l + 1] - 1 - s0;
            if (raw >= VCF_MAX_LINE) continue;
            const uint8_t* p = A.t + s0;
            const uint64_t n = raw && p[raw - 1] == '\r' ? raw - 1 : raw;
            uint32_t ntab = 0, d = (uint32_t)n;
            for (uint32_t w = 0; w < n; w += 32) {
                const uint32_t q = w + lane;
                const uint8_t b = q < n ? p[q] : 0;
                const unsigned tm = __ballot_sync(FULL_MASK, b == '\t');
                const unsigned dm = __ballot_sync(FULL_MASK, b == '\t' || b == ' ' || b == ':');
                if (ntab < 7 && b == '\t') { const uint32_t r = ntab + __popc(tm & ((1u << lane) - 1)); if (r < 7) S[l * VP_SLOTS + r] = q; }
                ntab = min(7u, ntab + __popc(tm));
                __syncwarp();
                if (ntab == 7) {
                    const uint32_t s7 = S[l * VP_SLOTS + 6] + 1;
                    const unsigned m = s7 <= w ? dm : (s7 - w >= 32 ? 0u : dm & (~0u << (s7 - w)));
                    if (m) { d = w + __ffs(m) - 1; break; }
                }
            }
            if (lane == 0) { S[l * VP_SLOTS + 7] = d; S[l * VP_SLOTS + 8] = ntab; }
        }
        __syncwarp();
        // each lane checks one line's fields from those positions (ParseVariant, vcf-files.go:773-782)
        const uint64_t k = k0 + lane;
        const bool live = lane < nl;
        uint32_t err = 0;
        uint64_t cs = 0, cn = 0;          // CHROM's bytes (from A.t)
        bool chrom_dot = false;           // CHROM is the missing entry "." with no byte to point at
        int64_t pos = -1;
        uint64_t ref_len = 1;
        if (live) {
            const uint64_t s0 = A.ls[k], raw = A.ls[k + 1] - 1 - s0;
            const uint8_t* p = A.t + s0;
            const uint64_t n = raw && p[raw - 1] == '\r' ? raw - 1 : raw;
            const uint32_t* P = S + lane * VP_SLOTS;
            if (raw >= VCF_MAX_LINE) err = VL_LONG;
            else {
                const uint32_t ntab = P[8];
                uint64_t idx = 0;
                for (uint32_t f = 0; f < 7 && !err; f++) {
                    if (idx >= n) { if (f == 0) chrom_dot = true; continue; }   // missingEntry past the end: every later field too
                    const bool dot = p[idx] == '.' && (idx + 1 >= n || p[idx + 1] == '\t');
                    uint64_t e;
                    if (f < ntab) e = P[f];
                    else if (dot) e = n;   // "." at the end of the line: missing, and the index lands past the end
                    else { err = VL_TAB; break; }
                    const uint64_t a = idx;
                    idx = e + 1;
                    if (f == 0) { cs = s0 + a; cn = e - a; }
                    else if (f == 1) { if (!dot && !parse_dec(p + a, e - a, true, INT32_MIN, INT32_MAX, &pos)) err = VL_POS; }
                    else if (f == 3) { ref_len = dot ? 1 : e - a; }
                    else if (f == 5 && !dot) {
                        int64_t x = 0;
                        const int fc = go_float(p + a, e - a, &x);
                        if (fc == GF_BAD) err = VL_QUAL;
                        else if (fc == GF_OVERFLOW) err = VL_QUAL_RANGE;
                        else if (fc == GF_BAND) {
                            const unsigned long long j = atomicAdd(A.n_band, 1ull);
                            A.band_line[j] = k; A.band_at[j] = ((s0 + a) << 16) | (e - a);
                        }
                    } else if (f == 6 && !dot) {   // doFilter: "PASS" must be followed by the tab, not by ';'
                        if (e - a > 4 && p[a] == 'P' && p[a + 1] == 'A' && p[a + 2] == 'S' && p[a + 3] == 'S' && p[a + 4] == ';') err = VL_TAB;
                    }
                }
                if (!err) err = info_walk(A.info, p, n, min(idx, n), ntab == 7 && idx <= n ? P[7] : n);
                if (!err && !chrom_dot && cn == 0) err = VL_CHROM;
            }
        }
        // the name: a line whose CHROM equals the previous lane's takes that lane's entry; the first line of each run looks it up
        const bool named = live && !err;
        const uint64_t pcs = __shfl_up_sync(FULL_MASK, cs, 1), pcn = __shfl_up_sync(FULL_MASK, cn, 1);
        const bool pnamed = __shfl_up_sync(FULL_MASK, (int)(named && !chrom_dot), 1) != 0;
        bool lead = named;
        if (named && !chrom_dot && lane > 0 && pnamed && pcn == cn) {
            const uint8_t* a = A.t + cs; const uint8_t* b = A.t + pcs;
            uint64_t j = 0;
            while (j < cn && a[j] == b[j]) j++;
            lead = j < cn;
        }
        const uint8_t dotname = '.';
        int e = lead ? (chrom_dot ? name_entry(A.dict, &dotname, 1) : name_entry(A.dict, A.t + cs, cn)) : -1;
        const unsigned below = __ballot_sync(FULL_MASK, lead) & (0xffffffffu >> (31 - lane));
        const int e_lead = __shfl_sync(FULL_MASK, e, below ? 31 - __clz(below) : (int)lane);
        if (named && !lead) e = e_lead;
        const uint32_t m = named && e >= 0 ? A.dict.all_off[e + 1] - A.dict.all_off[e] : 0;
        if (live) {
            A.emit[k] = m;
            if (named) { A.ent[k] = e; A.start[k] = (int32_t)pos; A.end[k] = (int32_t)((uint32_t)(int32_t)pos - 1u + (uint32_t)ref_len); }
            else atomicMin(A.small, ((unsigned long long)(A.line0 + k) << 8) | err);
        }
        const unsigned um = __ballot_sync(FULL_MASK, named && m == 0);   // accepted lines on a chromosome that is no @SQ SN ("*" included)
        if (lane == 0 && um) atomicAdd(A.small + 1, (unsigned long long)__popc(um));
        __syncwarp();
    }
}

// ---- the header, on the host ----
struct VcfInfo { std::string id; uint8_t type; int32_t number; };
struct VcfHeader { uint64_t lines = 0, bytes = 0; std::vector<VcfInfo> infos; };

// StringScanner (string-scanner.go) over one header line
struct HScan {
    const std::string& d; size_t i = 0;
    explicit HScan(const std::string& s) : d(s) {}
    void skip_space() { while (i < d.size() && d[i] == ' ') i++; }
};

// ParseMetaField (vcf-files.go:73-113): nullptr, or why it panics
inline const char* meta_field(HScan& sc, std::string& key, std::string& value) {
    sc.skip_space();
    size_t st = sc.i;
    while (sc.i < sc.d.size() && sc.d[sc.i] != ' ' && sc.d[sc.i] != '=') sc.i++;
    key = sc.d.substr(st, sc.i - st);
    sc.skip_space();
    if (sc.i >= sc.d.size() || sc.d[sc.i] != '=') return "invalid key=pair pair in a VCF meta-information line";
    sc.i++;
    sc.skip_space();
    if (sc.i >= sc.d.size()) return "a meta-information value is empty at the end of the line (index out of range)";
    st = sc.i;
    if (sc.d[sc.i] == '"') {
        value.clear();
        for (sc.i++; sc.i < sc.d.size(); sc.i++) {
            if (sc.d[sc.i] == '"') { sc.i++; return nullptr; }
            if (sc.d[sc.i] == '\\') sc.i++;
            if (sc.i >= sc.d.size()) return "a '\\' ends the line inside a quoted value (index out of range)";
            value += sc.d[sc.i];
        }
        return "missing closing \" in a VCF meta-information line";
    }
    for (; sc.i < sc.d.size(); sc.i++) {
        const char c = sc.d[sc.i];
        if (c == ' ' || c == ',' || c == '>') { value = sc.d.substr(st, sc.i - st); return nullptr; }
    }
    return "missing closing > in a VCF meta-information line";
}

// after a field: ',' continues, '>' ends, anything else (or the end of the line) panics
inline const char* meta_next(HScan& sc, bool* done) {
    sc.skip_space();
    if (sc.i >= sc.d.size()) return "a meta-information line ends after a field (index out of range)";
    if (sc.d[sc.i] == ',') { sc.i++; *done = false; return nullptr; }
    if (sc.d[sc.i] == '>') { sc.i++; *done = true; return nullptr; }
    return "invalid syntax in a VCF meta-information line";
}

// ParseMetaInformation (vcf-files.go:116-158)
inline const char* meta_information(HScan& sc) {
    if (sc.i >= sc.d.size()) return "empty meta-information value (index out of range)";
    if (sc.d[sc.i] != '<') return nullptr;
    sc.i++;
    bool id = false, done = false;
    std::string desc, key, value;
    std::vector<std::string> fields;
    while (!done) {
        if (const char* w = meta_field(sc, key, value)) return w;
        if (key == "ID") { if (id) return "multiple IDs in a VCF meta-information line"; id = true; }
        else if (key == "Description") { if (!desc.empty()) return "multiple Descriptions in a VCF meta-information line"; desc = value; }
        else { for (auto& f : fields) if (f == key) return "duplicate field key in a VCF meta-information line"; fields.push_back(key); }
        if (const char* w = meta_next(sc, &done)) return w;
    }
    return id ? nullptr : "missing ID in a VCF meta-information line";
}

// ParseFormatInformation (vcf-files.go:161-243), then CreateInfoParser / CreateFormatParser's panics (:442-477, :569-598)
inline const char* format_information(HScan& sc, bool info, VcfInfo* out) {
    if (sc.i >= sc.d.size()) return "empty INFO/FORMAT value (index out of range)";
    if (sc.d[sc.i] != '<') return "missing open angle bracket in a VCF INFO/FORMAT meta-information line";
    sc.i++;
    bool id = false, done = false;
    int32_t number = -5;   // InvalidNumber
    uint8_t type = VT_INVALID;
    std::string desc, key, value;
    std::vector<std::string> fields;
    while (!done) {
        if (const char* w = meta_field(sc, key, value)) return w;
        if (key == "ID") { if (id) return "multiple IDs in a VCF INFO/FORMAT meta-information line"; id = true; out->id = value; }
        else if (key == "Description") { if (!desc.empty()) return "multiple Descriptions in a VCF INFO/FORMAT meta-information line"; desc = value; }
        else if (key == "Number") {
            if (number > -5) return "multiple Number entries in a VCF INFO/FORMAT meta-information line";
            if (value == "a" || value == "A") number = -1;
            else if (value == "r" || value == "R") number = -2;
            else if (value == "g" || value == "G") number = -3;
            else if (value == ".") number = -4;
            else {
                const char* s = value.c_str(); size_t i = 0, n = value.size(); bool neg = false; int64_t v = 0;
                if (n && (s[0] == '+' || s[0] == '-')) { neg = s[0] == '-'; i = 1; }
                if (i >= n) return "Number: strconv.ParseInt(s, 10, 32) fails";
                for (; i < n; i++) { if (s[i] < '0' || s[i] > '9') return "Number: strconv.ParseInt(s, 10, 32) fails"; if (v < (1ll << 40)) v = v * 10 + (s[i] - '0'); }
                if (neg) v = -v;
                if (v < INT32_MIN || v > INT32_MAX) return "Number: strconv.ParseInt(s, 10, 32) fails";
                number = (int32_t)v;
            }
        } else if (key == "Type") {
            if (type != VT_INVALID) return "multiple types in a VCF INFO/FORMAT meta-information line";
            if (value == "Integer") type = VT_INTEGER;
            else if (value == "Float") type = VT_FLOAT;
            else if (value == "Flag") type = VT_FLAG;
            else if (value == "Character") type = VT_CHARACTER;
            else if (value == "String") type = VT_STRING;
            else return "unknown type in a VCF INFO/FORMAT meta-information line";
        } else { for (auto& f : fields) if (f == key) return "duplicate field key in a VCF meta-information line"; fields.push_back(key); }
        if (const char* w = meta_next(sc, &done)) return w;
    }
    if (!id) return "missing ID in a VCF INFO/FORMAT meta-information line";
    if (number <= -5) return "missing number entry in a VCF INFO/FORMAT meta-information line";
    if (type == VT_INVALID) return "missing type in a VCF INFO/FORMAT meta-information line";
    if (info && type == VT_FLAG && number != 0) return "INFO Type Flag with Number != 0 (CreateInfoParser)";
    if (!info && type == VT_FLAG) return "FORMAT Type Flag (CreateFormatParser: invalid FORMAT Type)";
    out->type = type; out->number = number;
    return nullptr;
}

// bytes of the file in order; more(buf) appends the next bytes to buf: > 0 appended, 0 at the end of the file, < 0 an error code
// (already reported)
template <class More>
struct HReader {
    More& more; std::vector<uint8_t> buf; size_t at = 0; uint64_t used = 0; int rc = 0; bool eof = false;
    explicit HReader(More& m) : more(m) {}
    int peek() {   // the next byte, -1 at the end of the file, -2 after an error
        while (at >= buf.size()) {
            if (eof) return -1;
            if (rc) return -2;
            buf.erase(buf.begin(), buf.begin() + at); at = 0;
            const int r = more(buf);
            if (r < 0) { rc = r; return -2; }
            if (r == 0) eof = true;
        }
        return buf[at];
    }
    int get() { const int c = peek(); if (c >= 0) { at++; used++; } return c; }
    // getLine (vcf-files.go:245-258): through '\n' (dropped with one '\r' before it) or the end of the file
    int line(std::string& s) {
        s.clear();
        for (;;) {
            const int c = get();
            if (c == -2) return rc;
            if (c < 0) return 0;
            if (c == '\n') { if (!s.empty() && s.back() == '\r') s.pop_back(); return 0; }
            s += (char)c;
        }
    }
};

// ParseHeader (vcf-files.go:261-305) and NewVariantParser's checks: 0 and *h, or E_VCF with *bad_line and *why, or another error code
template <class More>
int vcf_header(More& more, VcfHeader* h, uint64_t* bad_line, const char** why) {
    HReader<More> r(more);
    std::string line;
    uint64_t lines = 0;
    auto bad = [&](uint64_t l, const char* w) { *bad_line = l; *why = w; return E_VCF; };
    if (int rc = r.line(line)) return rc;
    lines++;
    if (line.size() < VCF_PREFIX_LEN) return bad(1, "the first line is shorter than \"##fileformat=VCFv4.\" (slice out of range)");
    if (line.compare(0, VCF_PREFIX_LEN, VCF_PREFIX) != 0) return bad(1, "invalid first line in a VCF file");
    for (;;) {
        int c = r.peek();
        if (c == -2) return r.rc;
        if (c != '#') return bad(lines + 1, "unexpected end of VCF header");
        r.get();
        c = r.peek();
        if (c == -2) return r.rc;
        if (c < 0) return bad(lines + 1, "unexpected end of VCF header");
        if (c != '#') break;
        r.get();
        if (int rc = r.line(line)) return rc;
        lines++;
        HScan sc(line);
        const size_t eq = line.find('=');
        if (eq == std::string::npos) return bad(lines, "invalid syntax in a VCF header (no '=')");
        const std::string key = line.substr(0, eq);
        sc.i = eq + 1;
        const char* w = nullptr;
        if (key == "fileformat") w = "multiple file format meta-information lines in a VCF file";
        else if (key == "INFO" || key == "FORMAT") {
            VcfInfo fi;
            w = format_information(sc, key == "INFO", &fi);
            if (!w && key == "INFO") h->infos.push_back(fi);
        } else w = meta_information(sc);
        if (w) return bad(lines, w);
    }
    if (int rc = r.line(line)) return rc;   // the #CHROM column line
    lines++;
    h->lines = lines; h->bytes = r.used;
    return E_OK;
}

}  // namespace
