// sam_ingest.cu -- SAM text alignment lines straight into the device columns (replaces the host-side parseSamAlignment,
// sam/sam-files.go:386-410, together with the formatBamAlignment, sam/bam-files.go:635-737, that a SAM-in / BAM-out run
// applies to every read).
//
// Every line becomes, on the device, exactly the BAM record formatBamAlignment(parseSamAlignment(line)) writes; the records
// then go through the BAM ingest core (bam_ingest_core: filters, RG:Z, sr bit, QUAL presence, the elp_fetch_bam arena).
//   sam_lines    two streaming passes over the text (16-byte loads): '\n' count per 64-byte chunk, exclusive scan, line starts
//   sam_measure  one warp per line: parse and validate, BAM record length of the line
//   sam_emit     one warp per line: the same parser (parse_line<true>) writes the record at its scanned offset
//   sam_fpatch   float values the device does not round itself (see parse_f32), rounded on the host with strtof
// The text is split like bufio.ScanLines: lines end at '\n', a '\r' before it is dropped, the last line may lack its '\n'.
#include <algorithm>
#include <cmath>
#include <cstdlib>
#include <locale.h>
#include "ctx.h"
#include "text_parse.cuh"
#include "../../include/elprep_b200.h"

struct SlowF { uint64_t text_off, out_off; uint32_t len, line; };   // one float value host-rounded: text, position in bam_raw, line

struct SamState {
    DBuf<uint8_t> text; DBuf<uint32_t> cnt, len; DBuf<uint64_t> cnt_off, ls;
    DBuf<SlowF> slow; DBuf<uint64_t> patch_off; DBuf<uint32_t> patch_bits;
    DBuf<uint8_t> lost;                       // per line: 1 if its RNAME / RNEXT text is lost in the record (see parse_line)
    DBuf<unsigned long long> d_small;         // [0] first error (line << 8 | SamErr), [1] floats handed to the host, [2] lines with a lost name
    uint64_t h_last = 0;                      // source of the virtual line end of a final line without '\n'
};

void free_state(SamState* S) { delete S; }

namespace {

// which field of the line failed; the smallest (line << 8 | code) of a call is reported
enum SamErr : uint32_t {
    SE_EMPTY = 1, SE_TABS, SE_QNAME, SE_FLAG, SE_POS, SE_MAPQ, SE_CIGAR, SE_CIGAR_LEN, SE_PNEXT, SE_TLEN, SE_QUAL,
    SE_TAG, SE_TAG_A, SE_TAG_I, SE_TAG_F, SE_TAG_H, SE_TAG_B, SE_TAG_TYPE, SE_FLOAT_RANGE,
    SE_CIGAR_LIMIT = 0x80, SE_RECORD_LIMIT
};
const char* sam_err_text(uint32_t e) {
    switch (e) {
        case SE_EMPTY: return "empty line";
        case SE_TABS: return "missing tabulator in SAM alignment line (fewer than 11 mandatory fields)";
        case SE_QNAME: return "QNAME longer than 254 bytes (BAM l_read_name would wrap)";
        case SE_FLAG: return "FLAG: strconv.ParseUint(s, 10, 16) fails";
        case SE_POS: return "POS: strconv.ParseInt(s, 10, 32) fails";
        case SE_MAPQ: return "MAPQ: strconv.ParseUint(s, 10, 8) fails";
        case SE_CIGAR: return "CIGAR: invalid operation or length";
        case SE_CIGAR_LEN: return "CIGAR: operation length of 2^28 or more (BAM len<<4 would overflow)";
        case SE_PNEXT: return "PNEXT: strconv.ParseInt(s, 10, 32) fails";
        case SE_TLEN: return "TLEN: strconv.ParseInt(s, 10, 32) fails";
        case SE_QUAL: return "QUAL and SEQ differ in length";
        case SE_TAG: return "optional field: invalid field tag or type separator";
        case SE_TAG_A: return "optional field of type A: not exactly one character";
        case SE_TAG_I: return "optional field of type i: not an integer in [-2^31, 2^32-1] (the BAM range)";
        case SE_TAG_F: return "optional field of type f: invalid float (hexadecimal floats are not supported)";
        case SE_TAG_H: return "optional field of type H: odd length or a non-hex digit";
        case SE_TAG_B: return "optional field of type B: invalid array type or entry";
        case SE_TAG_TYPE: return "optional field: unknown type";
        case SE_FLOAT_RANGE: return "optional field of type f: value out of float32 range";
        case SE_CIGAR_LIMIT: return "CIGAR with more than 65535 operations (the BAM CG:B convention is not supported)";
        case SE_RECORD_LIMIT: return "BAM record of 2^31 bytes or more";
        default: return "?";
    }
}

// ---- the line parser ----
struct SamArgs {
    const uint8_t* text; const uint64_t* ls; uint64_t n_lines;
    NameDict dict;             // "*" and @SQ SN, sorted, with their refid (the input name table while elp_set_input_dictionary is set)
    int32_t unreached_ref;     // refID of an RNAME that is neither "*" nor in dict: -1, or under REPLACE the entry whose remap drops the read
    uint32_t* len;             // measure: BAM record length per line
    uint8_t* lost;             // measure: 1 if the record loses the line's RNAME / RNEXT text
    const uint64_t* rec_off;   // emit: record offsets in out
    uint8_t* out;
    unsigned long long* small; SlowF* slow;
};

// first '\t' at or after `from`, or n: 32 bytes per step, one per lane (all lanes of the warp call it with the same arguments)
__device__ __forceinline__ uint64_t next_tab(const uint8_t* p, uint64_t from, uint64_t n) {
    const unsigned lane = threadIdx.x & 31;
    for (uint64_t b = from; b < n; b += 32) {
        const unsigned m = __ballot_sync(FULL_MASK, b + lane < n && p[b + lane] == '\t');
        if (m) return b + __ffs(m) - 1;
    }
    return n;
}

__device__ __forceinline__ bool ieq(const uint8_t* p, const char* s, int n) { for (int i = 0; i < n; i++) if ((p[i] | 0x20) != (uint8_t)s[i]) return false; return true; }

// strconv.ParseFloat(s, 32) -> float32 bits.  0: invalid syntax (hexadecimal floats included), 1: *bits is the correctly rounded value,
// 2: a valid decimal the host rounds (strtof).  The device rounds a decimal whose significand is below 2^24 and whose decimal exponent
// lies in [-10, 10]: both operands are then exact in float32, so one IEEE multiplication or division rounds correctly.
__device__ int parse_f32(const uint8_t* p, uint64_t n, uint32_t* bits) {
    uint64_t i = 0; bool neg = false;
    if (n && (p[0] == '+' || p[0] == '-')) { neg = p[0] == '-'; i = 1; }
    if (i < n && (p[i] | 0x20) == 'i') {                                     // strconv special(): inf, infinity, with an optional sign
        if ((n - i == 3 && ieq(p + i, "inf", 3)) || (n - i == 8 && ieq(p + i, "infinity", 8))) { *bits = neg ? 0xff800000u : 0x7f800000u; return 1; }
        return 0;
    }
    if (i == 0 && n == 3 && ieq(p, "nan", 3)) { *bits = 0x7fc00000u; return 1; }   // float32(math.NaN())
    uint64_t mant = 0; int64_t dp = 0; bool dig = false, dot = false, slow = false;
    for (; i < n; i++) {
        const uint8_t ch = p[i];
        if (ch == '.') { if (dot) break; dot = true; continue; }
        if (ch < '0' || ch > '9') break;
        dig = true;
        if (mant == 0 && ch == '0') { if (dot) dp--; continue; }
        if (mant < (1u << 24)) { mant = mant * 10 + (ch - '0'); if (dot) dp--; } else slow = true;
    }
    if (!dig) return 0;
    int64_t ex = 0;
    if (i < n && (p[i] | 0x20) == 'e') {
        i++;
        bool eneg = false;
        if (i < n && (p[i] == '+' || p[i] == '-')) { eneg = p[i] == '-'; i++; }
        if (i >= n) return 0;
        for (; i < n && p[i] >= '0' && p[i] <= '9'; i++) if (ex < 100000) ex = ex * 10 + (p[i] - '0');
        if (eneg) ex = -ex;
    }
    if (i != n) return 0;
    if (mant == 0) { *bits = neg ? 0x80000000u : 0u; return 1; }
    const int64_t e10 = dp + ex;
    if (slow || mant >= (1u << 24) || e10 < -10 || e10 > 10) return 2;
    float pw = 1.0f;                                                          // 10^|e10|: every step is exact up to 1e10
    for (int64_t q = e10 < 0 ? -e10 : e10; q > 0; q--) pw = __fmul_rn(pw, 10.0f);
    float f = (float)mant;
    f = e10 >= 0 ? __fmul_rn(f, pw) : __fdiv_rn(f, pw);
    *bits = __float_as_uint(neg ? -f : f);
    return 1;
}

__device__ __forceinline__ int cigar_code(uint8_t ch) {   // "MmIiDdNnSsHhPpXx=" -> BAM op (sam/sam-types.go:661-670)
    switch (ch | (ch >= 'A' ? 0x20 : 0)) {
        case 'm': return 0; case 'i': return 1; case 'd': return 2; case 'n': return 3; case 's': return 4;
        case 'h': return 5; case 'p': return 6; case '=': return 7; case 'x': return 8;
        default: return -1;
    }
}
__device__ __forceinline__ bool is_hex(uint8_t ch) { return (ch >= '0' && ch <= '9') || ((ch | 0x20) >= 'a' && (ch | 0x20) <= 'f'); }

template <bool W> __device__ __forceinline__ void put(uint8_t* o, uint32_t v, int nb) { if (W && (threadIdx.x & 31) == 0) for (int b = 0; b < nb; b++) o[b] = (uint8_t)(v >> (8 * b)); }

// a float value of an f tag or a B:f entry: the bits, or a placeholder and an entry of the host list (keep: this occurrence of the
// tag is the one written, so measure counts it and emit lists it)
template <bool W> __device__ int float_value(const SamArgs& A, const uint8_t* p, uint64_t a, uint64_t n, uint8_t* o, uint64_t s0, uint64_t oabs, uint64_t line, bool keep) {
    uint32_t bits = 0;
    const int r = parse_f32(p + a, n, &bits);
    if (!r) return SE_TAG_F;
    if (r == 2 && keep && (threadIdx.x & 31) == 0) {
        const unsigned long long j = atomicAdd(A.small + 1, 1ull);
        if (W) { SlowF sf; sf.text_off = s0 + a; sf.out_off = oabs; sf.len = (uint32_t)n; sf.line = (uint32_t)line; A.slow[j] = sf; }
    }
    put<W>(o, bits, 4);
    return 0;
}

// one optional field "TG:T:value" = p[a, b); writes it at o (absolute offset oabs in out) and returns its BAM size in *sz
template <bool W> __device__ int tag_value(const SamArgs& A, const uint8_t* p, uint64_t a, uint64_t b, uint8_t* o, uint64_t oabs, uint64_t s0, uint64_t line, bool keep, uint64_t* sz) {
    const unsigned lane = threadIdx.x & 31;
    const uint8_t ty = p[a + 3];
    const uint64_t v = a + 5, vn = b - v;
    put<W>(o, (uint32_t)p[a] | ((uint32_t)p[a + 1] << 8), 2);
    switch (ty) {
        case 'A':                                                            // parseSamChar: one byte, then a tab or the end of the line
            if (vn != 1) return SE_TAG_A;
            put<W>(o + 2, 'A' | ((uint32_t)p[v] << 8), 2); *sz = 4; return 0;
        case 'i': {                                                          // int64, written as the smallest BAM type that holds it (bam-files.go:492-525)
            int64_t x;
            if (!parse_dec(p + v, vn, true, -(1ll << 31), (1ll << 32) - 1, &x)) return SE_TAG_I;
            const uint8_t t = x < 0 ? (x >= -128 ? 'c' : x >= -32768 ? 's' : 'i') : (x <= 255 ? 'C' : x <= 65535 ? 'S' : 'I');
            const int nb = (t == 'c' || t == 'C') ? 1 : (t == 's' || t == 'S') ? 2 : 4;
            put<W>(o + 2, t, 1); put<W>(o + 3, (uint32_t)x, nb); *sz = 3 + nb; return 0;
        }
        case 'f':
            put<W>(o + 2, 'f', 1); *sz = 7;
            return float_value<W>(A, p, v, vn, o + 3, s0, oabs + 3, line, keep);
        case 'Z':
            put<W>(o + 2, 'Z', 1);
            if (W) { for (uint64_t j = lane; j < vn; j += 32) o[3 + j] = p[v + j]; put<W>(o + 3 + vn, 0, 1); }
            *sz = 3 + vn + 1; return 0;
        case 'H': {                                                          // hex pairs -> bytes -> upper-case hex again (bam-files.go:536-553)
            if (vn & 1) return SE_TAG_H;
            bool bad = false;
            for (uint64_t j0 = 0; j0 < vn && !bad; j0 += 32) bad = __any_sync(FULL_MASK, j0 + lane < vn && !is_hex(p[v + j0 + lane]));
            if (bad) return SE_TAG_H;
            put<W>(o + 2, 'H', 1);
            if (W) { for (uint64_t j = lane; j < vn; j += 32) { const uint8_t ch = p[v + j]; o[3 + j] = ch >= 'a' ? ch - 32 : ch; } put<W>(o + 3 + vn, 0, 1); }
            *sz = 3 + vn + 1; return 0;
        }
        case 'B': {                                                          // parseSamNumericArray (sam-files.go:237-317)
            if (vn < 2 || p[v + 1] != ',') return SE_TAG_B;
            const uint8_t sub = p[v];
            int64_t lo, hi; bool sg = false; int es = 4;
            switch (sub) {
                case 'c': lo = -128; hi = 127; sg = true; es = 1; break;
                case 'C': lo = 0; hi = 255; es = 1; break;
                case 's': case 'S': lo = 0; hi = 65535; es = 2; break;       // B:s goes through ParseUint(s, 10, 16) as well
                case 'i': lo = -(1ll << 31); hi = (1ll << 31) - 1; sg = true; break;
                case 'I': lo = 0; hi = (1ll << 32) - 1; break;
                case 'f': lo = hi = 0; break;
                default: return SE_TAG_B;
            }
            uint64_t cnt = 0;
            for (uint64_t x = v + 2;; cnt++) {
                uint64_t y = x;
                while (y < b && p[y] != ',') y++;
                uint8_t* e = o + 8 + (uint64_t)es * cnt;
                if (sub == 'f') { if (float_value<W>(A, p, x, y - x, e, s0, oabs + 8 + 4 * cnt, line, keep)) return SE_TAG_B; }
                else { int64_t z; if (!parse_dec(p + x, y - x, sg, lo, hi, &z)) return SE_TAG_B; put<W>(e, (uint32_t)z, es); }
                if (y == b) { cnt++; break; }
                x = y + 1;
            }
            put<W>(o + 2, 'B' | ((uint32_t)sub << 8), 2); put<W>(o + 4, (uint32_t)cnt, 4);
            *sz = 8 + (uint64_t)es * cnt; return 0;
        }
        default: return SE_TAG_TYPE;
    }
}

// parseSamAlignment + formatBamAlignment of line k.  W = false: validate and size (A.len[k]); W = true: write the record at
// A.out + A.rec_off[k].  Every lane runs the same control flow; lane 0 stores the serial parts, the warp copies the long ones.
template <bool W> __device__ int parse_line(const SamArgs& A, uint64_t k, const uint8_t* nib) {
    const unsigned lane = threadIdx.x & 31;
    const uint64_t s0 = A.ls[k];
    uint64_t n = A.ls[k + 1] - 1 - s0;
    const uint8_t* p = A.text + s0;
    if (n && p[n - 1] == '\r') n--;
    if (!n) return SE_EMPTY;
    uint64_t e[11];   // e[f]: the tab after mandatory field f (e[10]: end of QUAL)
    uint64_t x = 0;
#pragma unroll
    for (int f = 0; f < 11; f++) {
        e[f] = next_tab(p, x, n);
        if (f < 10 && e[f] == n) return SE_TABS;
        x = e[f] + 1;
    }
    const uint64_t lq = e[0];
    if (lq > 254) return SE_QNAME;
    int64_t flag, pos, mapq, pnext, tlen;
    if (!parse_dec(p + e[0] + 1, e[1] - e[0] - 1, false, 0, 65535, &flag)) return SE_FLAG;
    if (!parse_dec(p + e[2] + 1, e[3] - e[2] - 1, true, INT32_MIN, INT32_MAX, &pos)) return SE_POS;
    if (!parse_dec(p + e[3] + 1, e[4] - e[3] - 1, false, 0, 255, &mapq)) return SE_MAPQ;
    if (!parse_dec(p + e[6] + 1, e[7] - e[6] - 1, true, INT32_MIN, INT32_MAX, &pnext)) return SE_PNEXT;
    if (!parse_dec(p + e[7] + 1, e[8] - e[7] - 1, true, INT32_MIN, INT32_MAX, &tlen)) return SE_TLEN;
    const int32_t refid = refid_of(A.dict, p + e[1] + 1, e[2] - e[1] - 1);
    const bool rnext_eq = e[6] - e[5] - 1 == 1 && p[e[5] + 1] == '=';
    const int32_t nref = rnext_eq ? refid : refid_of(A.dict, p + e[5] + 1, e[6] - e[5] - 1);
    // names the record cannot give back to elp_fetch_sam: an RNAME that is neither "*" nor an @SQ name, likewise an RNEXT other than
    // "=", and RNEXT "=" with an RNAME that resolves to -1 ("*" included; the reference's SAM -> SAM text keeps the '=')
    const bool rname_star = e[2] - e[1] - 1 == 1 && p[e[1] + 1] == '*', rnext_star = e[6] - e[5] - 1 == 1 && p[e[5] + 1] == '*';
    const bool lost = (refid < 0 && !rname_star) || (!rnext_eq && !rnext_star && nref < 0) || (rnext_eq && refid < 0);
    const uint64_t L = e[9] - e[8] - 1;
    if (e[10] - e[9] - 1 != L) return SE_QUAL;
    uint8_t* o = W ? A.out + A.rec_off[k] : nullptr;
    const uint64_t ocig = 36 + lq + 1;
    // CIGAR (ScanCigarString, sam/sam-types.go:672-740): "*" -> no operations, adjacent equal operations merge
    uint32_t ncig = 0, refspan = 0;                                          // refspan: int32 arithmetic of bin(), as unsigned
    {
        const uint64_t c1 = e[5];
        uint64_t i = e[4] + 1;
        if (c1 - i == 1 && p[i] == '*') i = c1;
        int cur = -1; uint64_t cl = 0;
        for (;;) {
            const bool done = i >= c1;
            int op = -1; uint64_t ln = 0;
            if (!done) {
                uint64_t j = i;
                for (; j < c1 && p[j] >= '0' && p[j] <= '9'; j++) if (ln <= (uint64_t)INT32_MAX) ln = ln * 10 + (p[j] - '0');
                if (j == i || j == c1 || ln > (uint64_t)INT32_MAX) return SE_CIGAR;
                op = cigar_code(p[j]);
                if (op < 0) return SE_CIGAR;
                i = j + 1;
            }
            if (cur >= 0 && (done || op != cur)) {                           // flush the merged operation
                if (cl >= (1u << 28)) return SE_CIGAR_LEN;
                if (ncig < 65536) { if (W) put<W>(o + ocig + 4ull * ncig, (uint32_t)(cl << 4) | (uint32_t)cur, 4); }
                if (cur == 0 || cur == 2 || cur == 3 || cur == 7 || cur == 8) refspan += (uint32_t)cl;
                ncig++;
            }
            if (done) break;
            if (op == cur) cl += ln; else { cur = op; cl = ln; }
        }
    }
    if (ncig > 65535) return SE_CIGAR_LIMIT;
    const uint64_t oseq = ocig + 4ull * ncig, oqual = oseq + ((L + 1) >> 1), otag = oqual + L;
    // optional fields: tab-separated "TG:T:value"; a repeated tag keeps the position of its first occurrence and the value of its
    // last (SmallMap.Set, utils/small-map.go:59-67); every occurrence must parse
    uint64_t tsz = 0;
    for (uint64_t a = e[10] + 1; a < n;) {
        const uint64_t b = next_tab(p, a, n);
        if (b - a < 5 || p[a] == ':' || p[a + 1] == ':' || p[a + 2] != ':' || p[a + 4] != ':') return SE_TAG;
        bool dup = false;
        for (uint64_t y = e[10] + 1; y < a && !dup; y = next_tab(p, y, n) + 1) dup = p[y] == p[a] && p[y + 1] == p[a + 1];
        uint64_t sz = 0;
        if (dup) {
            const int r = tag_value<false>(A, p, a, b, nullptr, 0, s0, k, false, &sz);
            if (r) return r;
        } else {
            uint64_t la = a, lb = b;
            for (uint64_t y = b + 1; y < n;) {
                const uint64_t z = next_tab(p, y, n);
                if (z - y >= 3 && p[y] == p[a] && p[y + 1] == p[a + 1] && p[y + 2] == ':') { la = y; lb = z; }
                y = z + 1;
            }
            if (la != a) { const int r = tag_value<false>(A, p, a, b, nullptr, 0, s0, k, false, &sz); if (r) return r; }
            if (la + 5 > lb || p[la + 4] != ':') return SE_TAG;
            const int r = tag_value<W>(A, p, la, lb, W ? o + otag + tsz : nullptr, W ? A.rec_off[k] + otag + tsz : 0, s0, k, true, &sz);
            if (r) return r;
            tsz += sz;
        }
        a = b + 1;
    }
    const uint64_t rec = otag + tsz;
    if (rec >= (1ull << 31)) return SE_RECORD_LIMIT;
    if (!W) { if (lane == 0) { A.len[k] = (uint32_t)rec; A.lost[k] = lost; if (lost) atomicAdd(A.small + 2, 1ull); } return 0; }
    // bin() (bam-files.go:443-468) in int32 arithmetic; an unmapped read spans [beg, beg]
    const int32_t beg = (int32_t)((uint32_t)pos - 1u);
    const int32_t end = (flag & 4) ? beg : (int32_t)((uint32_t)beg + refspan - 1u);
    uint32_t bin = 0;
    if (beg >> 14 == end >> 14) bin = 4681u + (uint32_t)(beg >> 14);
    else if (beg >> 17 == end >> 17) bin = 585u + (uint32_t)(beg >> 17);
    else if (beg >> 20 == end >> 20) bin = 73u + (uint32_t)(beg >> 20);
    else if (beg >> 23 == end >> 23) bin = 9u + (uint32_t)(beg >> 23);
    else if (beg >> 26 == end >> 26) bin = 1u + (uint32_t)(beg >> 26);
    const int32_t rid = (refid < 0 && !rname_star) ? A.unreached_ref : refid;
    put<W>(o, (uint32_t)(rec - 4), 4); put<W>(o + 4, (uint32_t)rid, 4); put<W>(o + 8, (uint32_t)beg, 4);
    put<W>(o + 12, (uint32_t)(lq + 1) | ((uint32_t)mapq << 8) | ((bin & 0xffff) << 16), 4);
    put<W>(o + 16, ncig | ((uint32_t)flag << 16), 4); put<W>(o + 20, (uint32_t)L, 4); put<W>(o + 24, (uint32_t)nref, 4);
    put<W>(o + 28, (uint32_t)pnext - 1u, 4); put<W>(o + 32, (uint32_t)tlen, 4);
    for (uint64_t j = lane; j < lq; j += 32) o[36 + j] = p[j];
    put<W>(o + 36 + lq, 0, 1);
    const uint8_t* sq = p + e[8] + 1;
    for (uint64_t j = lane; j < (L + 1) >> 1; j += 32) o[oseq + j] = (uint8_t)((nib[sq[2 * j]] << 4) | (2 * j + 1 < L ? nib[sq[2 * j + 1]] : 0));
    const uint8_t* qu = p + e[9] + 1;
    for (uint64_t j = lane; j < L; j += 32) o[oqual + j] = (uint8_t)(qu[j] - 33);
    return 0;
}

template <bool W> __global__ void __launch_bounds__(256) sam_line_kernel(SamArgs A) {
    __shared__ uint8_t nib[256];   // baseToNibble (sam/sam-types.go:227-236): "=ACMGRSVTWYHKDBN", anything else 15
    for (int t = threadIdx.x; t < 256; t += blockDim.x) {
        const char* s = "=ACMGRSVTWYHKDBN";
        uint8_t v = 15;
        for (int q = 0; q < 16; q++) if ((uint8_t)s[q] == t) v = (uint8_t)q;
        nib[t] = v;
    }
    __syncthreads();
    const uint64_t k = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (k >= A.n_lines) return;
    const int r = parse_line<W>(A, k, nib);
    if (r && (threadIdx.x & 31) == 0) {
        atomicMin(A.small, ((unsigned long long)k << 8) | (unsigned long long)r);
        if (!W) A.len[k] = 0;
    }
}

// lost-name lines among the records the ingest filters kept: kept[i] is the start of a kept record, line_off the starts of all lines
__global__ void __launch_bounds__(256) sam_lost_kept_kernel(uint64_t nk, const uint64_t* __restrict__ kept, const uint64_t* __restrict__ line_off, uint64_t nl,
                                                             const uint8_t* __restrict__ lost, unsigned long long* __restrict__ cnt) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= nk) return;
    uint64_t lo = 0, hi = nl;
    while (hi - lo > 1) { const uint64_t mid = (lo + hi) >> 1; if (line_off[mid] <= kept[i]) lo = mid; else hi = mid; }
    if (lost[lo]) atomicAdd(cnt, 1ull);
}

__global__ void __launch_bounds__(256) sam_fpatch_kernel(uint64_t n, const uint64_t* __restrict__ off, const uint32_t* __restrict__ bits, uint8_t* __restrict__ out) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) for (int b = 0; b < 4; b++) out[off[i] + b] = (uint8_t)(bits[i] >> (8 * b));
}

// the RNAME / RNEXT dictionary (elp_config's names, or the input name table of elp_set_input_dictionary) and the error words, uploaded
// once per context and setting
int sam_tables(elp_ctx* c) {
    if (!c->sam) c->sam.reset(new SamState());
    CUDA_TRY(c, c->sam->d_small.fit(3));
    return c->dict_mode ? name_dict_build(c, c->in_dict, c->in_tab) : name_dict_upload(c);
}

// strconv.ParseFloat(s, 32) for a decimal the device already checked: strtof rounds correctly; only overflow is an error in Go
bool host_f32(const uint8_t* s, uint32_t n, uint32_t* bits) {
    static const locale_t C_LOCALE = newlocale(LC_ALL_MASK, "C", (locale_t)0);   // '.' whatever the process locale is
    std::string t(reinterpret_cast<const char*>(s), n);
    const float f = strtof_l(t.c_str(), nullptr, C_LOCALE);
    if (std::isinf(f)) return false;
    memcpy(bits, &f, 4);
    return true;
}

}  // namespace

extern "C" int elp_append_sam(elp_ctx* c, const char* text, uint64_t n_bytes) {
    if (!c || (!text && n_bytes)) return ELP_EINVAL;
    cudaSetDevice(c->device);
    std::lock_guard<std::mutex> lk(c->append_mu);
    if (c->sorted) return c->fail(E_STATE, "elp_append_sam after elp_sort_markdup (call elp_reset first)");
    TRY(relabel_check_selected(c, "elp_append_sam"));
    if (c->bgzf_open) return c->fail(E_STATE, "elp_append_sam while a BGZF file is open (elp_append_bgzf_end first)");
    if (c->n_contigs > 0 && !c->has_contig_names) return c->fail(E_INVAL, "elp_append_sam: the context was created without elp_config.contig_names, so RNAME / RNEXT cannot be resolved");
    if (n_bytes == 0) return ELP_OK;
    TRY(sam_tables(c));
    SamState& S = *c->sam;
    cudaStream_t s = c->stream;
    const uint8_t* h = reinterpret_cast<const uint8_t*>(text);
    const uint64_t n_chunks = (n_bytes + SAM_CHUNK - 1) / SAM_CHUNK, padded = n_chunks * SAM_CHUNK + 64;
    TRY(grow(c, S.text, padded, 0)); TRY(grow(c, S.cnt, n_chunks + 8, 0)); TRY(grow(c, S.cnt_off, n_chunks + 2, 0));
    CUDA_TRY(c, cudaMemcpyAsync(S.text.p, h, n_bytes, cudaMemcpyHostToDevice, s));
    CUDA_TRY(c, cudaMemsetAsync(S.text.p + n_bytes, 0, padded - n_bytes, s));
    // line finder
    c->begin("sam_lines", (double)n_bytes);
    sam_count_kernel<<<nblk(n_chunks, 256), 256, 0, s>>>(S.text.p, n_chunks, S.cnt.p);
    c->end(); LAUNCH_CHECK(c);
    TRY(exclusive_scan_u32_to_u64(c, S.cnt.p, S.cnt_off.p, n_chunks));
    uint64_t n_nl = 0;
    CUDA_TRY(c, cudaMemcpyAsync(&n_nl, S.cnt_off.p + n_chunks, 8, cudaMemcpyDeviceToHost, s));
    CUDA_TRY(c, cudaStreamSynchronize(s));
    const bool open_end = h[n_bytes - 1] != '\n';
    const uint64_t nl = n_nl + (open_end ? 1 : 0);   // lines
    if (c->n + nl >= (1ull << 32)) return c->fail(E_LIMIT, "more than 2^32-1 reads in one context");
    TRY(grow(c, S.ls, nl + 2, 0)); TRY(grow(c, S.len, nl + 8, 0)); TRY(grow(c, S.lost, nl + 8, 0)); TRY(grow(c, c->bam_off, nl + 2, 0));
    CUDA_TRY(c, cudaMemsetAsync(S.ls.p, 0, 8, s));
    c->begin("sam_lines", (double)n_bytes + 8.0 * (double)n_nl);
    sam_lines_kernel<<<nblk(n_chunks, 256), 256, 0, s>>>(S.text.p, n_chunks, S.cnt_off.p, S.ls.p);
    c->end(); LAUNCH_CHECK(c);
    S.h_last = n_bytes + 1;                                  // a virtual '\n' just past the text
    if (open_end) CUDA_TRY(c, cudaMemcpyAsync(S.ls.p + nl, &S.h_last, 8, cudaMemcpyHostToDevice, s));
    // measure: validate every line and size its record
    SamArgs A{};
    A.text = S.text.p; A.ls = S.ls.p; A.n_lines = nl;
    A.dict = c->dict_mode ? c->in_dict.view() : c->names.view();
    A.unreached_ref = (c->dict_mode & ELP_DICT_REPLACE) ? (int32_t)c->in_tab.size() : -1;
    A.len = S.len.p; A.lost = S.lost.p; A.rec_off = c->bam_off.p; A.small = S.d_small.p;
    CUDA_TRY(c, cudaMemsetAsync(S.d_small.p, 0xff, 8, s)); CUDA_TRY(c, cudaMemsetAsync(S.d_small.p + 1, 0, 16, s));
    c->begin("sam_measure", (double)n_bytes);
    sam_line_kernel<false><<<nblk(nl * 32, 256), 256, 0, s>>>(A);
    c->end(); LAUNCH_CHECK(c);
    TRY(exclusive_scan_u32_to_u64(c, S.len.p, c->bam_off.p, nl));
    unsigned long long small[3]; uint64_t total = 0;
    CUDA_TRY(c, cudaMemcpyAsync(small, S.d_small.p, 24, cudaMemcpyDeviceToHost, s));
    CUDA_TRY(c, cudaMemcpyAsync(&total, c->bam_off.p + nl, 8, cudaMemcpyDeviceToHost, s));
    CUDA_TRY(c, cudaStreamSynchronize(s));
    if (small[0] != ~0ull) {
        const uint32_t code = (uint32_t)(small[0] & 0xff);
        return c->fail(code >= SE_CIGAR_LIMIT ? E_LIMIT : E_SAM, "elp_append_sam: line %llu (0-based, within the call): %s", (unsigned long long)(small[0] >> 8), sam_err_text(code));
    }
    const uint64_t n_slow = small[1];
    // emit: the same parser writes every record at its offset
    TRY(grow(c, c->bam_raw, total + 64, 0)); TRY(grow(c, S.slow, n_slow + 1, 0));
    A.out = c->bam_raw.p; A.slow = S.slow.p;
    CUDA_TRY(c, cudaMemsetAsync(S.d_small.p + 1, 0, 8, s));
    c->begin("sam_emit", (double)n_bytes + (double)total);
    sam_line_kernel<true><<<nblk(nl * 32, 256), 256, 0, s>>>(A);
    c->end(); LAUNCH_CHECK(c);
    if (n_slow) {   // float values outside the device's exact range: strtof on the host, patched into the staged records
        std::vector<SlowF> sl(n_slow);
        CUDA_TRY(c, cudaMemcpyAsync(sl.data(), S.slow.p, n_slow * sizeof(SlowF), cudaMemcpyDeviceToHost, s));
        CUDA_TRY(c, cudaStreamSynchronize(s));
        std::vector<uint64_t> po(n_slow); std::vector<uint32_t> pb(n_slow);
        uint64_t bad = ~0ull;
        for (uint64_t i = 0; i < n_slow; i++) {
            po[i] = sl[i].out_off;
            if (!host_f32(h + sl[i].text_off, sl[i].len, &pb[i])) bad = std::min<uint64_t>(bad, sl[i].line);
        }
        if (bad != ~0ull) return c->fail(E_SAM, "elp_append_sam: line %llu (0-based, within the call): %s", (unsigned long long)bad, sam_err_text(SE_FLOAT_RANGE));
        TRY(grow(c, S.patch_off, n_slow, 0)); TRY(grow(c, S.patch_bits, n_slow, 0));
        CUDA_TRY(c, cudaMemcpyAsync(S.patch_off.p, po.data(), n_slow * 8, cudaMemcpyHostToDevice, s));
        CUDA_TRY(c, cudaMemcpyAsync(S.patch_bits.p, pb.data(), n_slow * 4, cudaMemcpyHostToDevice, s));
        c->begin("sam_fpatch", 12.0 * (double)n_slow);
        sam_fpatch_kernel<<<nblk(n_slow, 256), 256, 0, s>>>(n_slow, S.patch_off.p, S.patch_bits.p, c->bam_raw.p);
        c->end(); LAUNCH_CHECK(c);
        CUDA_TRY(c, cudaStreamSynchronize(s));   // (po / pb are pageable host memory)
    }
    const uint64_t n0 = c->n;
    TRY(bam_ingest_core(c, total, nl, true));
    uint64_t lost = small[2];
    if (lost && ingest_keep_on(c)) {   // count only the lines the filters kept (bam_start: their record starts)
        const uint64_t nk = c->n - n0;
        CUDA_TRY(c, cudaMemsetAsync(S.d_small.p + 2, 0, 8, s));
        if (nk) { sam_lost_kept_kernel<<<nblk(nk, 256), 256, 0, s>>>(nk, c->bam_start.p, c->bam_off.p, nl, S.lost.p, S.d_small.p + 2); c->launches++; LAUNCH_CHECK(c); }
        CUDA_TRY(c, cudaMemcpyAsync(&lost, S.d_small.p + 2, 8, cudaMemcpyDeviceToHost, s));
        CUDA_TRY(c, cudaStreamSynchronize(s));
    }
    c->n_sam_lost_names += lost;
    return ELP_OK;
}
