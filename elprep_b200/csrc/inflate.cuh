// inflate.cuh -- the DEFLATE decoder (RFC 1951) and the CRC-32 of bgzf_inflate.cu, written once for a team of lanes: on the device the
// team is one warp (every lane decodes the same symbols from the same bit buffer, so control flow stays warp-uniform; table builds and
// copies are split over the lanes), on the host it is one thread.  tests/c/inflate_check.cpp compiles this very file with g++ and
// compares it stream by stream with zlib.
//
// Acceptance is zlib's: inflateInit2(-15) + inflate(Z_FINISH) into exactly isize bytes must end in Z_STREAM_END with isize bytes out
// (elp_bgzf_inflate).  So: block type 3, HLIT > 286, HDIST > 30, an over-subscribed set, an incomplete set (except a lone code of
// length 1 in the literal/length or distance set), repeat code 16 first, a repeat past HLIT + HDIST, no code for symbol 256,
// literal/length symbols 286 and 287 and distance codes 30 and 31 of the fixed code, a distance past the start of the output, a stored
// block whose NLEN is not ~LEN, output beyond isize, fewer than isize bytes, and a stream that needs bits past the end of its input are
// all errors; bytes after the final block are ignored, as zlib ignores them.
//
// Bounds hold by construction: input is only read below n_in (bytes past it read as zero and are counted as consumed, which fails the
// stream), output is only written below isize, and every loop either writes output or consumes at least 3 bits.
#pragma once
#include <cstdint>

#ifdef __CUDACC__
#define INF_HD __host__ __device__ __forceinline__
#else
#define INF_HD inline
#endif

namespace dfl {

enum Status : uint32_t {
    OK = 0, E_TRUNC = 1, E_BTYPE = 2, E_STORED = 3, E_COUNTS = 4, E_CLEN_SET = 5, E_REPEAT = 6, E_LEN_SET = 7, E_DIST_SET = 8,
    E_NO_EOB = 9, E_CODE = 10, E_DCODE = 11, E_FAR = 12, E_OVER = 13, E_SHORT = 14, E_CRC = 15,
};
inline const char* status_text(uint32_t s) {
    switch (s) {
        case E_TRUNC: return "DEFLATE stream runs past the end of the block";
        case E_BTYPE: return "invalid block type";
        case E_STORED: return "invalid stored block lengths";
        case E_COUNTS: return "too many length or distance symbols";
        case E_CLEN_SET: return "invalid code lengths set";
        case E_REPEAT: return "invalid bit length repeat";
        case E_LEN_SET: return "invalid literal/lengths set";
        case E_DIST_SET: return "invalid distances set";
        case E_NO_EOB: return "invalid code -- missing end-of-block";
        case E_CODE: return "invalid literal/length code";
        case E_DCODE: return "invalid distance code";
        case E_FAR: return "invalid distance too far back";
        case E_OVER: return "more output than ISIZE";
        case E_SHORT: return "less output than ISIZE";
        case E_CRC: return "CRC-32 mismatch";
        default: return "ok";
    }
}

// one thread as a team of one (host)
struct Serial {
    static constexpr unsigned size = 1;
    unsigned lane = 0;
    INF_HD void sync() const {}
};

constexpr int LBITS = 10, DBITS = 8, CBITS = 7, MAXBITS = 15;
constexpr uint16_t LONG = 0xffff;   // primary entry: a prefix of a code longer than the primary index

// per-decoder scratch (shared memory on the device): a primary look-up table per code, indexed by the next pbits bits of the stream,
// entry = symbol | length << 9 (0: no code starts with these bits); codes longer than pbits go through the canonical walk of decode_canon
// over the per-length counts and the symbols in code order.
struct Tables {
    uint16_t lprim[1 << LBITS];
    uint16_t dprim[1 << DBITS];
    uint16_t cprim[1 << CBITS];
    uint16_t lsym[288], dsym[32], csym[19];
    uint16_t lcnt[16], dcnt[16], ccnt[16];
    uint8_t lens[288 + 32];
    uint8_t clens[20];
};

// canonical decode of the next bits (LSB first) over codes of at most maxbits bits; returns the code length, 0 if none matches
INF_HD int decode_canon(uint32_t bits, int maxbits, const uint16_t* cnt, const uint16_t* sym, int* out) {
    int code = 0, first = 0, index = 0;
    for (int len = 1; len <= maxbits; len++) {
        code |= (int)((bits >> (len - 1)) & 1u);
        const int count = cnt[len];
        if (code < first + count) { *out = sym[index + (code - first)]; return len; }
        index += count; first += count; first <<= 1; code <<= 1;
    }
    return 0;
}

// table of n code lengths (inflate_table of zlib: kind 0 = the code-length code, which must be complete; kind 1 = literal/length or
// distance code, incomplete only as a single code of length 1).  An empty set builds and fails on first use.
template <class Team>
INF_HD uint32_t build(const Team& t, const uint8_t* len, int n, uint16_t* cnt, uint16_t* sym, uint16_t* prim, int pbits, int kind, uint32_t err) {
    for (unsigned L = t.lane; L < 16; L += t.size) {
        uint16_t k = 0;
        for (int s = 0; s < n; s++) k += len[s] == L;
        cnt[L] = k;
    }
    t.sync();
    int left = 1, maxl = 0;
    for (int L = 1; L <= MAXBITS; L++) {
        left <<= 1; left -= cnt[L];
        if (left < 0) return err;                                   // over-subscribed
        if (cnt[L]) maxl = L;
    }
    if (maxl && left > 0 && (kind == 0 || maxl != 1)) return err;   // incomplete
    for (unsigned L = t.lane; L < 16; L += t.size) {
        if (L == 0) continue;
        int o = 0;
        for (unsigned k = 1; k < L; k++) o += cnt[k];
        for (int s = 0; s < n; s++) if (len[s] == L) sym[o++] = (uint16_t)s;
    }
    t.sync();
    for (unsigned i = t.lane; i < (1u << pbits); i += t.size) {
        int s = 0;
        const int l = maxl ? decode_canon(i, pbits, cnt, sym, &s) : 0;
        prim[i] = l ? (uint16_t)(s | (l << 9)) : (maxl > pbits ? LONG : (uint16_t)0);
    }
    t.sync();
    return OK;
}

// LSB-first bit reader over in[0, n); bytes past n read as zero and count as consumed
struct Bits {
    const uint8_t* in; uint32_t n, pos; uint64_t buf; uint32_t cnt;
    INF_HD void refill() { while (cnt <= 56) { buf |= (uint64_t)(pos < n ? in[pos] : 0u) << cnt; pos++; cnt += 8; } }
    INF_HD uint32_t peek(int k) const { return (uint32_t)(buf & ((1ull << k) - 1)); }
    INF_HD void drop(int k) { buf >>= k; cnt -= k; }
    INF_HD uint32_t get(int k) { const uint32_t v = peek(k); drop(k); return v; }
    INF_HD bool overrun() const { return (uint64_t)pos * 8 - cnt > (uint64_t)n * 8; }
};

// one symbol of a code (needs MAXBITS bits in the buffer); -1 if no code matches
INF_HD int decode_sym(Bits& b, const uint16_t* prim, int pbits, const uint16_t* cnt, const uint16_t* sym) {
    const uint16_t e = prim[b.peek(pbits)];
    int s = -1, l = 0;
    if (e == LONG) l = decode_canon(b.peek(MAXBITS), MAXBITS, cnt, sym, &s);
    else if (e) { s = e & 511; l = e >> 9; }
    if (!l) return -1;
    b.drop(l);
    return s;
}

// length base / extra bits of literal/length symbol 257 + s (s < 29) and of distance code d (d < 30), RFC 1951 3.2.5
INF_HD uint32_t len_extra(int s) { return (s < 8 || s == 28) ? 0u : (uint32_t)((s - 4) >> 2); }
INF_HD uint32_t len_base(int s) { return s < 8 ? (uint32_t)s + 3 : (s == 28 ? 258u : ((4u + (s & 3)) << len_extra(s)) + 3); }
INF_HD uint32_t dist_extra(int d) { return d < 4 ? 0u : (uint32_t)((d - 2) >> 1); }
INF_HD uint32_t dist_base(int d) { return d < 4 ? (uint32_t)d + 1 : ((2u + (d & 1)) << dist_extra(d)) + 1; }

// inflate one raw DEFLATE stream in[0, n_in) into out[0, isize); returns a Status.  All lanes of the team call it with the same arguments.
template <class Team>
INF_HD uint32_t inflate_stream(const Team& t, Tables& T, const uint8_t* in, uint32_t n_in, uint8_t* out, uint32_t isize) {
    Bits b{in, n_in, 0, 0, 0};
    uint32_t opos = 0;
    for (;;) {
        b.refill();
        const uint32_t final_ = b.get(1), type = b.get(2);
        if (type == 0) {
            b.drop(b.cnt & 7);                                      // to a byte boundary
            const uint32_t len = b.get(16), nlen = b.get(16);
            if (len != (~nlen & 0xffffu)) return b.overrun() ? E_TRUNC : E_STORED;
            const uint32_t at = b.pos - b.cnt / 8;                   // first byte of the stored data
            if ((uint64_t)at + len > n_in) return E_TRUNC;
            if (opos + len > isize) return E_OVER;
            for (uint32_t i = t.lane; i < len; i += t.size) out[opos + i] = in[at + i];
            opos += len;
            b.pos = at + len; b.buf = 0; b.cnt = 0;
        } else if (type == 1 || type == 2) {
            if (type == 1) {
                for (unsigned i = t.lane; i < 320; i += t.size) T.lens[i] = i < 144 ? 8 : (i < 256 ? 9 : (i < 280 ? 7 : (i < 288 ? 8 : 5)));
                t.sync();
                build(t, T.lens, 288, T.lcnt, T.lsym, T.lprim, LBITS, 1, E_LEN_SET);
                build(t, T.lens + 288, 32, T.dcnt, T.dsym, T.dprim, DBITS, 1, E_DIST_SET);
            } else {
                const uint32_t hlit = b.get(5) + 257, hdist = b.get(5) + 1, hclen = b.get(4) + 4;
                if (hlit > 286 || hdist > 30) return E_COUNTS;
                b.refill();
                const uint8_t order[19] = {16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15};
                uint32_t cl[19];
                for (int i = 0; i < 19; i++) cl[i] = 0;
                for (uint32_t i = 0; i < hclen; i++) cl[order[i]] = b.get(3);   // 19 * 3 = 57 bits: the buffer holds them after refill
                t.sync();
                for (unsigned i = t.lane; i < 19; i += t.size) T.clens[i] = (uint8_t)cl[i];
                t.sync();
                uint32_t rc = build(t, T.clens, 19, T.ccnt, T.csym, T.cprim, CBITS, 0, E_CLEN_SET);
                if (rc) return rc;
                const uint32_t total = hlit + hdist;
                uint32_t i = 0, last = 0;
                while (i < total) {
                    b.refill();
                    const int s = decode_sym(b, T.cprim, CBITS, T.ccnt, T.csym);
                    if (s < 0) return b.overrun() ? E_TRUNC : E_CLEN_SET;
                    uint32_t v, rep;
                    if (s < 16) { v = (uint32_t)s; rep = 1; last = v; }
                    else if (s == 16) { if (i == 0) return E_REPEAT; v = last; rep = 3 + b.get(2); }
                    else if (s == 17) { v = 0; rep = 3 + b.get(3); last = 0; }
                    else { v = 0; rep = 11 + b.get(7); last = 0; }
                    if (i + rep > total) return E_REPEAT;
                    for (uint32_t k = t.lane; k < rep; k += t.size) T.lens[i + k] = (uint8_t)v;
                    i += rep;
                }
                if (b.overrun()) return E_TRUNC;
                t.sync();
                if (T.lens[256] == 0) return E_NO_EOB;
                rc = build(t, T.lens, (int)hlit, T.lcnt, T.lsym, T.lprim, LBITS, 1, E_LEN_SET);
                if (rc) return rc;
                rc = build(t, T.lens + hlit, (int)hdist, T.dcnt, T.dsym, T.dprim, DBITS, 1, E_DIST_SET);
                if (rc) return rc;
            }
            for (;;) {
                b.refill();                                          // 57+ bits: code 15 + extra 5 + distance code 15 + extra 13
                const int s = decode_sym(b, T.lprim, LBITS, T.lcnt, T.lsym);
                if (s < 0) return b.overrun() ? E_TRUNC : E_CODE;
                if (s < 256) {
                    if (opos >= isize) return b.overrun() ? E_TRUNC : E_OVER;
                    if (t.lane == 0) out[opos] = (uint8_t)s;
                    opos++;
                    continue;
                }
                if (s == 256) break;
                if (s >= 286) return E_CODE;
                const int ls = s - 257;
                const uint32_t len = len_base(ls) + b.get((int)len_extra(ls));
                const int ds = decode_sym(b, T.dprim, DBITS, T.dcnt, T.dsym);
                if (ds < 0 || ds >= 30) return b.overrun() ? E_TRUNC : E_DCODE;
                const uint32_t dist = dist_base(ds) + b.get((int)dist_extra(ds));
                if (b.overrun()) return E_TRUNC;
                if (dist > opos) return E_FAR;
                if (opos + len > isize) return E_OVER;
                t.sync();                                            // literals and copies of other lanes are visible
                uint8_t* o = out + opos;
                if (dist >= len) { for (uint32_t k = t.lane; k < len; k += t.size) o[k] = o[(int64_t)k - (int64_t)dist]; }
                else { for (uint32_t k = t.lane; k < len; k += t.size) o[k] = o[(int64_t)(k % dist) - (int64_t)dist]; }   // overlapping: byte k from pos - d + (k mod d)
                opos += len;
            }
            if (b.overrun()) return E_TRUNC;
        } else {
            return b.overrun() ? E_TRUNC : E_BTYPE;
        }
        if (b.overrun()) return E_TRUNC;
        if (final_) break;
    }
    t.sync();
    return opos == isize ? (uint32_t)OK : (uint32_t)E_SHORT;
}

// ---- CRC-32 (the gzip polynomial, reflected) ----
INF_HD uint32_t crc_table_entry(uint32_t i) { uint32_t c = i; for (int k = 0; k < 8; k++) c = (c & 1) ? (c >> 1) ^ 0xedb88320u : c >> 1; return c; }
// crc32 of n bytes continuing crc (as zlib's crc32(crc, p, n)); tab: the 256 entries of crc_table_entry
INF_HD uint32_t crc_bytes(const uint32_t* tab, uint32_t crc, const uint8_t* p, uint32_t n) {
    uint32_t c = ~crc;
    for (uint32_t i = 0; i < n; i++) c = tab[(c ^ p[i]) & 255u] ^ (c >> 8);
    return ~c;
}
// a(x) * b(x) mod p(x), reflected (zlib multmodp)
INF_HD uint32_t multmodp(uint32_t a, uint32_t b) {
    uint32_t m = 1u << 31, p = 0;
    for (;;) {
        if (a & m) { p ^= b; if ((a & (m - 1)) == 0) break; }
        m >>= 1;
        b = (b & 1) ? (b >> 1) ^ 0xedb88320u : b >> 1;
    }
    return p;
}
// x2n[k] = x^(2^k) mod p(x), k < 32
INF_HD void x2n_table(uint32_t* x2n) { uint32_t p = 1u << 30; x2n[0] = p; for (int k = 1; k < 32; k++) x2n[k] = p = multmodp(p, p); }
// the crc32_combine shift: crc of A followed by n_bytes more bytes contributes this to the crc of the whole (zlib crc32_combine)
INF_HD uint32_t crc_shift(const uint32_t* x2n, uint32_t crc, uint64_t n_bytes) {
    uint32_t p = 1u << 31;
    for (unsigned k = 3; n_bytes; n_bytes >>= 1, k++) if (n_bytes & 1) p = multmodp(x2n[k & 31], p);
    return multmodp(p, crc);
}

#ifdef __CUDACC__
// crc32 of p[0, n) by one warp: lane k takes the k-th 1/32 slice, shifts its crc past the bytes after the slice, and the slices fold by XOR
// (ctab: crc_table_entry, x2n: x2n_table); every lane returns the whole crc
__device__ __forceinline__ uint32_t warp_crc(const uint32_t* ctab, const uint32_t* x2n, const uint8_t* p, uint32_t n, unsigned lane) {
    const uint32_t chunk = (n + 31) / 32, a = min(n, lane * chunk), e = min(n, a + chunk);
    uint32_t v = crc_shift(x2n, crc_bytes(ctab, 0, p + a, e - a), n - e);
    for (int o = 16; o; o >>= 1) v ^= __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
#endif

}  // namespace dfl
