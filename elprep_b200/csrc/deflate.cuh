// deflate.cuh -- the DEFLATE encoder (RFC 1951) of bgzf_deflate.cu, written once for a team of lanes, as inflate.cuh is: on the device the
// team is one CTA per BGZF block (the hash chain is built by its first warp, everything else is split over all lanes), on the host it is
// one thread (SerialEnc).  tests/c/deflate_check.cpp compiles this very file with g++ and checks it against zlib and against inflate.cuh.
//
// One call encodes n <= 65535 bytes as one final DEFLATE block: dynamic Huffman codes (BTYPE 2), or a stored block (BTYPE 0) when that is
// smaller.  The stages, each a pure function of the input bytes (so the bytes out never depend on the team size or on timing):
//   chain    prev[p] = the nearest q < p whose 3-byte hash equals p's (NIL if none).  Built in chunks of the chain team's size over a head
//            table; within a chunk, lanes with the same hash are grouped (__match_any_sync on the device), and each lane links to the
//            nearest lower lane of its group or else to the head; the highest lane of a group then updates the head.
//   matches  match[p] = the longest match at p over at most CHAIN links of the chain (distance <= 32768, length 3..258, the nearest
//            of equal lengths; a length-3 match farther than TOO_FAR bytes is dropped, as zlib's lazy levels drop it).
//   parse    one-step lazy: next(p) = p + 1 when p has no match or p + 1 has a longer one, else p + the match length.  The parse is the
//            chain 0 -> next(0) -> ... ; it is found without a serial walk of the block: each lane walks its segment of the block from a
//            guessed entry (the segment's first byte) to its exit (the first parse position at or past the segment's end); repair rounds
//            re-walk every segment whose entry differs from its predecessor's exit until all agree.  Segment 0 starts right, and a
//            segment that starts at its right predecessor's exit is right, so the result is exactly the serial parse (bam_frame's
//            argument, DESIGN.md §3c).
//   codes    symbol histograms (integer adds: order-free), then code lengths on one lane: a two-queue Huffman build over the symbols
//            sorted by (frequency, symbol), limited to 15 bits (7 for the code-length code) by moving overflow down the Kraft sum and
//            re-assigning lengths in frequency order.  Every code is complete: a set of fewer than two symbols is padded with
//            zero-frequency symbols (0, then 1), as zlib pads, so no decoder (zlib, Go's compress/flate) can refuse it.
//   emit     per-segment bit counts, an exclusive scan, then each lane ORs its tokens' bits into the output words at its offset (disjoint
//            bits, so the order of the ORs does not matter).
#pragma once
#include <cstdint>
#include "inflate.cuh"

namespace dfl {

constexpr int HASH_BITS = 15;
constexpr uint32_t HASH_SIZE = 1u << HASH_BITS;
constexpr uint16_t NIL = 0xffff;
constexpr int CHAIN = 8;                      // chain links walked per position
constexpr uint32_t MAX_BLOCK = 65535;         // input bytes per call (one stored block holds at most this many)
constexpr uint32_t MIN_MATCH = 3, MAX_MATCH = 258, WINDOW = 32768, TOO_FAR = 4096;
constexpr unsigned MAX_TEAM = 256;            // segments of the parse: one per lane
constexpr int NLIT = 286, NDIST = 30, NCL = 19;

// the output of a block never exceeds the stored block: 5 bytes + n; the caller's word buffer holds stored_bytes(n) rounded up to words
INF_HD constexpr uint32_t stored_bytes(uint32_t n) { return n + 5; }

INF_HD int hibit(uint32_t x) {
#ifdef __CUDA_ARCH__
    return 31 - __clz((int)x);
#else
    return 31 - __builtin_clz(x);
#endif
}

// one thread as a team of one, and as its own chain team
struct SerialEnc : Serial {
    INF_HD bool any(bool b) const { return b; }
    INF_HD void or32(uint32_t* p, uint32_t v) const { *p |= v; }
    INF_HD void add32(uint32_t* p, uint32_t v) const { *p += v; }
    INF_HD bool chain_lane() const { return true; }
    INF_HD const SerialEnc& chain() const { return *this; }
    INF_HD uint32_t same(uint32_t) const { return 1u; }     // lanes of the chunk with the same hash (bit per lane)
    INF_HD uint32_t lt() const { return 0u; }               // lanes below this one
};

// per-position scratch (global memory on the device): 65536 entries each
struct EncScratch { uint16_t* prev; uint32_t* match; };   // match: length << 16 | distance (0: none)

// the Huffman build of one code (lane 0), alive only after the chain is built: it shares the head table's storage
struct HuffTmp {
    uint16_t sorted[NLIT];                    // used symbols by (frequency, symbol)
    uint16_t parent[2 * NLIT];
    uint32_t iw[NLIT];                        // weights of the internal nodes, in creation order
    uint8_t depth[2 * NLIT];
    uint8_t inset[NLIT];                      // symbol takes part in the code (used, or padding)
    uint32_t cnt[MAXBITS + 2];
};

struct EncShared {
    union { uint16_t head[HASH_SIZE]; HuffTmp h; } u;
    uint32_t lfreq[NLIT], dfreq[NDIST], cfreq[NCL];
    uint16_t lcode[NLIT], dcode[NDIST], ccode[NCL];
    uint8_t llen[NLIT], dlen[NDIST], clen[NCL];
    uint32_t seg_exit[MAX_TEAM], seg_bits[MAX_TEAM];
    uint16_t rle[NLIT + NDIST];               // the code-length symbols of the header: symbol | extra value << 5
    uint32_t n_rle, hlit, hdist, hclen, hdr_bits, total_bits, stored;
};

INF_HD uint32_t hash3(const uint8_t* p) { return (((uint32_t)p[0] | ((uint32_t)p[1] << 8) | ((uint32_t)p[2] << 16)) * 0x9E3779B1u) >> (32 - HASH_BITS); }

// length 3..258 -> literal/length symbol - 257 (0..28); distance 1..32768 -> distance code (0..29) (RFC 1951 3.2.5)
INF_HD int len_sym(uint32_t L) {
    if (L == MAX_MATCH) return 28;
    const uint32_t v = L - 3;
    if (v < 8) return (int)v;
    const int e = hibit(v) - 2;
    return 4 * e + (int)(v >> e);
}
INF_HD int dist_sym(uint32_t d) {
    const uint32_t v = d - 1;
    if (v < 4) return (int)v;
    const int e = hibit(v) - 1;
    return 2 * e + (int)(v >> e);
}

INF_HD uint32_t rev_bits(uint32_t code, int len) { uint32_t r = 0; for (int i = 0; i < len; i++) r |= ((code >> i) & 1u) << (len - 1 - i); return r; }

// OR n <= 48 bits of v into the LSB-first bit stream out at bit position pos
template <class Team>
INF_HD void put_bits(const Team& t, uint32_t* out, uint64_t pos, uint64_t v, int n) {
    while (n > 0) {
        const int sh = (int)(pos & 31), k = n < 32 - sh ? n : 32 - sh;
        t.or32(out + (pos >> 5), (uint32_t)(v & ((1ull << k) - 1)) << sh);
        v >>= k; pos += (uint64_t)k; n -= k;
    }
}

// ---- stage 1: the hash chain (the chain team only; head initialised to NIL) ----
template <class W>
INF_HD void build_chain(const W& w, uint16_t* head, uint16_t* prev, const uint8_t* in, uint32_t n) {
    for (uint32_t base = 0; base < n; base += W::size) {
        const uint32_t p = base + w.lane;
        const bool valid = p + MIN_MATCH <= n;
        const uint32_t h = valid ? hash3(in + p) : HASH_SIZE + w.lane;   // (lanes without a hash group alone)
        const uint32_t same = w.same(h), below = same & w.lt();
        uint16_t pv = NIL;
        if (valid) pv = below ? (uint16_t)(base + (uint32_t)hibit(below)) : head[h];
        w.sync();
        if (valid && (same >> w.lane) == 1u) head[h] = (uint16_t)p;       // the highest lane of its group
        if (p < n) prev[p] = pv;
        w.sync();
    }
}

// ---- stage 2: the longest match at p ----
INF_HD uint32_t find_match(const uint16_t* prev, const uint8_t* in, uint32_t n, uint32_t p) {
    if (p + MIN_MATCH > n) return 0;
    const uint32_t maxlen = n - p < MAX_MATCH ? n - p : MAX_MATCH;
    uint32_t best = 0, bd = 0, cand = prev[p];
    for (int k = 0; k < CHAIN && cand != NIL; k++) {
        const uint32_t d = p - cand;
        if (d > WINDOW) break;
        if (in[cand + best] == in[p + best]) {
            uint32_t l = 0;
            while (l < maxlen && in[cand + l] == in[p + l]) l++;
            if (l > best) { best = l; bd = d; if (l == maxlen) break; }
        }
        cand = prev[cand];
    }
    if (best < MIN_MATCH || (best == MIN_MATCH && bd > TOO_FAR)) return 0;
    return best << 16 | bd;
}

// ---- stage 3: the parse ----
INF_HD uint32_t next_pos(const uint32_t* match, uint32_t p, uint32_t n) {
    const uint32_t L = match[p] >> 16;
    if (L < MIN_MATCH) return p + 1;
    if (p + 1 < n && (match[p + 1] >> 16) > L) return p + 1;          // a longer match starts at the next byte: a literal here
    return p + L;
}
// first parse position at or past end, walking from e
INF_HD uint32_t walk(const uint32_t* match, uint32_t n, uint32_t e, uint32_t end) {
    uint32_t p = e;
    while (p < end) p = next_pos(match, p, n);
    return p;
}

// ---- stage 4: code lengths of one code over nsym symbols, at most limit bits, complete (all lanes call) ----
template <class Team>
INF_HD void build_lengths(const Team& t, HuffTmp& H, const uint32_t* freq, int nsym, int limit, uint8_t* len) {
    if (t.lane == 0) {
        int m = 0, only = -1;
        for (int s = 0; s < nsym; s++) { H.inset[s] = freq[s] != 0; if (freq[s]) { m++; only = s; } }
        if (m == 0) { H.inset[0] = H.inset[1] = 1; }
        else if (m == 1) H.inset[only == 0 ? 1 : 0] = 1;
    }
    t.sync();
    for (unsigned s = t.lane; s < (unsigned)nsym; s += Team::size) {   // rank of s by (frequency, symbol) among the code's symbols
        len[s] = 0;
        if (!H.inset[s]) continue;
        const uint64_t key = (uint64_t)freq[s] << 9 | s;
        int r = 0;
        for (int j = 0; j < nsym; j++) r += H.inset[j] && (((uint64_t)freq[j] << 9 | (uint32_t)j) < key);
        H.sorted[r] = (uint16_t)s;
    }
    t.sync();
    if (t.lane == 0) {
        int m = 0;
        for (int s = 0; s < nsym; s++) m += H.inset[s];
        // two-queue Huffman: leaves 0..m-1 in sorted order, internal nodes m..2m-2 in creation order (their weights never decrease)
        int li = 0, ii = 0;
        for (int j = 0; j < m - 1; j++) {
            uint32_t wsum = 0;
            for (int k = 0; k < 2; k++) {
                int node;
                if (li < m && (ii >= j || freq[H.sorted[li]] <= H.iw[ii])) { node = li; wsum += freq[H.sorted[li]]; li++; }
                else { node = m + ii; wsum += H.iw[ii]; ii++; }
                H.parent[node] = (uint16_t)(m + j);
            }
            H.iw[j] = wsum;
        }
        if (m >= 2) H.depth[2 * m - 2] = 0;                             // (the root; the padding above makes m >= 2)
        for (int v = 2 * m - 3; v >= 0; v--) H.depth[v] = (uint8_t)(H.depth[H.parent[v]] + 1);
        for (int L = 0; L <= MAXBITS + 1; L++) H.cnt[L] = 0;
        for (int k = 0; k < m; k++) H.cnt[H.depth[k] < limit ? H.depth[k] : limit]++;
        // clamping to limit over-subscribes the code: move leaves down until the Kraft sum is exactly 1
        uint32_t total = 0;
        for (int L = 1; L <= limit; L++) total += H.cnt[L] << (limit - L);
        while (total != (1u << limit)) {
            H.cnt[limit]--;
            for (int L = limit - 1; L > 0; L--) if (H.cnt[L]) { H.cnt[L]--; H.cnt[L + 1] += 2; break; }
            total--;
        }
        int k = 0;                                                      // the rarest symbols get the longest codes
        for (int L = limit; L > 0; L--) for (uint32_t c = 0; c < H.cnt[L]; c++) len[H.sorted[k++]] = (uint8_t)L;
    }
    t.sync();
}

// canonical codes (RFC 1951 3.2.2), bit-reversed for LSB-first output
INF_HD void canon_codes(const uint8_t* len, int nsym, uint16_t* code) {
    uint32_t cnt[MAXBITS + 1], next[MAXBITS + 1];
    for (int L = 0; L <= MAXBITS; L++) cnt[L] = 0;
    for (int s = 0; s < nsym; s++) cnt[len[s]]++;
    cnt[0] = 0;
    uint32_t c = 0;
    for (int L = 1; L <= MAXBITS; L++) { c = (c + cnt[L - 1]) << 1; next[L] = c; }
    for (int s = 0; s < nsym; s++) if (len[s]) code[s] = (uint16_t)rev_bits(next[len[s]]++, len[s]);
}

// bits of the token at p (next position q)
INF_HD uint32_t token_bits(const EncShared& S, const uint8_t* in, const uint32_t* match, uint32_t p, uint32_t q) {
    if (q == p + 1) return S.llen[in[p]];
    const uint32_t L = match[p] >> 16, d = match[p] & 0xffff;
    const int ls = len_sym(L), ds = dist_sym(d);
    return S.llen[257 + ls] + len_extra(ls) + S.dlen[ds] + dist_extra(ds);
}

// encode in[0, n) (n <= MAX_BLOCK) as one final DEFLATE block into out (words, at least stored_bytes(n) bytes rounded up); returns the
// bytes written.  All lanes of the team call it with the same arguments.
template <class Team>
INF_HD uint32_t deflate_block(const Team& t, EncShared& S, EncScratch sc, const uint8_t* in, uint32_t n, uint32_t* out) {
    static_assert(Team::size <= MAX_TEAM, "one parse segment per lane");
    // 1. chain
    for (uint32_t i = t.lane; i < HASH_SIZE; i += Team::size) S.u.head[i] = NIL;
    t.sync();
    if (t.chain_lane()) build_chain(t.chain(), S.u.head, sc.prev, in, n);
    t.sync();
    // 2. matches
    for (uint32_t p = t.lane; p < n; p += Team::size) sc.match[p] = find_match(sc.prev, in, n, p);
    for (uint32_t s = t.lane; s < NLIT; s += Team::size) S.lfreq[s] = 0;
    for (uint32_t s = t.lane; s < NDIST; s += Team::size) S.dfreq[s] = 0;
    t.sync();
    // 3. parse: segment per lane, guessed entries, repair rounds
    const uint32_t seg = (n + Team::size - 1) / Team::size;
    const uint32_t s0 = t.lane * seg < n ? t.lane * seg : n, s1 = s0 + seg < n ? s0 + seg : n;
    uint32_t entry = s0, exit_ = walk(sc.match, n, entry, s1);
    S.seg_exit[t.lane] = exit_;
    t.sync();
    for (;;) {
        const uint32_t want = t.lane ? S.seg_exit[t.lane - 1] : 0;
        const bool bad = want != entry;
        if (bad) { entry = want; exit_ = walk(sc.match, n, entry, s1); }
        if (!t.any(bad)) break;
        S.seg_exit[t.lane] = exit_;
        t.sync();
    }
    // 4. histograms and codes
    for (uint32_t p = entry; p < s1;) {
        const uint32_t q = next_pos(sc.match, p, n);
        if (q == p + 1) t.add32(&S.lfreq[in[p]], 1);
        else { t.add32(&S.lfreq[257 + len_sym(sc.match[p] >> 16)], 1); t.add32(&S.dfreq[dist_sym(sc.match[p] & 0xffff)], 1); }
        p = q;
    }
    t.sync();
    if (t.lane == 0) S.lfreq[256] = 1;                                  // end of block
    t.sync();
    build_lengths(t, S.u.h, S.lfreq, NLIT, MAXBITS, S.llen);
    build_lengths(t, S.u.h, S.dfreq, NDIST, MAXBITS, S.dlen);
    if (t.lane == 0) {
        canon_codes(S.llen, NLIT, S.lcode);
        canon_codes(S.dlen, NDIST, S.dcode);
        uint32_t hlit = NLIT, hdist = NDIST;
        while (S.llen[hlit - 1] == 0) hlit--;                           // (>= 257: the end-of-block code is there)
        while (S.dlen[hdist - 1] == 0) hdist--;                         // (>= 2: the code has two symbols at least)
        S.hlit = hlit; S.hdist = hdist;
        // run-length code of the lengths, literal/length and distance lengths as one sequence
        for (int s = 0; s < NCL; s++) S.cfreq[s] = 0;
        const uint32_t total = hlit + hdist;
        uint32_t nr = 0;
        for (uint32_t i = 0; i < total;) {
            const uint8_t v = i < hlit ? S.llen[i] : S.dlen[i - hlit];
            uint32_t run = 1;
            while (i + run < total && (i + run < hlit ? S.llen[i + run] : S.dlen[i + run - hlit]) == v) run++;
            if (v == 0 && run >= 11) { const uint32_t r = run < 138 ? run : 138; S.rle[nr++] = (uint16_t)(18 | (r - 11) << 5); S.cfreq[18]++; i += r; continue; }
            if (v == 0 && run >= 3) { const uint32_t r = run < 10 ? run : 10; S.rle[nr++] = (uint16_t)(17 | (r - 3) << 5); S.cfreq[17]++; i += r; continue; }
            S.rle[nr++] = v; S.cfreq[v]++; i++;
            if (v == 0) continue;
            for (uint32_t rest = run - 1; rest >= 3;) {
                const uint32_t r = rest < 6 ? rest : 6;
                S.rle[nr++] = (uint16_t)(16 | (r - 3) << 5); S.cfreq[16]++; i += r; rest -= r;
            }
        }
        S.n_rle = nr;
    }
    t.sync();
    build_lengths(t, S.u.h, S.cfreq, NCL, 7, S.clen);
    if (t.lane == 0) {
        canon_codes(S.clen, NCL, S.ccode);
        const uint8_t order[19] = {16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15};
        uint32_t hclen = 19;
        while (hclen > 4 && S.clen[order[hclen - 1]] == 0) hclen--;
        S.hclen = hclen;
        uint32_t bits = 3 + 5 + 5 + 4 + 3 * hclen;
        for (uint32_t i = 0; i < S.n_rle; i++) {
            const uint32_t s = S.rle[i] & 31;
            bits += S.clen[s] + (s == 16 ? 2 : s == 17 ? 3 : s == 18 ? 7 : 0);
        }
        S.hdr_bits = bits;
    }
    t.sync();
    // 5. bit offsets: per-segment sums, scanned
    uint32_t mine = 0;
    for (uint32_t p = entry; p < s1;) { const uint32_t q = next_pos(sc.match, p, n); mine += token_bits(S, in, sc.match, p, q); p = q; }
    S.seg_bits[t.lane] = mine;
    t.sync();
    if (t.lane == 0) {
        uint32_t acc = S.hdr_bits;
        for (unsigned k = 0; k < Team::size; k++) { const uint32_t b = S.seg_bits[k]; S.seg_bits[k] = acc; acc += b; }
        S.total_bits = acc + S.llen[256];
        S.stored = stored_bytes(n) < (S.total_bits + 7) / 8;
    }
    t.sync();
    uint8_t* ob = reinterpret_cast<uint8_t*>(out);
    if (S.stored) {
        if (t.lane == 0) { ob[0] = 1; ob[1] = (uint8_t)n; ob[2] = (uint8_t)(n >> 8); ob[3] = (uint8_t)~n; ob[4] = (uint8_t)(~n >> 8); }
        for (uint32_t i = t.lane; i < n; i += Team::size) ob[5 + i] = in[i];
        t.sync();
        return stored_bytes(n);
    }
    // 6. emit
    const uint32_t nw = (S.total_bits + 31) / 32;
    for (uint32_t i = t.lane; i < nw; i += Team::size) out[i] = 0;
    t.sync();
    if (t.lane == 0) {
        uint64_t pos = 0;
        put_bits(t, out, pos, 1 | 2 << 1, 3); pos += 3;                  // BFINAL, BTYPE 2
        put_bits(t, out, pos, S.hlit - 257, 5); pos += 5;
        put_bits(t, out, pos, S.hdist - 1, 5); pos += 5;
        put_bits(t, out, pos, S.hclen - 4, 4); pos += 4;
        const uint8_t order[19] = {16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15};
        for (uint32_t i = 0; i < S.hclen; i++) { put_bits(t, out, pos, S.clen[order[i]], 3); pos += 3; }
        for (uint32_t i = 0; i < S.n_rle; i++) {
            const uint32_t s = S.rle[i] & 31, x = S.rle[i] >> 5;
            put_bits(t, out, pos, S.ccode[s], S.clen[s]); pos += S.clen[s];
            const int xb = s == 16 ? 2 : s == 17 ? 3 : s == 18 ? 7 : 0;
            if (xb) { put_bits(t, out, pos, x, xb); pos += (uint64_t)xb; }
        }
        put_bits(t, out, S.total_bits - S.llen[256], S.lcode[256], S.llen[256]);
    }
    uint64_t pos = S.seg_bits[t.lane];
    for (uint32_t p = entry; p < s1;) {
        const uint32_t q = next_pos(sc.match, p, n);
        if (q == p + 1) { put_bits(t, out, pos, S.lcode[in[p]], S.llen[in[p]]); pos += S.llen[in[p]]; }
        else {
            const uint32_t L = sc.match[p] >> 16, d = sc.match[p] & 0xffff;
            const int ls = len_sym(L), ds = dist_sym(d);
            uint64_t v = S.lcode[257 + ls]; int nb = S.llen[257 + ls];
            v |= (uint64_t)(L - len_base(ls)) << nb; nb += (int)len_extra(ls);
            v |= (uint64_t)S.dcode[ds] << nb; nb += S.dlen[ds];
            v |= (uint64_t)(d - dist_base(ds)) << nb; nb += (int)dist_extra(ds);
            put_bits(t, out, pos, v, nb); pos += (uint64_t)nb;
        }
        p = q;
    }
    t.sync();
    return (S.total_bits + 7) / 8;
}

}  // namespace dfl
