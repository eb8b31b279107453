// optical.cu -- duplication metrics and optical-duplicate counting on the device
// (replaces filters.MarkOpticalDuplicates, filters/mark-optical-duplicates.go:468-517, with its helpers :50-93,176-447,
// filters/graph.go:24-85, filters/unpedantic.go:32-34; the derived metrics :519-581 and PrintDuplicatesMetrics :601-699
// run on the host below).
//
// The reference walks the sorted reads, re-joins the mates of every duplicate pair, looks the pair's origin up in the
// `pairs` map and hangs the first-of-pair read on the origin's list; then, per origin, it clusters the list members that
// sit on the same (read group, tile) within the pixel distance.  Here the pair list of phase_markdup is still sorted by
// the pair signature, so an origin's list is simply a run of equal signatures:
//   * every pair of a run other than the winner has both mates flagged 0x400 (classifyPair :375-395), i.e. is attached;
//     the winner is the origin and contributes its own first-of-pair read (:276-286) -- so the list is the whole run and
//     neither the winner's identity nor the order of the pairs inside the run (arrival order) matters: every count below,
//     including the LIST_CAP test, is taken over the whole run;
//   * singletons (the vast majority) only bump duplicatesCountHistogram[1] / nonOptical[1] and need no QNAME parse;
//   * runs of <= 32 pairs are clustered by one thread (sequential union-find), longer ones by one block
//     (lock-free union-find with atomicCAS hooking).  Σ(cluster size − 1) = members − clusters.
// Counters are integers, so any summation order gives the reference's numbers.
#include "ctx.h"
#include "gomath.hpp"
#include "../../include/elprep_b200.h"
#include <algorithm>
#include <climits>
#include <cmath>

namespace {

constexpr int LIST_CAP = 300000;        // :291-299, :330
constexpr int SMALL_MAX = 32;

// device-side accumulators
struct OptAcc {
    unsigned long long* ctr;     // [slots][OPT_NCTR]
    unsigned long long* hist;    // [slots][3][OPT_HBINS]
    unsigned long long* ovf;     // overflow triples (slot<<2|which, key) pairs
    uint32_t* ovf_n; uint32_t ovf_cap;
    uint32_t* big; uint32_t* big_n; uint32_t big_cap;
};

__device__ __forceinline__ void hist_inc(const OptAcc& A, int slot, int which, long long key) {
    if (key < OPT_HBINS) atomicAdd(A.hist + ((size_t)slot * 3 + which) * OPT_HBINS + key, 1ull);
    else {
        const uint32_t k = atomicAdd(A.ovf_n, 1u);
        if (k < A.ovf_cap) { A.ovf[2 * (size_t)k] = (unsigned long long)(slot * 4 + which); A.ovf[2 * (size_t)k + 1] = (unsigned long long)key; }
    }
}
// incrementDuplicatesCountsHistograms (:150-174) for one origin
__device__ __forceinline__ void origin_done(const OptAcc& A, int slot, long long n_f, long long n_r, long long opt_f, long long opt_r) {
    const long long dupcount = min(n_f, (long long)LIST_CAP + 1) + min(n_r, (long long)LIST_CAP + 1), optical = opt_f + opt_r;
    hist_inc(A, slot, 0, dupcount);
    if (dupcount - optical > 0) hist_inc(A, slot, 1, dupcount - optical);
    if (optical > 0) { hist_inc(A, slot, 2, optical + 1); atomicAdd(A.ctr + (size_t)slot * OPT_NCTR + 6, (unsigned long long)optical); }
}

// ---- per-read counters (:473-494) ----
__global__ void __launch_bounds__(256) opt_read_counters_kernel(uint64_t n, const uint16_t* __restrict__ flag, const int32_t* __restrict__ rg,
                                                                 const int32_t* __restrict__ rg_lib, int n_rg, unsigned long long* __restrict__ ctr) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    int code = -1;   // slot * 8 + class; a read can be in two classes: examined + duplicate fragment
    int code2 = -1;
    if (i < n) {
        const uint16_t f = flag[i]; const int32_t g = rg[i];
        const int slot = ((g >= 0 && g < n_rg) ? rg_lib[g] : -1) + 1;
        if (f & F_UNMAPPED) code = slot * 8 + 3;
        else if (f & (F_SECONDARY | F_SUPPLEMENTARY)) code = slot * 8 + 2;
        else {
            const bool frag = (f & (F_MULTIPLE | F_NEXTUNMAPPED)) != F_MULTIPLE;
            code = slot * 8 + (frag ? 0 : 1);
            if (frag && (f & F_DUPLICATE)) code2 = slot * 8 + 4;
        }
    }
    // warp-aggregated atomics
    for (int pass = 0; pass < 2; pass++) {
        const int cd = pass ? code2 : code;
        const unsigned act = __ballot_sync(FULL_MASK, cd >= 0);
        if (cd >= 0) {
            const unsigned peers = __match_any_sync(act, cd);
            if ((int)(threadIdx.x & 31) == __ffs(peers) - 1) atomicAdd(ctr + (size_t)(cd >> 3) * OPT_NCTR + (cd & 7), (unsigned long long)__popc(peers));
        }
    }
}

// strconv.ParseInt(s, 10, 64): 0 ok, 1 syntax/range error (the reference panics, internal/strconv.go:27-33)
__device__ int parse_i64(const uint8_t* s, int n, long long* out) {
    int i = 0; bool neg = false;
    if (n > 0 && (s[0] == '+' || s[0] == '-')) { neg = s[0] == '-'; i = 1; }
    if (i >= n) return 1;
    unsigned long long v = 0; const unsigned long long lim = neg ? (1ull << 63) : (1ull << 63) - 1;
    for (; i < n; i++) {
        if (s[i] < '0' || s[i] > '9') return 1;
        const unsigned long long d = (unsigned long long)(s[i] - '0');
        if (v > (lim - d) / 10) return 1;
        v = v * 10 + d;
    }
    *out = neg ? (long long)(0ull - v) : (long long)v;
    return 0;
}

// the pair keys are the signature alone: one word (u64) or two (u128 as lo,hi)
__device__ __forceinline__ bool same_group(const uint64_t* keys, uint64_t a, uint64_t b, int words) {
    return words == 1 ? keys[a] == keys[b] : (keys[2 * a] == keys[2 * b] && keys[2 * a + 1] == keys[2 * b + 1]);
}

// member info bits (m_info): bit0 strand of the list read, bit1 parse error, bit2 value outside int32, bits 8.. = rg + 1
#define MI_REV 1u
#define MI_PERR 2u
#define MI_PLIM 4u

struct MemberArgs {
    uint64_t npairs; const uint64_t* keys; const uint32_t* vals; int key_words;
    const uint32_t* pair_a; const uint32_t* pair_b; const uint16_t* flag; const int32_t* rg; const int32_t* rg_lib; int n_rg;
    const uint64_t* qname_off; const uint8_t* qname;
    int32_t* m_t; int32_t* m_x; int32_t* m_y; uint32_t* m_info;
};

// one thread per sorted pair: ReadPairDuplicates (:189), singleton origins, member records of longer runs (computeTileInfo :50-71)
__global__ void __launch_bounds__(256) opt_members_kernel(MemberArgs M, OptAcc A) {
    const uint64_t j = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    int slot = -1; bool both_dup = false, single = false;
    if (j < M.npairs) {
        const uint32_t p = M.vals[j], a1 = M.pair_a[p], a2 = M.pair_b[p];
        const uint16_t f1 = M.flag[a1], f2 = M.flag[a2];
        const int32_t g = M.rg[a1];
        slot = ((g >= 0 && g < M.n_rg) ? M.rg_lib[g] : -1) + 1;
        both_dup = (f1 & F_DUPLICATE) && (f2 & F_DUPLICATE);
        const bool head = j == 0 || !same_group(M.keys, j - 1, j, M.key_words);
        const bool last = j + 1 == M.npairs || !same_group(M.keys, j, j + 1, M.key_words);
        single = head && last;
        if (!single) {
            const uint32_t e = (f1 & F_FIRST) ? a1 : a2;                       // :216-221, :276-281
            uint32_t info = ((M.flag[e] & F_REVERSED) ? MI_REV : 0u) | ((uint32_t)(M.rg[e] + 1) << 8);
            const uint8_t* q = M.qname + M.qname_off[e]; const int n = (int)(M.qname_off[e + 1] - M.qname_off[e]);
            int start[8], end[8], nc = 0, b = 0;
            for (int i = 0; i <= n; i++) if (i == n || q[i] == ':') { if (nc < 8) { start[nc] = b; end[nc] = i; } nc++; b = i + 1; }
            long long t = -1, x = -1, y = -1;
            const int f0 = nc == 7 ? 4 : (nc == 5 ? 2 : -1);
            if (f0 >= 0) {
                if (parse_i64(q + start[f0], end[f0] - start[f0], &t) | parse_i64(q + start[f0 + 1], end[f0 + 1] - start[f0 + 1], &x) |
                    parse_i64(q + start[f0 + 2], end[f0 + 2] - start[f0 + 2], &y)) { info |= MI_PERR; t = -1; }
                else if (t < INT_MIN || t > INT_MAX || x < INT_MIN || x > INT_MAX || y < INT_MIN || y > INT_MAX) { info |= MI_PLIM; t = -1; }
            }
            M.m_t[j] = (int32_t)t; M.m_x[j] = (int32_t)x; M.m_y[j] = (int32_t)y; M.m_info[j] = info;
        }
    }
    const unsigned lane = threadIdx.x & 31;
    {   // ReadPairDuplicates
        const int cd = both_dup ? slot : -1;
        const unsigned act = __ballot_sync(FULL_MASK, cd >= 0);
        if (cd >= 0) { const unsigned peers = __match_any_sync(act, cd); if ((int)lane == __ffs(peers) - 1) atomicAdd(A.ctr + (size_t)cd * OPT_NCTR + 5, (unsigned long long)__popc(peers)); }
    }
    {   // singleton origins: duplicatesCount = 1, no optical duplicates
        const int cd = single ? slot : -1;
        const unsigned act = __ballot_sync(FULL_MASK, cd >= 0);
        if (cd >= 0) {
            const unsigned peers = __match_any_sync(act, cd);
            if ((int)lane == __ffs(peers) - 1) {
                atomicAdd(A.hist + ((size_t)cd * 3 + 0) * OPT_HBINS + 1, (unsigned long long)__popc(peers));
                atomicAdd(A.hist + ((size_t)cd * 3 + 1) * OPT_HBINS + 1, (unsigned long long)__popc(peers));
            }
        }
    }
}

__device__ __forceinline__ bool optical_edge(const MemberArgs& M, uint64_t a, uint64_t b, int dist) {
    const uint32_t ia = M.m_info[a], ib = M.m_info[b];
    if (((ia ^ ib) & ~(MI_PERR | MI_PLIM)) != 0) return false;     // same strand list, same read group (:83, :248)
    const int32_t ta = M.m_t[a];
    if (ta == -1 || ta != M.m_t[b]) return false;                   // :86-91
    const long long dx = (long long)M.m_x[a] - M.m_x[b], dy = (long long)M.m_y[a] - M.m_y[b];
    return (dx < 0 ? -dx : dx) <= dist && (dy < 0 ? -dy : dy) <= dist;   // unpedantic.go:32-34
}

// runs of 2..32 pairs: one thread per run head; longer runs are queued for the block kernel
__global__ void __launch_bounds__(256) opt_small_groups_kernel(MemberArgs M, OptAcc A, int dist, uint32_t* __restrict__ err) {
    const uint64_t j = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= M.npairs) return;
    if (j > 0 && same_group(M.keys, j - 1, j, M.key_words)) return;
    uint64_t e = j + 1;
    while (e < M.npairs && e - j <= SMALL_MAX && same_group(M.keys, j, e, M.key_words)) e++;
    const int n = (int)(e - j);
    if (n == 1) return;
    if (n > SMALL_MAX) { const uint32_t k = atomicAdd(A.big_n, 1u); if (k < A.big_cap) A.big[k] = (uint32_t)j; return; }
    uint8_t par[SMALL_MAX];
    int n_f = 0, n_r = 0; uint32_t bad_f = 0, bad_r = 0;
    for (int i = 0; i < n; i++) {
        par[i] = (uint8_t)i;
        const uint32_t info = M.m_info[j + i];
        if (info & MI_REV) { n_r++; bad_r |= info & (MI_PERR | MI_PLIM); } else { n_f++; bad_f |= info & (MI_PERR | MI_PLIM); }
    }
    // a list of fewer than two reads is never parsed (:339-341)
    const uint32_t bad = (n_f >= 2 ? bad_f : 0u) | (n_r >= 2 ? bad_r : 0u);
    if (bad) { atomicOr(err, (bad & MI_PERR) ? DERR_TILE : DERR_TILE_RANGE); return; }
    for (int a = 0; a < n; a++)
        for (int b = a + 1; b < n; b++)
            if (optical_edge(M, j + a, j + b, dist)) {
                int ra = a; while (par[ra] != ra) ra = par[ra];
                int rb = b; while (par[rb] != rb) rb = par[rb];
                if (ra != rb) par[max(ra, rb)] = (uint8_t)min(ra, rb);
            }
    int roots_f = 0, roots_r = 0;
    for (int i = 0; i < n; i++) if (par[i] == i) { if (M.m_info[j + i] & MI_REV) roots_r++; else roots_f++; }
    const uint32_t p = M.vals[j]; const int32_t g = M.rg[M.pair_a[p]];
    const int slot = ((g >= 0 && g < M.n_rg) ? M.rg_lib[g] : -1) + 1;
    origin_done(A, slot, n_f, n_r, n_f - roots_f, n_r - roots_r);
}

__device__ __forceinline__ uint32_t uf_find(uint32_t* par, uint32_t x) {
    uint32_t p = par[x];
    while (p != x) { const uint32_t gp = par[p]; if (gp != p) atomicCAS(par + x, p, gp); x = p; p = par[x]; }   // path halving, races are benign
    return x;
}
__device__ __forceinline__ void uf_union(uint32_t* par, uint32_t a, uint32_t b) {
    for (;;) {
        a = uf_find(par, a); b = uf_find(par, b);
        if (a == b) return;
        if (a < b) { const uint32_t t = a; a = b; b = t; }
        if (atomicCAS(par + a, a, b) == a) return;     // hook the larger root under the smaller one
    }
}

// runs of more than 32 pairs: one block per run. par[] holds run-relative parents.
__global__ void __launch_bounds__(256) opt_big_groups_kernel(MemberArgs M, OptAcc A, int dist, uint32_t* __restrict__ par_all, uint32_t* __restrict__ err) {
    const uint64_t j = A.big[blockIdx.x];
    __shared__ unsigned long long s_end;
    __shared__ unsigned long long s_cnt[4];   // n_f, n_r, roots_f, roots_r
    __shared__ uint32_t s_bad[2];
    if (threadIdx.x == 0) { s_end = M.npairs; s_cnt[0] = s_cnt[1] = s_cnt[2] = s_cnt[3] = 0; s_bad[0] = s_bad[1] = 0; }
    __syncthreads();
    for (uint64_t base = j + 1; base < M.npairs; base += blockDim.x) {     // cooperative search for the end of the run
        const uint64_t t = base + threadIdx.x;
        if (t < M.npairs && !same_group(M.keys, j, t, M.key_words)) atomicMin(&s_end, (unsigned long long)t);
        __syncthreads();
        if (s_end != M.npairs) break;
    }
    __syncthreads();
    const uint64_t e = s_end; const uint32_t n = (uint32_t)(e - j);
    uint32_t* par = par_all + j;
    unsigned long long c_f = 0, c_r = 0; uint32_t bf = 0, br = 0;
    for (uint32_t i = threadIdx.x; i < n; i += blockDim.x) {
        par[i] = i;
        const uint32_t info = M.m_info[j + i];
        if (info & MI_REV) { c_r++; br |= info & (MI_PERR | MI_PLIM); } else { c_f++; bf |= info & (MI_PERR | MI_PLIM); }
    }
    atomicAdd(&s_cnt[0], c_f); atomicAdd(&s_cnt[1], c_r); atomicOr(&s_bad[0], bf); atomicOr(&s_bad[1], br);
    __syncthreads();
    const unsigned long long n_f = s_cnt[0], n_r = s_cnt[1];
    const bool do_f = n_f >= 2 && n_f <= LIST_CAP, do_r = n_r >= 2 && n_r <= LIST_CAP;   // :330-341
    const uint32_t bad = (do_f ? s_bad[0] : 0u) | (do_r ? s_bad[1] : 0u);
    if (bad) { if (threadIdx.x == 0) atomicOr(err, (bad & MI_PERR) ? DERR_TILE : DERR_TILE_RANGE); return; }
    for (uint32_t a = threadIdx.x; a < n; a += blockDim.x) {
        const bool rev = M.m_info[j + a] & MI_REV;
        if (!(rev ? do_r : do_f)) continue;
        for (uint32_t b = a + 1; b < n; b++) if (optical_edge(M, j + a, j + b, dist)) uf_union(par, a, b);
    }
    __syncthreads();
    unsigned long long r_f = 0, r_r = 0;
    for (uint32_t i = threadIdx.x; i < n; i += blockDim.x) if (par[i] == i) { if (M.m_info[j + i] & MI_REV) r_r++; else r_f++; }
    atomicAdd(&s_cnt[2], r_f); atomicAdd(&s_cnt[3], r_r);
    __syncthreads();
    if (threadIdx.x == 0) {
        const uint32_t p = M.vals[j]; const int32_t g = M.rg[M.pair_a[p]];
        const int slot = ((g >= 0 && g < M.n_rg) ? M.rg_lib[g] : -1) + 1;
        origin_done(A, slot, (long long)n_f, (long long)n_r, do_f ? (long long)(n_f - s_cnt[2]) : 0, do_r ? (long long)(n_r - s_cnt[3]) : 0);
    }
}

inline unsigned nblk(uint64_t n, int t) { return (unsigned)((n + t - 1) / t); }

}  // namespace

// ---------------------------------------------------------------- host side
static int opt_alloc(elp_ctx* c) {
    const size_t slots = (size_t)c->n_lib + 1;
    if (!c->d_opt_ctr) {
        CUDA_TRY(c, cudaMalloc(&c->d_opt_ctr, slots * OPT_NCTR * 8));
        CUDA_TRY(c, cudaMalloc(&c->d_opt_hist, slots * 3 * OPT_HBINS * 8));
        CUDA_TRY(c, cudaMalloc(&c->d_opt_ovf, (size_t)OPT_OVF_CAP * 16));
        CUDA_TRY(c, cudaMalloc(&c->d_opt_small, 16));
    }
    CUDA_TRY(c, cudaMemsetAsync(c->d_opt_ctr, 0, slots * OPT_NCTR * 8, c->stream));
    CUDA_TRY(c, cudaMemsetAsync(c->d_opt_hist, 0, slots * 3 * OPT_HBINS * 8, c->stream));
    CUDA_TRY(c, cudaMemsetAsync(c->d_opt_small, 0, 16, c->stream));
    return E_OK;
}

// called by phase_markdup after pair_mark (npairs may be 0: then only the per-read counters run)
int phase_optical(elp_ctx* c, uint64_t npairs, const uint64_t* sorted_keys, const uint32_t* sorted_vals, int key_words) {
    int rc = opt_alloc(c);
    if (rc) return rc;
    const uint64_t n = c->n;
    const size_t slots = (size_t)c->n_lib + 1;
    OptAcc A{};
    A.ctr = reinterpret_cast<unsigned long long*>(c->d_opt_ctr); A.hist = reinterpret_cast<unsigned long long*>(c->d_opt_hist);
    A.ovf = reinterpret_cast<unsigned long long*>(c->d_opt_ovf); A.ovf_n = c->d_opt_small; A.ovf_cap = OPT_OVF_CAP;
    A.big_n = c->d_opt_small + 1;
    if (n) {
        c->begin("opt_read_counters", (double)n * 6);
        opt_read_counters_kernel<<<nblk(n, 256), 256, 0, c->stream>>>(n, c->flag.p, c->rg.p, c->d_rg_lib, c->n_rg, A.ctr);
        c->end(); LAUNCH_CHECK(c);
    }
    uint32_t small[4] = {0, 0, 0, 0};
    if (npairs) {
        // scratch: keys_b (2n+4 u64) is free after pair_keys_kernel; npairs <= n/2, so five u32 arrays of npairs fit
        uint32_t* base = reinterpret_cast<uint32_t*>(c->keys_b.p);
        MemberArgs M{};
        M.npairs = npairs; M.keys = sorted_keys; M.vals = sorted_vals; M.key_words = key_words; M.pair_a = c->pair_a.p; M.pair_b = c->pair_b.p;
        M.flag = c->flag.p; M.rg = c->rg.p; M.rg_lib = c->d_rg_lib; M.n_rg = c->n_rg; M.qname_off = c->qname_off.p; M.qname = c->qname.p;
        M.m_t = reinterpret_cast<int32_t*>(base); M.m_x = reinterpret_cast<int32_t*>(base + npairs); M.m_y = reinterpret_cast<int32_t*>(base + 2 * npairs);
        M.m_info = base + 3 * npairs;
        uint32_t* par = base + 4 * npairs;
        A.big = c->scan_tmp.p; A.big_cap = (uint32_t)std::min<uint64_t>(c->scan_tmp.cap, npairs / SMALL_MAX + 1);
        c->begin("opt_members", (double)npairs * (16 + 4 + 8 + 4 + 40));
        opt_members_kernel<<<nblk(npairs, 256), 256, 0, c->stream>>>(M, A);
        c->end(); LAUNCH_CHECK(c);
        c->begin("opt_small_groups", (double)npairs * 16);
        opt_small_groups_kernel<<<nblk(npairs, 256), 256, 0, c->stream>>>(M, A, c->optical_pixel_distance, c->d_err);
        c->end(); LAUNCH_CHECK(c);
        CUDA_TRY(c, cudaMemcpyAsync(small, c->d_opt_small, 16, cudaMemcpyDeviceToHost, c->stream));
        CUDA_TRY(c, cudaStreamSynchronize(c->stream));
        if (small[1] > A.big_cap) return c->fail(E_CUDA, "optical: long-run queue overflow (%u > %u)", small[1], A.big_cap);
        if (small[1]) {
            c->begin("opt_big_groups", (double)small[1] * 33 * 16);
            opt_big_groups_kernel<<<small[1], 256, 0, c->stream>>>(M, A, c->optical_pixel_distance, par, c->d_err);
            c->end(); LAUNCH_CHECK(c);
        }
    }
    rc = check_device_errors(c);
    if (rc) return rc;
    // bring the accumulators back
    std::vector<unsigned long long> h_ctr(slots * OPT_NCTR), h_hist(slots * 3 * OPT_HBINS);
    CUDA_TRY(c, cudaMemcpyAsync(h_ctr.data(), c->d_opt_ctr, h_ctr.size() * 8, cudaMemcpyDeviceToHost, c->stream));
    CUDA_TRY(c, cudaMemcpyAsync(h_hist.data(), c->d_opt_hist, h_hist.size() * 8, cudaMemcpyDeviceToHost, c->stream));
    CUDA_TRY(c, cudaMemcpyAsync(small, c->d_opt_small, 16, cudaMemcpyDeviceToHost, c->stream));
    CUDA_TRY(c, cudaStreamSynchronize(c->stream));
    if (small[0] > OPT_OVF_CAP) return c->fail(E_LIMIT, "optical: more than %d histogram keys above %d", OPT_OVF_CAP, OPT_HBINS);
    std::vector<unsigned long long> h_ovf(2 * (size_t)small[0]);
    if (small[0]) { CUDA_TRY(c, cudaMemcpyAsync(h_ovf.data(), c->d_opt_ovf, h_ovf.size() * 8, cudaMemcpyDeviceToHost, c->stream)); CUDA_TRY(c, cudaStreamSynchronize(c->stream)); }
    c->opt.assign(slots, DupCounters{});
    for (size_t s = 0; s < slots; s++) {
        DupCounters& d = c->opt[s];
        for (int k = 0; k < 7; k++) d.ctr[k] = (int64_t)h_ctr[s * OPT_NCTR + k];
        for (int w = 0; w < 3; w++)
            for (int k = 0; k < OPT_HBINS; k++) { const unsigned long long v = h_hist[(s * 3 + w) * OPT_HBINS + k]; if (v) d.hist[w][k] += (int64_t)v; }
    }
    for (uint32_t k = 0; k < small[0]; k++) { const unsigned long long sw = h_ovf[2 * (size_t)k]; c->opt[sw >> 2].hist[sw & 3][(int64_t)h_ovf[2 * (size_t)k + 1]] += 1; }
    c->opt_valid = true;
    return E_OK;
}

// estimateLibrarySize (:533-562)
static int64_t estimate_library_size(int64_t n_pairs, int64_t n_unique) {
    const double n = (double)n_pairs, cc = (double)n_unique;
    if (n_pairs > 0 && n_pairs - n_unique > 0) {
        auto f = [&](double x) { return cc / x - 1 + gomath::Exp(-n / x); };
        double m = 1.0, M = 100.0;
        double fd = f(M * cc);
        while (fd >= 0.0) { M *= 10.0; fd = f(M * cc); }
        for (int i = 0; i < 40; i++) {
            const double r = (m + M) / 2.0, u = f(r * cc);
            if (u == 0.0) break;
            if (u > 0.0) m = r;
            if (u < 0.0) M = r;
        }
        return (int64_t)(cc * ((m + M) / 2.0));
    }
    return 0;
}

// calculateDerivedDuplicateMetrics (:519-525), estimateRoi (:570-572), histogramRoi (:574-581)
// DupCounters.ctr[1] counts paired READS (the reference halves after its reduction, :503-505; keeping reads makes the sum
// over several workers exact); everything derived uses pairs.
static void derive(const DupCounters& d0, elp_dup_metrics* m) {
    DupCounters d = d0; d.ctr[1] = d0.ctr[1] / 2;
    m->paired_reads_examined = d0.ctr[1];
    m->unpaired_reads_examined = d.ctr[0]; m->read_pairs_examined = d.ctr[1]; m->secondary_or_supplementary_reads = d.ctr[2]; m->unmapped_reads = d.ctr[3];
    m->unpaired_read_duplicates = d.ctr[4]; m->read_pair_duplicates = d.ctr[5]; m->read_pair_optical_duplicates = d.ctr[6];
    m->estimated_library_size = 0; m->has_roi = 0;
    for (double& v : m->roi) v = 0;
    if (d.ctr[1] > 0) {
        m->estimated_library_size = estimate_library_size(d.ctr[1] - d.ctr[6], d.ctr[1] - d.ctr[5]);
        const int64_t uniq = d.ctr[1] - d.ctr[5];
        for (int64_t x = 1; x <= 100; x++)
            m->roi[x - 1] = (double)m->estimated_library_size * (1.0 - gomath::Exp(-(double)(x * d.ctr[1]) / (double)m->estimated_library_size)) / (double)uniq;
        m->has_roi = 1;
    }
    m->percent_duplication = (double)(d.ctr[4] + d.ctr[5] * 2) / (double)(d.ctr[0] + d.ctr[1] * 2);
}

// formatFloat (:583-599)
static std::string format_float(double f) {
    if (f != f) return "NaN";
    if (std::isinf(f)) return f > 0 ? "+Inf" : "-Inf";
    char buf[64]; snprintf(buf, sizeof buf, "%.6f", f);
    std::string s = buf;
    const size_t dot = s.find('.');
    if (dot == std::string::npos) return s;
    for (size_t j = s.size() - 1; j > dot; j--) if (s[j] != '0') return s.substr(0, j + 1);
    return s;
}

static const char* slot_name(const elp_ctx* c, int slot) { return slot == 0 ? "Unknown Library" : c->lib_names[slot - 1].c_str(); }

extern "C" {

int32_t elp_optical_n_libraries(const elp_ctx* c) { return c ? c->n_lib + 1 : 0; }
const char* elp_optical_library_name(const elp_ctx* c, int32_t slot) { return (c && slot >= 0 && slot <= c->n_lib) ? slot_name(c, slot) : nullptr; }

int elp_optical_metrics(elp_ctx* c, int32_t slot, elp_dup_metrics* out) {
    if (!c || !out) return ELP_EINVAL;
    if (!c->opt_valid) return c->fail(E_STATE, "elp_optical_metrics before elp_sort_markdup(.., ELP_MARKDUP_OPTICAL)");
    if (slot < 0 || slot > c->n_lib) return c->fail(E_INVAL, "elp_optical_metrics: slot %d out of range", slot);
    derive(c->opt[slot], out);
    return ELP_OK;
}

int64_t elp_optical_histogram(elp_ctx* c, int32_t slot, int32_t which, int64_t* keys, int64_t* counts, int64_t cap) {
    if (!c || !c->opt_valid || slot < 0 || slot > c->n_lib || which < 0 || which > 2) return -1;
    int64_t k = 0;
    for (auto& kv : c->opt[slot].hist[which]) { if (keys && counts && k < cap) { keys[k] = kv.first; counts[k] = kv.second; } k++; }
    return k;
}

int elp_optical_merge(elp_ctx* c, int32_t slot, const int64_t* counters7, int32_t which, const int64_t* keys, const int64_t* counts, int64_t n) {
    if (!c) return ELP_EINVAL;
    if (slot < 0 || slot > c->n_lib) return c->fail(E_INVAL, "elp_optical_merge: slot %d out of range", slot);
    if (!c->opt_valid) { c->opt.assign((size_t)c->n_lib + 1, DupCounters{}); c->opt_valid = true; }
    if (counters7) for (int k = 0; k < 7; k++) c->opt[slot].ctr[k] += counters7[k];
    if (keys && counts) { if (which < 0 || which > 2) return c->fail(E_INVAL, "elp_optical_merge: which"); for (int64_t k = 0; k < n; k++) c->opt[slot].hist[which][keys[k]] += counts[k]; }
    return ELP_OK;
}

int elp_print_duplicates_metrics(elp_ctx* c, const char* path, const char* command_line, const char* started_on) {
    if (!c || !path) return ELP_EINVAL;
    if (!c->opt_valid) return c->fail(E_STATE, "elp_print_duplicates_metrics before elp_sort_markdup(.., ELP_MARKDUP_OPTICAL)");
    FILE* f = fopen(path, "w");
    if (!f) return c->fail(E_INVAL, "cannot create %s", path);
    const int n = c->n_lib + 1;
    std::vector<int> ord(n);
    for (int i = 0; i < n; i++) ord[i] = i;
    std::stable_sort(ord.begin(), ord.end(), [&](int a, int b) { return strcmp(slot_name(c, a), slot_name(c, b)) < 0; });
    fprintf(f, "## htsjdk.samtools.metrics.StringHeader\n# %s\n## htsjdk.samtools.metrics.StringHeader\n# Started on: %s\n\n## METRICS CLASS\tpicard.sam.DuplicationMetrics\n",
            command_line ? command_line : "", started_on ? started_on : "");
    fprintf(f, "LIBRARY\tUNPAIRED_READS_EXAMINED\tREAD_PAIRS_EXAMINED\tSECONDARY_OR_SUPPLEMENTARY_RDS\tUNMAPPED_READS\tUNPAIRED_READ_DUPLICATES\tREAD_PAIR_DUPLICATES\tREAD_PAIR_OPTICAL_DUPLICATES\tPERCENT_DUPLICATION\tESTIMATED_LIBRARY_SIZE\n");
    int the = -1; bool many = false;
    elp_dup_metrics m;
    for (int k = 0; k < n; k++) {
        derive(c->opt[ord[k]], &m);
        fprintf(f, "%s\t%lld\t%lld\t%lld\t%lld\t%lld\t%lld\t%lld\t%s", slot_name(c, ord[k]), (long long)m.unpaired_reads_examined, (long long)m.read_pairs_examined,
                (long long)m.secondary_or_supplementary_reads, (long long)m.unmapped_reads, (long long)m.unpaired_read_duplicates, (long long)m.read_pair_duplicates,
                (long long)m.read_pair_optical_duplicates, format_float(m.percent_duplication).c_str());
        if (m.read_pairs_examined > 0) { fprintf(f, "\t%lld", (long long)m.estimated_library_size); if (the >= 0) many = true; the = ord[k]; }
        fprintf(f, "\n");
    }
    fprintf(f, "\n");
    if (many || the < 0) { fprintf(f, "\n"); fclose(f); return ELP_OK; }       // histogram only for exactly one library (:631-647)
    derive(c->opt[the], &m);
    const DupCounters& d = c->opt[the];
    auto hv = [&](int w, int64_t k) -> long long { auto it = d.hist[w].find(k); return it == d.hist[w].end() ? 0LL : (long long)it->second; };
    fprintf(f, "## HISTOGRAM\tjava.lang.Double\nBIN\tCoverageMult\tall_sets\toptical_sets\tnon_optical_sets\n");
    for (int i = 0; i < 100; i++) fprintf(f, "%d.0\t%s\t%lld\t%lld\t%lld\n", i + 1, format_float(m.roi[i]).c_str(), hv(0, i + 1), hv(2, i + 1), hv(1, i + 1));
    std::map<int64_t, int> rest;
    for (int w = 0; w < 3; w++) for (auto& kv : d.hist[w]) if (kv.first > 100) rest[kv.first] = 1;
    for (auto& kv : rest) fprintf(f, "%lld.0\t0\t%lld\t%lld\t%lld\n", (long long)kv.first, hv(0, kv.first), hv(2, kv.first), hv(1, kv.first));
    fprintf(f, "\n");
    fclose(f);
    return ELP_OK;
}

}  // extern "C"
