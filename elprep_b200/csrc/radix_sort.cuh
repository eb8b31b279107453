// radix_sort.cuh -- hand-written onesweep LSD radix sort for sm_90a (keys u32, u64 or u128, u32 payload).
//
// Replaces pargo sort.StableSort as used by By(CoordinateLess).ParallelStableSort (sam/sam-types.go:599-641)
// and the sharded-map grouping of filters/mark-duplicates.go:210-396 (sort-by-key + segmented scan instead of
// LoadOrStore).  Stable, so equal keys keep arrival order exactly as the reference's stable merge sort does.
//
// Structure (one read of the keys for all digit histograms, then ONE read + ONE write of keys and payload per
// digit pass -- algorithmic bytes N*(K + 2*P*(K+V)), SURVEY.md section 8d):
//   rs_hist_kernel      all P digit histograms in a single pass over the keys (shared-memory counters)
//   rs_scan_kernel      exclusive scan of each 256-bin histogram -> global digit offsets
//   rs_onesweep_kernel  per pass: warp-striped coalesced key loads, per-warp ranking with match.any,
//                       chained-scan (decoupled look-back) across tiles for the global digit offsets, tile-local
//                       reorder through shared memory so the scatter leaves in digit-contiguous runs.
// Keys are compacted by the caller; the sort orders by bits [lo_bit, lo_bit + key_bits) in P = ceil(key_bits/8) passes with
// balanced digit widths <= 8.  Bits below lo_bit travel with the key unsorted (equal ranges keep arrival order).
#pragma once
#include "common.cuh"

namespace rs {

constexpr int RADIX = 256;
constexpr int MAX_PASSES = 16;
constexpr uint32_t ST_PARTIAL = 1u << 30, ST_INCLUSIVE = 2u << 30, ST_VALMASK = (1u << 30) - 1;

struct Plan {
    int n_passes;
    int shift[MAX_PASSES];
    int bits[MAX_PASSES];
};

inline Plan make_plan(int key_bits, int lo_bit = 0) {
    Plan p{};
    if (key_bits < 1) key_bits = 1;
    p.n_passes = (key_bits + 7) / 8;
    int base = key_bits / p.n_passes, extra = key_bits % p.n_passes, s = lo_bit;
    for (int i = 0; i < p.n_passes; i++) {
        p.bits[i] = base + (i < extra ? 1 : 0);
        p.shift[i] = s;
        s += p.bits[i];
    }
    return p;
}

struct K32 {
    uint32_t v;
    __device__ __forceinline__ static K32 load(const K32* p) { K32 k; k.v = ld_stream_u32(reinterpret_cast<const uint32_t*>(p)); return k; }
    __device__ __forceinline__ uint32_t digit(int shift, uint32_t mask) const { return (v >> shift) & mask; }
};
struct K64 {
    uint64_t v;
    __device__ __forceinline__ static K64 load(const K64* p) { K64 k; k.v = ld_stream_u64(reinterpret_cast<const uint64_t*>(p)); return k; }
    __device__ __forceinline__ uint32_t digit(int shift, uint32_t mask) const { return (uint32_t)(v >> shift) & mask; }
};
struct __align__(16) K128 {
    uint64_t lo, hi;
    __device__ __forceinline__ static K128 load(const K128* p) { uint4 r = ld_stream_u4(p); K128 k; k.lo = (uint64_t)r.x | ((uint64_t)r.y << 32); k.hi = (uint64_t)r.z | ((uint64_t)r.w << 32); return k; }
    __device__ __forceinline__ uint32_t digit(int shift, uint32_t mask) const {
        uint64_t w = shift >= 64 ? (hi >> (shift - 64)) : (shift == 0 ? lo : ((lo >> shift) | (hi << (64 - shift))));
        return (uint32_t)w & mask;
    }
};

// ---------------------------------------------------------------- all digit histograms in one pass
template <class K>
__global__ void __launch_bounds__(512) rs_hist_kernel(const K* __restrict__ keys, uint64_t n, Plan plan, uint32_t* __restrict__ ghist) {
    __shared__ uint32_t sh[MAX_PASSES * RADIX];
    for (int i = threadIdx.x; i < plan.n_passes * RADIX; i += blockDim.x) sh[i] = 0;
    __syncthreads();
    const unsigned lane = lane_id();
    const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; (i - lane) < n; i += stride) {
        bool valid = i < n;
        K k{};
        if (valid) k = K::load(keys + i);
        unsigned vmask = __ballot_sync(FULL_MASK, valid);
#pragma unroll 1
        for (int p = 0; p < plan.n_passes; p++) {
            uint32_t d = valid ? k.digit(plan.shift[p], (1u << plan.bits[p]) - 1) : 0xffffffffu;
            // sorted / low-entropy inputs: the whole warp hits one bin -> one add instead of a 32-way same-address conflict
            uint32_t d0 = __shfl_sync(FULL_MASK, d, __ffs(vmask) - 1);
            bool uni = __all_sync(FULL_MASK, !valid || d == d0);
            if (uni) { if (lane == (unsigned)(__ffs(vmask) - 1)) atomicAdd(&sh[p * RADIX + d0], __popc(vmask)); }
            else if (valid) atomicAdd(&sh[p * RADIX + d], 1u);
        }
    }
    __syncthreads();
    for (int i = threadIdx.x; i < plan.n_passes * RADIX; i += blockDim.x) { uint32_t c = sh[i]; if (c) atomicAdd(&ghist[i], c); }
}

// exclusive scan of each pass' 256-bin histogram (one block per pass)
static __global__ void rs_scan_kernel(const uint32_t* __restrict__ ghist, uint32_t* __restrict__ gofs) {
    __shared__ uint32_t wsum[8];
    const int p = blockIdx.x, d = threadIdx.x;
    uint32_t c = ghist[p * RADIX + d], x = c;
    const unsigned lane = d & 31, w = d >> 5;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { uint32_t y = __shfl_up_sync(FULL_MASK, x, o); if (lane >= (unsigned)o) x += y; }
    if (lane == 31) wsum[w] = x;
    __syncthreads();
    uint32_t add = 0;
    for (unsigned i = 0; i < w; i++) add += wsum[i];
    gofs[p * RADIX + d] = x - c + add;
}

#ifdef RS_TIMING
// phase timestamps (clock64 of thread 0) of sampled tiles, read back by elp_debug_sort_u64
static __device__ long long rs_tstamp[8 * 4096];
#define RS_STAMP(k) do { if (tid == 0 && (tile & 1) == 0 && (tile >> 1) < 4096) rs_tstamp[(tile >> 1) * 8 + (k)] = clock64(); } while (0)
#else
#define RS_STAMP(k) do { } while (0)
#endif
// ---------------------------------------------------------------- one digit pass
template <class K, int THREADS, int ITEMS, int MIN_CTAS>
__global__ void __launch_bounds__(THREADS, MIN_CTAS) rs_onesweep_kernel(const K* __restrict__ keys_in, K* __restrict__ keys_out,
                                                              const uint32_t* __restrict__ vals_in, uint32_t* __restrict__ vals_out,
                                                              uint64_t n, int shift, int bits, const uint32_t* __restrict__ gofs,
                                                              uint32_t* __restrict__ status, uint32_t* __restrict__ tile_counter) {
    constexpr int WARPS = THREADS / 32, TILE = THREADS * ITEMS;
    static_assert(THREADS >= RADIX && THREADS % 32 == 0, "one look-back thread per digit");
    static_assert(TILE % 4 == 0, "tiles start 16-byte aligned in the payload");
    extern __shared__ __align__(16) unsigned char smem_raw[];
    uint32_t* warp_hist = reinterpret_cast<uint32_t*>(smem_raw);                // [WARPS][RADIX]
    K* sk = reinterpret_cast<K*>(smem_raw + (size_t)WARPS * RADIX * 4);         // [TILE]; reused for the payload
    uint32_t* sv = reinterpret_cast<uint32_t*>(sk);
    uint32_t* stage_v = reinterpret_cast<uint32_t*>(smem_raw + (size_t)WARPS * RADIX * 4 + (size_t)TILE * sizeof(K));   // [TILE] payload in arrival order
    __shared__ uint32_t s_tile, digit_start[RADIX], gbase[RADIX], wsum[RADIX / 32];

    const unsigned tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const uint32_t mask = (1u << bits) - 1;
    if (tid == 0) s_tile = atomicAdd(tile_counter, 1u);   // ticket: a tile only ever waits on tiles that already started
    for (int i = tid; i < WARPS * RADIX; i += THREADS) warp_hist[i] = 0;
    __syncthreads();
    const uint32_t tile = s_tile;
    RS_STAMP(0);
    const uint64_t base = (uint64_t)tile * TILE;
    const uint32_t n_valid = (uint32_t)((n - base) < (uint64_t)TILE ? (n - base) : (uint64_t)TILE);

    // warp-striped loads: element (warp, j, lane) <-> tile index warp*ITEMS*32 + j*32 + lane (stable order = that index)
    K key[ITEMS];
    uint32_t rank[ITEMS];
    const uint32_t wbase = warp * ITEMS * 32 + lane;
#pragma unroll
    for (int j = 0; j < ITEMS; j++) {
        uint32_t t = wbase + j * 32;
        if (t < n_valid) key[j] = K::load(keys_in + base + t);
    }
    // the payload is only needed after the keys are ranked and written: copy it to shared memory asynchronously now
    // (16 bytes per request; a tile starts at a multiple of TILE elements, so the addresses are 16-byte aligned)
    {
        const uint32_t* vsrc = vals_in + base;
        for (uint32_t q = tid * 4; q < (uint32_t)TILE; q += THREADS * 4) {
            if (q + 4 <= n_valid) {
                const uint32_t dsts = (uint32_t)__cvta_generic_to_shared(stage_v + q);
                asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(dsts), "l"(vsrc + q) : "memory");
            } else {
                for (uint32_t e = q; e < q + 4 && e < n_valid; e++) stage_v[e] = vsrc[e];
            }
        }
        asm volatile("cp.async.commit_group;" ::: "memory");
    }
    RS_STAMP(1);
    uint32_t* wh = warp_hist + warp * RADIX;
#pragma unroll
    for (int j = 0; j < ITEMS; j++) {
        const bool valid = (wbase + j * 32) < n_valid;
        const uint32_t d = valid ? key[j].digit(shift, mask) : (0x100u + lane);   // invalid lanes match nobody
        const uint32_t peers = __match_any_sync(FULL_MASK, d);
        // every peer reads the running count, then the leader adds the peer count (no atomic with a return value, no shuffle);
        // __syncwarp orders the add before the next item's reads
        const uint32_t old = valid ? wh[d] : 0u;
        __syncwarp();
        if (valid && (peers & lanemask_lt()) == 0) wh[d] = old + (uint32_t)__popc(peers);
        __syncwarp();
        rank[j] = old + __popc(peers & lanemask_lt());
    }
    __syncthreads();
    RS_STAMP(2);

    // per digit: exclusive scan over warps, tile total (published at once for the successors' look-back), then exclusive
    // scan over digits
    uint32_t total = 0;
    uint32_t* my = status + (uint64_t)tile * RADIX + tid;
    if (tid < RADIX) {
        uint32_t run = 0;
#pragma unroll
        for (int w = 0; w < WARPS; w++) { uint32_t c = warp_hist[w * RADIX + tid]; warp_hist[w * RADIX + tid] = run; run += c; }
        total = run;
        if (tile > 0) st_relaxed_u32(my, total | ST_PARTIAL);
        uint32_t x = total;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) { uint32_t y = __shfl_up_sync(FULL_MASK, x, o); if (lane >= (unsigned)o) x += y; }
        if (lane == 31) wsum[warp] = x;
        digit_start[tid] = x - total;   // warp-local exclusive; warp sums added below
    }
    __syncthreads();
    // chained scan across tiles (decoupled look-back), one thread per digit.  Flag and value travel in ONE 32-bit word, so
    // relaxed accesses are enough (no other data is published through it).  The walk back over predecessor tiles issues LB
    // independent loads per step, and the first step is issued BEFORE the tile-local scatter so that its round trip overlaps it.
#ifndef RS_LB
#define RS_LB 8
#endif
    constexpr int LB = RS_LB;
    uint32_t lb_first[LB];
    uint32_t dstart = 0;
    if (tid < RADIX) {
        uint32_t add = 0;
        for (unsigned i = 0; i < warp; i++) add += wsum[i];
        dstart = digit_start[tid] + add;
        digit_start[tid] = dstart;
        if (tile > 0) {
#pragma unroll
            for (int j = 0; j < LB; j++) lb_first[j] = ((int64_t)tile - 1 - j >= 0) ? ld_relaxed_u32(status + (uint64_t)(tile - 1 - j) * RADIX + tid) : ST_INCLUSIVE;
        }
    }
    __syncthreads();
    RS_STAMP(3);

    // tile-local reorder through shared memory (needs only tile-local offsets)
#pragma unroll
    for (int j = 0; j < ITEMS; j++) {
        if ((wbase + j * 32) < n_valid) {
            const uint32_t d = key[j].digit(shift, mask);
            rank[j] += digit_start[d] + wh[d];
            sk[rank[j]] = key[j];
        }
    }
    // finish the look-back
    if (tid < RADIX) {
        uint32_t excl = 0;
        if (tile > 0) {
            int64_t t = (int64_t)tile - 1;
            bool done = false, first = true;
            while (!done) {
                uint32_t svv[LB];
#pragma unroll
                for (int j = 0; j < LB; j++) svv[j] = first ? lb_first[j] : ((t - j >= 0) ? ld_relaxed_u32(status + (uint64_t)(t - j) * RADIX + tid) : ST_INCLUSIVE);
                first = false;
#pragma unroll
                for (int j = 0; j < LB; j++) {
                    if (done) break;
                    uint32_t sx = svv[j];
                    while ((sx >> 30) == 0) {   // predecessor not published yet
                        sx = ld_relaxed_u32(status + (uint64_t)(t - j) * RADIX + tid);
                    }
                    excl += sx & ST_VALMASK;
                    if ((sx >> 30) == 2) done = true;
                }
                t -= LB;
            }
        }
        st_relaxed_u32(my, ((excl + total) & ST_VALMASK) | ST_INCLUSIVE);
        gbase[tid] = gofs[tid] + excl - dstart;   // modulo 2^32: final index = gbase[d] + tile-local sorted position
    }
    // digit-contiguous (coalesced) global writes
    __syncthreads();
    RS_STAMP(4);
    uint32_t dst[ITEMS];
#pragma unroll
    for (int k = 0; k < ITEMS; k++) {
        const uint32_t s = tid + k * THREADS;
        if (s < n_valid) {
            const K kk = sk[s];
            dst[k] = gbase[kk.digit(shift, mask)] + s;
            keys_out[dst[k]] = kk;
        }
    }
    asm volatile("cp.async.wait_group 0;" ::: "memory");
    __syncthreads();
    RS_STAMP(5);
#pragma unroll
    for (int j = 0; j < ITEMS; j++)
        if ((wbase + j * 32) < n_valid) sv[rank[j]] = stage_v[wbase + j * 32];
    __syncthreads();
    RS_STAMP(6);
#pragma unroll
    for (int k = 0; k < ITEMS; k++) {
        const uint32_t s = tid + k * THREADS;
        if (s < n_valid) vals_out[dst[k]] = sv[s];
    }
    RS_STAMP(7);
}

// ---------------------------------------------------------------- host driver
template <class K> struct Cfg;
// 384 x 16 keys per tile, 2 CTAs per SM: on an H100 (tools/sort_roofline.py) this beat 256 x 12 at 4 CTAs (the look-back
// wait dominated), 256 x 24 at 2, and 384 x 24 / 384 x 30 / 512 x 16 at 1 CTA per SM (ranking latency with 12-16 warps per SM)
#ifndef RS64_THREADS
#define RS64_THREADS 384
#define RS64_ITEMS 16
#define RS64_MINCTAS 2
#endif
#ifndef RS32_THREADS
#define RS32_THREADS 384
#define RS32_ITEMS 16
#define RS32_MINCTAS 2
#endif
template <> struct Cfg<K32> { static constexpr int THREADS = RS32_THREADS, ITEMS = RS32_ITEMS, MIN_CTAS = RS32_MINCTAS; };
template <> struct Cfg<K64> { static constexpr int THREADS = RS64_THREADS, ITEMS = RS64_ITEMS, MIN_CTAS = RS64_MINCTAS; };
template <> struct Cfg<K128> { static constexpr int THREADS = 256, ITEMS = 8, MIN_CTAS = 4; };

template <class K> inline size_t tile_size() { return (size_t)Cfg<K>::THREADS * Cfg<K>::ITEMS; }
template <class K> inline size_t smem_bytes() { return (size_t)(Cfg<K>::THREADS / 32) * RADIX * 4 + tile_size<K>() * sizeof(K) + tile_size<K>() * 4; }
template <class K> inline size_t status_bytes_needed(uint64_t n, int key_bits) {
    Plan p = make_plan(key_bits);
    uint64_t tiles = (n + tile_size<K>() - 1) / tile_size<K>();
    return (size_t)p.n_passes * tiles * RADIX * 4;
}

}  // namespace rs
