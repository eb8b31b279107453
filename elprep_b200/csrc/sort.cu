// sort.cu -- host drivers for the onesweep radix sort (radix_sort.cuh) and the device prefix sums.
#include "ctx.h"

namespace {

template <class K>
int radix_sort_impl(elp_ctx* c, K* ka, K* kb, uint32_t* va, uint32_t* vb, uint64_t n, int key_bits, bool* result_in_b, const char* tag, int lo_bit) {
    using namespace rs;
    *result_in_b = false;
    if (n == 0) return E_OK;
    if (n >= (1ull << 30)) return c->fail(E_LIMIT, "radix sort: %llu keys exceed the 2^30 limit of the look-back status words", (unsigned long long)n);
    if (lo_bit < 0 || lo_bit + key_bits > (int)(8 * sizeof(K))) return c->fail(E_INVAL, "radix sort: bits [%d, %d) outside the key", lo_bit, lo_bit + key_bits);
    Plan plan = make_plan(key_bits, lo_bit);
    SortWorkspace& ws = c->ws;
    CUDA_TRY(c, ws.ghist.fit(MAX_PASSES * RADIX)); CUDA_TRY(c, ws.gofs.fit(MAX_PASSES * RADIX)); CUDA_TRY(c, ws.counters.fit(MAX_PASSES));
    const size_t tile = tile_size<K>();
    const uint64_t tiles = (n + tile - 1) / tile;
    const size_t need = (size_t)plan.n_passes * tiles * RADIX;   // status words
    if (need > ws.status.cap) {
        if (ws.status.p) cudaStreamSynchronize(c->stream);
        CUDA_TRY(c, ws.status.fit(need + need / 4));
    }
    CUDA_TRY(c, cudaMemsetAsync(ws.ghist.p, 0, MAX_PASSES * RADIX * 4, c->stream));
    CUDA_TRY(c, cudaMemsetAsync(ws.counters.p, 0, MAX_PASSES * 4, c->stream));
    CUDA_TRY(c, cudaMemsetAsync(ws.status.p, 0, need * 4, c->stream));

    int dev_sms = 132;
    cudaDeviceGetAttribute(&dev_sms, cudaDevAttrMultiProcessorCount, c->device);
    std::string nm = std::string("radix_hist_") + tag;
    {
        uint64_t want = (n + 512 * 8 - 1) / (512 * 8);
        int grid = (int)std::min<uint64_t>(want, (uint64_t)dev_sms * 4);
        if (grid < 1) grid = 1;
        c->begin(nm.c_str(), (double)n * sizeof(K));
        rs_hist_kernel<K><<<grid, 512, 0, c->stream>>>(ka, n, plan, ws.ghist.p);
        c->end();
        LAUNCH_CHECK(c);
        c->begin("radix_scan", 0);
        rs_scan_kernel<<<plan.n_passes, RADIX, 0, c->stream>>>(ws.ghist.p, ws.gofs.p);
        c->end();
        LAUNCH_CHECK(c);
    }
    if ((reinterpret_cast<uintptr_t>(va) | reinterpret_cast<uintptr_t>(vb)) & 15) return c->fail(E_INVAL, "radix sort: payload buffers must be 16-byte aligned");
    auto kern = rs_onesweep_kernel<K, Cfg<K>::THREADS, Cfg<K>::ITEMS, Cfg<K>::MIN_CTAS>;
    const size_t smem = smem_bytes<K>();
    CUDA_TRY(c, cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));   // per device: set on every call (cheap)
    nm = std::string("radix_onesweep_") + tag;
    K* in = ka; K* out = kb; uint32_t* vin = va; uint32_t* vout = vb;
    for (int p = 0; p < plan.n_passes; p++) {
        c->begin(nm.c_str(), (double)n * 2.0 * (sizeof(K) + 4));
        kern<<<(unsigned)tiles, Cfg<K>::THREADS, smem, c->stream>>>(in, out, vin, vout, n, plan.shift[p], plan.bits[p], ws.gofs.p + p * RADIX,
                                                                   ws.status.p + (size_t)p * tiles * RADIX, ws.counters.p + p);
        c->end();
        LAUNCH_CHECK(c);
        std::swap(in, out); std::swap(vin, vout);
    }
    *result_in_b = (plan.n_passes & 1) != 0;
    return E_OK;
}

// ---- single-pass exclusive scan (decoupled look-back over ticketed tiles) ----
// A tile loads SCAN_TILE inputs warp-striped (coalesced), transposes them through shared memory so that each thread scans
// SCAN_ITEMS consecutive values, publishes its aggregate, looks back over its predecessors with one warp (32 tiles per
// step) and stores the exclusive prefixes warp-striped again.  Tiles take tickets in start order, so a tile only ever
// waits on tiles that are already running.  Status per tile: flag (0 none, 1 aggregate, 2 inclusive prefix) released
// after the value it guards; aggregate and inclusive prefix live in separate words so a reader never pairs a flag with
// the other value.
constexpr int SCAN_T = 256, SCAN_ITEMS = 16, SCAN_TILE = SCAN_T * SCAN_ITEMS;
__device__ __forceinline__ int scan_pad(int i) { return i + (i >> 4); }   // one pad word per 16: blocked reads are conflict-free

__device__ __forceinline__ uint64_t ld_relaxed_u64(const uint64_t* p) {
    uint64_t r;
    asm volatile("ld.relaxed.gpu.global.u64 %0, [%1];" : "=l"(r) : "l"(p) : "memory");
    return r;
}

template <class TIn>
__global__ void __launch_bounds__(SCAN_T) scan_kernel(const TIn* __restrict__ in, uint64_t n, uint64_t base, uint64_t* __restrict__ out,
                                                     uint64_t* __restrict__ agg, uint64_t* __restrict__ incl, uint32_t* __restrict__ flag,
                                                     uint32_t* __restrict__ counter) {
    constexpr int WARPS = SCAN_T / 32;
    __shared__ uint64_t sh[SCAN_TILE + SCAN_TILE / 16];
    __shared__ uint64_t wofs[WARPS];
    __shared__ uint64_t s_excl;
    __shared__ uint32_t s_tile;
    const unsigned tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    if (tid == 0) s_tile = atomicAdd(counter, 1u);
    __syncthreads();
    const uint32_t tile = s_tile;
    const uint64_t t0 = (uint64_t)tile * SCAN_TILE;
    const uint32_t n_valid = (uint32_t)((n - t0) < (uint64_t)SCAN_TILE ? (n - t0) : (uint64_t)SCAN_TILE);
#pragma unroll
    for (int j = 0; j < SCAN_ITEMS; j++) {
        const int s = j * SCAN_T + tid;
        sh[scan_pad(s)] = (uint32_t)s < n_valid ? (uint64_t)in[t0 + s] : 0;
    }
    __syncthreads();
    uint64_t v[SCAN_ITEMS], sum = 0;
#pragma unroll
    for (int j = 0; j < SCAN_ITEMS; j++) { v[j] = sh[scan_pad(tid * SCAN_ITEMS + j)]; sum += v[j]; }
    uint64_t x = sum;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { uint64_t y = __shfl_up_sync(FULL_MASK, x, o); if (lane >= (unsigned)o) x += y; }
    if (lane == 31) wofs[warp] = x;
    __syncthreads();
    if (warp == 0) {
        const uint64_t wt = lane < WARPS ? wofs[lane] : 0;
        uint64_t wx = wt;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) { uint64_t y = __shfl_up_sync(FULL_MASK, wx, o); if (lane >= (unsigned)o) wx += y; }
        const uint64_t total = __shfl_sync(FULL_MASK, wx, WARPS - 1);
        if (lane < WARPS) wofs[lane] = wx - wt;
        uint64_t excl = 0;
        if (tile == 0) {
            if (lane == 0) { incl[0] = total; st_release_u32(flag, 2u); }
        } else {
            if (lane == 0) { agg[tile] = total; st_release_u32(flag + tile, 1u); }
            // lane l inspects tile t - l; the walk stops at the nearest tile that has its inclusive prefix
            for (int64_t t = (int64_t)tile - 1;; t -= 32) {
                const int64_t tt = t - (int64_t)lane;
                uint32_t f = tt >= 0 ? ld_acquire_u32(flag + tt) : 2u;
                while (__any_sync(FULL_MASK, f == 0)) { if (f == 0) f = ld_acquire_u32(flag + tt); }
                const unsigned stop_mask = __ballot_sync(FULL_MASK, f == 2);
                const unsigned stop = stop_mask ? (unsigned)(__ffs(stop_mask) - 1) : 31u;
                uint64_t val = 0;
                if (lane <= stop && tt >= 0) val = f == 2 ? ld_relaxed_u64(incl + tt) : ld_relaxed_u64(agg + tt);
#pragma unroll
                for (int o = 16; o; o >>= 1) val += __shfl_xor_sync(FULL_MASK, val, o);
                excl += val;
                if (stop_mask) break;
            }
            if (lane == 0) { incl[tile] = excl + total; st_release_u32(flag + tile, 2u); }
        }
        if (lane == 0) {
            s_excl = excl;
            if (t0 + n_valid == n) out[n] = base + excl + total;   // the last tile writes the total
        }
    }
    __syncthreads();
    uint64_t run = base + s_excl + wofs[warp] + x - sum;
#pragma unroll
    for (int j = 0; j < SCAN_ITEMS; j++) { sh[scan_pad(tid * SCAN_ITEMS + j)] = run; run += v[j]; }
    __syncthreads();
#pragma unroll
    for (int j = 0; j < SCAN_ITEMS; j++) {
        const int s = j * SCAN_T + tid;
        if ((uint32_t)s < n_valid) out[t0 + s] = sh[scan_pad(s)];
    }
}

template <class TIn>
int scan_impl(elp_ctx* c, const TIn* in, uint64_t* out, uint64_t n, uint64_t base) {
    if (n == 0) { CUDA_TRY(c, cudaMemcpyAsync(out, &base, 8, cudaMemcpyHostToDevice, c->stream)); cudaStreamSynchronize(c->stream); return E_OK; }
    const uint64_t tiles = (n + SCAN_TILE - 1) / SCAN_TILE;
    if (tiles >= (1ull << 31)) return c->fail(E_LIMIT, "exclusive scan: %llu values exceed the tile count limit", (unsigned long long)n);
    // u32 buffer: [agg u64 x tiles][incl u64 x tiles][flag u32 x tiles][ticket counter]
    CUDA_TRY(c, c->scan_blk.reserve(tiles * 5 + 2, c->stream));
    uint64_t* agg = reinterpret_cast<uint64_t*>(c->scan_blk.p);
    uint64_t* incl = agg + tiles;
    uint32_t* flag = reinterpret_cast<uint32_t*>(incl + tiles);
    CUDA_TRY(c, cudaMemsetAsync(flag, 0, (tiles + 1) * 4, c->stream));
    c->begin("prefix_scan", (double)n * (sizeof(TIn) + 8));
    scan_kernel<TIn><<<(unsigned)tiles, SCAN_T, 0, c->stream>>>(in, n, base, out, agg, incl, flag, flag + tiles);
    c->end(); LAUNCH_CHECK(c);
    return E_OK;
}

}  // namespace

int radix_sort_u32(elp_ctx* c, uint32_t* ka, uint32_t* kb, uint32_t* va, uint32_t* vb, uint64_t n, int key_bits, bool* result_in_b, const char* tag, int lo_bit) {
    return radix_sort_impl<rs::K32>(c, reinterpret_cast<rs::K32*>(ka), reinterpret_cast<rs::K32*>(kb), va, vb, n, key_bits, result_in_b, tag, lo_bit);
}
int radix_sort_u64(elp_ctx* c, uint64_t* ka, uint64_t* kb, uint32_t* va, uint32_t* vb, uint64_t n, int key_bits, bool* result_in_b, const char* tag, int lo_bit) {
    return radix_sort_impl<rs::K64>(c, reinterpret_cast<rs::K64*>(ka), reinterpret_cast<rs::K64*>(kb), va, vb, n, key_bits, result_in_b, tag, lo_bit);
}
int radix_sort_u128(elp_ctx* c, uint64_t* ka, uint64_t* kb, uint32_t* va, uint32_t* vb, uint64_t n, int key_bits, bool* result_in_b, const char* tag, int lo_bit) {
    return radix_sort_impl<rs::K128>(c, reinterpret_cast<rs::K128*>(ka), reinterpret_cast<rs::K128*>(kb), va, vb, n, key_bits, result_in_b, tag, lo_bit);
}
int exclusive_scan_u32_to_u64(elp_ctx* c, const uint32_t* in, uint64_t* out, uint64_t n) { return scan_impl<uint32_t>(c, in, out, n, 0); }
int exclusive_scan_u64_from_u32(elp_ctx* c, const uint32_t* in, uint64_t* out, uint64_t n, uint64_t base) { return scan_impl<uint32_t>(c, in, out, n, base); }
int exclusive_scan_u64(elp_ctx* c, const uint64_t* in, uint64_t* out, uint64_t n, uint64_t base) { return scan_impl<uint64_t>(c, in, out, n, base); }

#ifdef RS_TIMING
#include <cstdio>
// prints the mean clock cycles between the phase stamps of the sampled tiles of the LAST pass
void rs_dump_timing() {
    static long long h[8 * 4096];
    cudaDeviceSynchronize();
    cudaMemcpyFromSymbol(h, rs::rs_tstamp, sizeof h);
    double acc[7] = {0, 0, 0, 0, 0, 0, 0}; int cnt = 0;
    for (int t = 8; t < 4096; t++) { const long long* p = h + 8 * t; if (p[7] <= p[0] || p[0] == 0) continue; for (int k = 0; k < 7; k++) acc[k] += (double)(p[k + 1] - p[k]); cnt++; }
    const char* names[7] = {"load-issue", "rank", "scan+lookback", "scatter-smem", "write-keys", "load-vals", "write-vals"};
    fprintf(stderr, "onesweep phase cycles over %d sampled tiles:", cnt);
    for (int k = 0; k < 7; k++) fprintf(stderr, "  %s %.0f", names[k], cnt ? acc[k] / cnt : 0.0);
    fprintf(stderr, "\n");
}
#endif
