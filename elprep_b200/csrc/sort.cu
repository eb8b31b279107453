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
    Workspace& ws = c->ws;
    if (!ws.ghist) {
        CUDA_TRY(c, cudaMalloc(&ws.ghist, MAX_PASSES * RADIX * 4));
        CUDA_TRY(c, cudaMalloc(&ws.gofs, MAX_PASSES * RADIX * 4));
        CUDA_TRY(c, cudaMalloc(&ws.counters, MAX_PASSES * 4));
    }
    const size_t tile = tile_size<K>();
    const uint64_t tiles = (n + tile - 1) / tile;
    const size_t need = (size_t)plan.n_passes * tiles * RADIX * 4;
    if (need > ws.status_bytes) {
        if (ws.status) { cudaStreamSynchronize(c->stream); cudaFree(ws.status); }
        ws.status_bytes = need + need / 4;
        CUDA_TRY(c, cudaMalloc(&ws.status, ws.status_bytes));
    }
    CUDA_TRY(c, cudaMemsetAsync(ws.ghist, 0, MAX_PASSES * RADIX * 4, c->stream));
    CUDA_TRY(c, cudaMemsetAsync(ws.counters, 0, MAX_PASSES * 4, c->stream));
    CUDA_TRY(c, cudaMemsetAsync(ws.status, 0, need, c->stream));

    int dev_sms = 132;
    cudaDeviceGetAttribute(&dev_sms, cudaDevAttrMultiProcessorCount, c->device);
    std::string nm = std::string("radix_hist_") + tag;
    {
        uint64_t want = (n + 512 * 8 - 1) / (512 * 8);
        int grid = (int)std::min<uint64_t>(want, (uint64_t)dev_sms * 4);
        if (grid < 1) grid = 1;
        c->begin(nm.c_str(), (double)n * sizeof(K));
        rs_hist_kernel<K><<<grid, 512, 0, c->stream>>>(ka, n, plan, ws.ghist);
        c->end();
        LAUNCH_CHECK(c);
        c->begin("radix_scan", 0);
        rs_scan_kernel<<<plan.n_passes, RADIX, 0, c->stream>>>(ws.ghist, ws.gofs);
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
        kern<<<(unsigned)tiles, Cfg<K>::THREADS, smem, c->stream>>>(in, out, vin, vout, n, plan.shift[p], plan.bits[p], ws.gofs + p * RADIX,
                                                                   ws.status + (size_t)p * tiles * RADIX, ws.counters + p);
        c->end();
        LAUNCH_CHECK(c);
        std::swap(in, out); std::swap(vin, vout);
    }
    *result_in_b = (plan.n_passes & 1) != 0;
    return E_OK;
}

// ---- 3-kernel exclusive scan (block reduce -> scan of block sums -> downsweep) ----
constexpr int SCAN_T = 512, SCAN_ITEMS = 8, SCAN_TILE = SCAN_T * SCAN_ITEMS;

template <class TIn>
__global__ void __launch_bounds__(SCAN_T) scan_reduce_kernel(const TIn* __restrict__ in, uint64_t n, uint64_t* __restrict__ blk) {
    __shared__ uint64_t ws[SCAN_T / 32];
    uint64_t base = (uint64_t)blockIdx.x * SCAN_TILE, s = 0;
    for (int k = 0; k < SCAN_ITEMS; k++) { uint64_t i = base + (uint64_t)k * SCAN_T + threadIdx.x; if (i < n) s += (uint64_t)in[i]; }
    for (int o = 16; o; o >>= 1) s += __shfl_down_sync(FULL_MASK, s, o);
    if ((threadIdx.x & 31) == 0) ws[threadIdx.x >> 5] = s;
    __syncthreads();
    if (threadIdx.x == 0) { uint64_t t = 0; for (int i = 0; i < SCAN_T / 32; i++) t += ws[i]; blk[blockIdx.x] = t; }
}
__global__ void __launch_bounds__(1024) scan_blocks_kernel(uint64_t* __restrict__ blk, uint64_t nblk, uint64_t base) {
    __shared__ uint64_t ws[32];
    __shared__ uint64_t carry;
    if (threadIdx.x == 0) carry = base;
    __syncthreads();
    for (uint64_t b0 = 0; b0 < nblk; b0 += 1024) {
        uint64_t i = b0 + threadIdx.x;
        uint64_t v = i < nblk ? blk[i] : 0, x = v;
        unsigned lane = threadIdx.x & 31, w = threadIdx.x >> 5;
        for (int o = 1; o < 32; o <<= 1) { uint64_t y = __shfl_up_sync(FULL_MASK, x, o); if (lane >= (unsigned)o) x += y; }
        if (lane == 31) ws[w] = x;
        __syncthreads();
        uint64_t add = carry;
        for (unsigned k = 0; k < w; k++) add += ws[k];
        if (i < nblk) blk[i] = x - v + add;
        __syncthreads();
        if (threadIdx.x == 1023) carry = x + add;
        __syncthreads();
    }
}
template <class TIn>
__global__ void __launch_bounds__(SCAN_T) scan_down_kernel(const TIn* __restrict__ in, uint64_t n, const uint64_t* __restrict__ blk, uint64_t* __restrict__ out) {
    __shared__ uint64_t ws[SCAN_T / 32];
    uint64_t base = (uint64_t)blockIdx.x * SCAN_TILE + (uint64_t)threadIdx.x * SCAN_ITEMS;   // blocked arrangement
    uint64_t v[SCAN_ITEMS], s = 0;
    for (int k = 0; k < SCAN_ITEMS; k++) { uint64_t i = base + k; v[k] = i < n ? (uint64_t)in[i] : 0; s += v[k]; }
    uint64_t x = s;
    unsigned lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    for (int o = 1; o < 32; o <<= 1) { uint64_t y = __shfl_up_sync(FULL_MASK, x, o); if (lane >= (unsigned)o) x += y; }
    if (lane == 31) ws[w] = x;
    __syncthreads();
    uint64_t add = blk[blockIdx.x];
    for (unsigned k = 0; k < w; k++) add += ws[k];
    uint64_t run = x - s + add;
    for (int k = 0; k < SCAN_ITEMS; k++) { uint64_t i = base + k; if (i < n) out[i] = run; run += v[k]; }
    if (base <= n && n < base + SCAN_ITEMS) {   // the thread owning position n writes the total
        uint64_t r2 = x - s + add;
        for (int k = 0; k < SCAN_ITEMS && base + k < n; k++) r2 += v[k];
        out[n] = r2;
    }
}

template <class TIn>
int scan_impl(elp_ctx* c, const TIn* in, uint64_t* out, uint64_t n, uint64_t base) {
    if (n == 0) { CUDA_TRY(c, cudaMemcpyAsync(out, &base, 8, cudaMemcpyHostToDevice, c->stream)); cudaStreamSynchronize(c->stream); return E_OK; }
    uint64_t nblk = (n + SCAN_TILE - 1) / SCAN_TILE;
    // position n may fall into block index n/SCAN_TILE == nblk when n is a multiple of the tile: launch one more block for it
    uint64_t nblk_down = n / SCAN_TILE + 1;
    CUDA_TRY(c, c->scan_blk.reserve((nblk_down + 1) * 2, c->stream));   // u32 buffer reused as u64 storage
    uint64_t* blk = reinterpret_cast<uint64_t*>(c->scan_blk.p);
    CUDA_TRY(c, cudaMemsetAsync(blk, 0, (nblk_down + 1) * 8, c->stream));
    c->begin("scan_reduce", (double)n * sizeof(TIn));
    scan_reduce_kernel<TIn><<<(unsigned)nblk, SCAN_T, 0, c->stream>>>(in, n, blk);
    c->end(); LAUNCH_CHECK(c);
    c->begin("scan_blocks", 0);
    scan_blocks_kernel<<<1, 1024, 0, c->stream>>>(blk, nblk_down, base);
    c->end(); LAUNCH_CHECK(c);
    c->begin("scan_down", (double)n * (sizeof(TIn) + 8));
    scan_down_kernel<TIn><<<(unsigned)nblk_down, SCAN_T, 0, c->stream>>>(in, n, blk, out);
    c->end(); LAUNCH_CHECK(c);
    return E_OK;
}

}  // namespace

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
