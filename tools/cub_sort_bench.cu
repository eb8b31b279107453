// cub_sort_bench.cu -- YARD-STICK ONLY (SURVEY.md section 7 step 6): cub::DeviceRadixSort::SortPairs on the same problems the
// library's own onesweep sort is timed on (tools/sort_roofline.py: u64 keys, 30 M, 32 bits; u64 keys, 15 M, 62 bits; u32 keys,
// 30 M, 32 bits; plus the older 34 / 40 / 64-bit u64 cases), 32-bit payload, on the same box.
// A stand-alone binary: nothing of CUB is linked into libelprep_b200.so or used on the product path.
//   nvcc -O3 -std=c++17 -gencode arch=compute_90a,code=sm_90a -o tools/_build/cub_sort_bench tools/cub_sort_bench.cu
#include <cub/cub.cuh>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <vector>

static uint64_t mix(uint64_t z) { z += 0x9E3779B97F4A7C15ULL; z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ULL; z = (z ^ (z >> 27)) * 0x94D049BB133111EBULL; return z ^ (z >> 31); }

// best of 4 timed sorts (after one warm-up) of n random keys with `bits` significant bits; prints one JSON object
template <class K>
static void run(size_t n, int bits, bool first) {
    std::vector<K> hk(n); std::vector<uint32_t> hv(n);
    for (size_t i = 0; i < n; i++) { hk[i] = (K)(mix(i) & (bits == 64 ? ~0ull : ((1ull << bits) - 1))); hv[i] = (uint32_t)i; }
    K *ka, *kb; uint32_t *va, *vb;
    cudaMalloc(&ka, n * sizeof(K)); cudaMalloc(&kb, n * sizeof(K)); cudaMalloc(&va, n * 4); cudaMalloc(&vb, n * 4);
    cudaEvent_t e0, e1; cudaEventCreate(&e0); cudaEventCreate(&e1);
    size_t tmp_bytes = 0; void* tmp = nullptr;
    cub::DoubleBuffer<K> dk(ka, kb); cub::DoubleBuffer<uint32_t> dv(va, vb);
    cub::DeviceRadixSort::SortPairs(nullptr, tmp_bytes, dk, dv, (int)n, 0, bits);
    cudaMalloc(&tmp, tmp_bytes);
    float best = 1e30f;
    for (int rep = 0; rep < 5; rep++) {
        cudaMemcpy(ka, hk.data(), n * sizeof(K), cudaMemcpyHostToDevice); cudaMemcpy(va, hv.data(), n * 4, cudaMemcpyHostToDevice);   // also evicts L2
        cub::DoubleBuffer<K> k2(ka, kb); cub::DoubleBuffer<uint32_t> v2(va, vb);
        cudaEventRecord(e0);
        cub::DeviceRadixSort::SortPairs(tmp, tmp_bytes, k2, v2, (int)n, 0, bits);
        cudaEventRecord(e1); cudaEventSynchronize(e1);
        float ms; cudaEventElapsedTime(&ms, e0, e1);
        if (rep > 0 && ms < best) best = ms;
        if (rep == 4) {   // sortedness check
            cudaMemcpy(hk.data(), k2.Current(), n * sizeof(K), cudaMemcpyDeviceToHost);
            bool ok = true; for (size_t i = 1; i < n; i++) if (hk[i - 1] > hk[i]) { ok = false; break; }
            const int passes = (bits + 7) / 8;
            const double kbytes = (double)sizeof(K), alg = (double)n * (kbytes + 2.0 * passes * (kbytes + 4.0));
            printf("%s{\"key\": \"u%d\", \"n\": %zu, \"key_bits\": %d, \"ms\": %.4f, \"sorted\": %s, \"passes_8bit\": %d, \"GBps_alg\": %.1f, \"frac_of_3350\": %.3f}",
                   first ? "" : ", ", (int)(8 * sizeof(K)), n, bits, best, ok ? "true" : "false", passes, alg / (best * 1e-3) / 1e9, alg / (best * 1e-3) / 1e9 / 3350.0);
        }
    }
    cudaFree(tmp); cudaFree(ka); cudaFree(kb); cudaFree(va); cudaFree(vb);
    cudaEventDestroy(e0); cudaEventDestroy(e1);
}

int main(int argc, char** argv) {
    const size_t n = argc > 1 ? strtoull(argv[1], nullptr, 10) : 30000000ull;
    printf("{\"tool\": \"cub::DeviceRadixSort::SortPairs (CUB %d, yard-stick only)\", \"results\": [", CUB_VERSION);
    run<uint64_t>(n, 32, true);
    run<uint64_t>(n / 2, 62, false);
    run<uint32_t>(n, 32, false);
    const int bits_list[3] = {34, 40, 64};
    for (int bits : bits_list) run<uint64_t>(n, bits, false);
    // plain device copy for context (the roofline denominator is measured the same way)
    uint64_t *a, *b; cudaMalloc(&a, n * 8); cudaMalloc(&b, n * 8);
    cudaEvent_t e0, e1; cudaEventCreate(&e0); cudaEventCreate(&e1);
    cudaMemcpy(b, a, n * 8, cudaMemcpyDeviceToDevice);
    cudaEventRecord(e0); for (int r = 0; r < 10; r++) cudaMemcpyAsync(b, a, n * 8, cudaMemcpyDeviceToDevice); cudaEventRecord(e1); cudaEventSynchronize(e1);
    float ms; cudaEventElapsedTime(&ms, e0, e1);
    printf("], \"d2d_copy_GBps\": %.1f}\n", 10.0 * 2.0 * n * 8 / (ms * 1e-3) / 1e9);
    return 0;
}
