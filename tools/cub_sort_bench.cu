// cub_sort_bench.cu -- YARD-STICK ONLY (SURVEY.md section 7 step 6): cub::DeviceRadixSort::SortPairs on the same problem the
// library's own onesweep sort is timed on (30 M 64-bit keys, 34 / 40 / 64 significant bits, 32-bit payload), on the same box.
// A stand-alone binary: nothing of CUB is linked into libelprep_b200.so or used on the product path.
//   nvcc -O3 -std=c++17 -gencode arch=compute_90a,code=sm_90a -o tools/_build/cub_sort_bench tools/cub_sort_bench.cu
#include <cub/cub.cuh>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <vector>

static uint64_t mix(uint64_t z) { z += 0x9E3779B97F4A7C15ULL; z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ULL; z = (z ^ (z >> 27)) * 0x94D049BB133111EBULL; return z ^ (z >> 31); }

int main(int argc, char** argv) {
    const size_t n = argc > 1 ? strtoull(argv[1], nullptr, 10) : 30000000ull;
    std::vector<uint64_t> hk(n); std::vector<uint32_t> hv(n);
    uint64_t *ka, *kb; uint32_t *va, *vb;
    cudaMalloc(&ka, n * 8); cudaMalloc(&kb, n * 8); cudaMalloc(&va, n * 4); cudaMalloc(&vb, n * 4);
    cudaEvent_t e0, e1; cudaEventCreate(&e0); cudaEventCreate(&e1);
    const int bits_list[3] = {34, 40, 64};
    printf("{\"tool\": \"cub::DeviceRadixSort::SortPairs (CUB %d, yard-stick only)\", \"n\": %zu, \"results\": [", CUB_VERSION, n);
    for (int bi = 0; bi < 3; bi++) {
        const int bits = bits_list[bi];
        for (size_t i = 0; i < n; i++) { hk[i] = mix(i) & (bits == 64 ? ~0ull : ((1ull << bits) - 1)); hv[i] = (uint32_t)i; }
        size_t tmp_bytes = 0; void* tmp = nullptr;
        cub::DoubleBuffer<uint64_t> dk(ka, kb); cub::DoubleBuffer<uint32_t> dv(va, vb);
        cub::DeviceRadixSort::SortPairs(nullptr, tmp_bytes, dk, dv, (int)n, 0, bits);
        cudaMalloc(&tmp, tmp_bytes);
        float best = 1e30f;
        for (int rep = 0; rep < 5; rep++) {
            cudaMemcpy(ka, hk.data(), n * 8, cudaMemcpyHostToDevice); cudaMemcpy(va, hv.data(), n * 4, cudaMemcpyHostToDevice);   // also evicts L2
            cub::DoubleBuffer<uint64_t> k2(ka, kb); cub::DoubleBuffer<uint32_t> v2(va, vb);
            cudaEventRecord(e0);
            cub::DeviceRadixSort::SortPairs(tmp, tmp_bytes, k2, v2, (int)n, 0, bits);
            cudaEventRecord(e1); cudaEventSynchronize(e1);
            float ms; cudaEventElapsedTime(&ms, e0, e1);
            if (rep > 0 && ms < best) best = ms;
            if (rep == 4) {   // sortedness check
                cudaMemcpy(hk.data(), k2.Current(), n * 8, cudaMemcpyDeviceToHost);
                bool ok = true; for (size_t i = 1; i < n; i++) if (hk[i - 1] > hk[i]) { ok = false; break; }
                const int passes = (bits + 7) / 8;
                printf("%s{\"key_bits\": %d, \"ms\": %.4f, \"sorted\": %s, \"passes_8bit\": %d, \"GBps_alg\": %.1f, \"frac_of_3350\": %.3f}", bi ? ", " : "", bits, best, ok ? "true" : "false",
                       passes, (double)n * (8.0 + 2.0 * passes * 12.0) / (best * 1e-3) / 1e9, (double)n * (8.0 + 2.0 * passes * 12.0) / (best * 1e-3) / 1e9 / 3350.0);
            }
        }
        cudaFree(tmp);
    }
    // plain device copy for context (the roofline denominator is measured the same way)
    cudaEventRecord(e0); for (int r = 0; r < 10; r++) cudaMemcpyAsync(kb, ka, n * 8, cudaMemcpyDeviceToDevice); cudaEventRecord(e1); cudaEventSynchronize(e1);
    float ms; cudaEventElapsedTime(&ms, e0, e1);
    printf("], \"d2d_copy_GBps\": %.1f}\n", 10.0 * 2.0 * n * 8 / (ms * 1e-3) / 1e9);
    return 0;
}
