// refhot.cuh -- reference bases -> the one-hot nibbles every BQSR gather kernel reads, low nibble first (A/a/* 1, C/c 2, G/g 4, T/t 8,
// everything else 0: never equal to a read base).  Packed by pack_reference (bqsr_gather.cu, elp_set_reference) and elp_load_reference
// (reference_load.cu).  Include after ctx.h.
#pragma once

namespace {

__device__ __forceinline__ uint32_t hot_nibble(uint8_t b) {
    if (b == 'A' || b == 'a' || b == '*') return 1;
    if (b == 'C' || b == 'c') return 2;
    if (b == 'G' || b == 'g') return 4;
    if (b == 'T' || b == 't') return 8;
    return 0;
}

// ref[0, n) -> out[0, n_out): the whole contig, one output byte (two bases) per thread
__global__ void __launch_bounds__(256) ref_pack_hot_kernel(const uint8_t* __restrict__ ref, uint64_t n, uint8_t* __restrict__ out, uint64_t n_out) {
    const uint64_t t = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= n_out) return;
    uint32_t v = 0;
#pragma unroll
    for (int h = 0; h < 2; h++) {
        const uint64_t j = 2 * t + h;
        if (j < n) v |= hot_nibble(ref[j]) << (4 * h);
    }
    out[t] = (uint8_t)v;
}

// ref[0, n) are the bases [b0, b0 + n) of a contig: their nibbles are ORed into the zeroed out, so that a span that starts or ends at an
// odd base shares its edge byte with the span before or after it (spans of one contig run in stream order)
__global__ void __launch_bounds__(256) ref_pack_span_kernel(const uint8_t* __restrict__ ref, uint64_t n, uint64_t b0, uint8_t* __restrict__ out) {
    const uint64_t t = b0 / 2 + (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;   // output byte: bases 2t, 2t + 1
    if (2 * t >= b0 + n) return;
    uint32_t v = 0;
#pragma unroll
    for (int h = 0; h < 2; h++) {
        const uint64_t j = 2 * t + h;
        if (j >= b0 && j < b0 + n) v |= hot_nibble(ref[j - b0]) << (4 * h);
    }
    out[t] |= (uint8_t)v;
}

}  // namespace
