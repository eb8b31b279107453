// regions.cuh -- the device side of RemoveNonOverlappingReads (filters/simple-filters.go:310-328), shared by the ingest filter
// (bam_keep_kernel, bam_ingest.cu) and the filter after duplicate marking (target_keep_kernel, target_regions.cu).
#pragma once
#include <cstdint>

// intervals.Overlap (intervals/intervals.go:146-164) over one contig's flattened, start-sorted (start, end) pairs
__device__ inline bool overlap_any(const int32_t* __restrict__ iv, uint64_t n, int32_t start, int32_t end) {
    const int32_t end_1 = (int32_t)((uint32_t)end - 1u), start_1 = (int32_t)((uint32_t)start - 1u);   // end-1, start-1 in Go's int32: they wrap
    int64_t left = 0, right = (int64_t)n - 1;
    while (left <= right) {
        const int64_t mid = (left + right) / 2;
        const int32_t is = iv[2 * mid], ie = iv[2 * mid + 1];
        if (is > end_1) right = mid - 1;
        else if (ie <= start_1) left = mid + 1;
        else return true;
    }
    return false;
}
