// tagwalk.cuh -- the one statement of the BAM optional-field grammar (sam/bam-files.go:369-397) for the write-phase kernels: where a field
// ends, and whether the output field filter (elp_set_output_filter) drops it.  format_line (sam_format.cu) and the BAM field-filter
// kernels (bam_ingest.cu) walk a record's fields with field_end; the ingest validated every record, so no bound is checked here beyond
// the record's end.  field_end is warp-collective (Z / H search their NUL with a ballot): every lane of the warp must call it with the
// same arguments.
#pragma once
#include <cstdint>
#include "common.cuh"

namespace tagwalk {

__device__ __forceinline__ uint32_t rd32(const uint8_t* p) { return (uint32_t)p[0] | ((uint32_t)p[1] << 8) | ((uint32_t)p[2] << 16) | ((uint32_t)p[3] << 24); }

// first NUL at or after `from` (the ingest checked that there is one before n)
__device__ __forceinline__ uint64_t find_nul(const uint8_t* p, uint64_t from, uint64_t n) {
    const unsigned lane = threadIdx.x & 31;
    for (uint64_t b = from; b < n; b += 32) {
        const unsigned m = __ballot_sync(FULL_MASK, b + lane < n && p[b + lane] == 0);
        if (m) return b + __ffs(m) - 1;
    }
    return n;
}

// bytes per element of a B array of subtype sub (c C: 1, s S: 2, i I f: 4)
__device__ __forceinline__ int elem_size(uint8_t sub) { return (sub == 'c' || sub == 'C') ? 1 : ((sub == 's' || sub == 'S') ? 2 : 4); }

// end of the field whose tag starts at r[t] (t + 3 <= rec): tag[2] type[1] value; Z / H end behind their NUL, B is subtype, count and
// count x element size.  A type the ingest does not accept ends the walk (rec).
__device__ __forceinline__ uint64_t field_end(const uint8_t* r, uint64_t t, uint64_t rec) {
    const uint64_t v = t + 3;
    switch (r[t + 2]) {
        case 'A': case 'c': case 'C': return v + 1;
        case 's': case 'S': return v + 2;
        case 'i': case 'I': case 'f': return v + 4;
        case 'Z': case 'H': return find_nul(r, v, rec) + 1;
        case 'B': return v + 5 + (uint64_t)elem_size(r[v]) * rd32(r + v + 1);
        default: return rec;
    }
}

// the output field filter: bit (t0 | t1 << 8) of the 65 536-bit table is set when the field with tag t0 t1 is dropped
__device__ __forceinline__ bool dropped(const uint32_t* __restrict__ tab, uint8_t t0, uint8_t t1) {
    const uint32_t i = (uint32_t)t0 | ((uint32_t)t1 << 8);
    return (__ldg(tab + (i >> 5)) >> (i & 31)) & 1u;
}

}  // namespace tagwalk
