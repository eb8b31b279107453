// common.cuh -- shared device/host helpers for the elprep_b200 CUDA library (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <cstdint>
#include <cstdio>
#include <string>

#define ELP_WARP 32
#define FULL_MASK 0xffffffffu

// ---- status codes (mirror include/elprep_b200.h) ----
#define E_OK 0
#define E_INVAL (-1)
#define E_NODEVICE (-2)
#define E_CUDA (-3)
#define E_NOMEM (-4)
#define E_QUAL (-10)
#define E_NORG (-11)
#define E_CYCLE (-12)
#define E_CLIP (-13)
#define E_REFEND (-14)
#define E_LIMIT (-15)
#define E_TILE (-17)
#define E_BAM (-18)
#define E_SAM (-20)
#define E_STATE (-16)

// device-side error word bits (one u32 in global memory, OR-ed by kernels, read by the host after the phase)
#define DERR_QUAL 0x1u
#define DERR_NORG 0x2u
#define DERR_CYCLE 0x4u
#define DERR_CLIP 0x8u
#define DERR_REFEND 0x10u
#define DERR_CIGAR_LIMIT 0x20u
#define DERR_QUAL_RANGE 0x40u
#define DERR_READLEN_LIMIT 0x80u
#define DERR_TILE 0x100u         // QNAME tile/x/y field that strconv.ParseInt rejects (mark-optical-duplicates.go:57-64)
#define DERR_TILE_RANGE 0x200u   // tile/x/y outside int32
#define DERR_BAM 0x400u          // malformed BAM record (lengths / optional fields do not add up)
#define DERR_BAM_RG 0x800u       // RG:Z value that is not an @RG ID of the header
#define DERR_BAM_CG 0x1000u      // CG:B long-CIGAR convention
#define DERR_CLEANSAM 0x4000u    // "Unexpected non-0 relative clipping position in CleanSam." (filters/utils.go:96)
#define DERR_SPREAD_NAME 0x2000u // QNAME longer than a spread record holds (comm.cu)

// FLAG bits (sam/sam-types.go:485-520)
#define F_MULTIPLE 0x1
#define F_PROPER 0x2
#define F_UNMAPPED 0x4
#define F_NEXTUNMAPPED 0x8
#define F_REVERSED 0x10
#define F_NEXTREVERSED 0x20
#define F_FIRST 0x40
#define F_LAST 0x80
#define F_SECONDARY 0x100
#define F_QCFAILED 0x200
#define F_DUPLICATE 0x400
#define F_SUPPLEMENTARY 0x800

__device__ __forceinline__ unsigned lane_id() { return threadIdx.x & 31; }
__device__ __forceinline__ unsigned lanemask_lt() { unsigned m; asm("mov.u32 %0, %%lanemask_lt;" : "=r"(m)); return m; }

// streaming (read-once) loads: bypass L1 allocation
__device__ __forceinline__ uint4 ld_stream_u4(const void* p) {
    uint4 r;
    asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(p));
    return r;
}
__device__ __forceinline__ uint64_t ld_stream_u64(const uint64_t* p) {
    uint64_t r;
    asm volatile("ld.global.nc.L1::no_allocate.u64 %0, [%1];" : "=l"(r) : "l"(p));
    return r;
}
__device__ __forceinline__ uint32_t ld_stream_u32(const uint32_t* p) {
    uint32_t r;
    asm volatile("ld.global.nc.L1::no_allocate.u32 %0, [%1];" : "=r"(r) : "l"(p));
    return r;
}
// acquire/release accessors for decoupled look-back status words
__device__ __forceinline__ uint32_t ld_acquire_u32(const uint32_t* p) {
    uint32_t r;
    asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(r) : "l"(p) : "memory");
    return r;
}
__device__ __forceinline__ void st_release_u32(uint32_t* p, uint32_t v) {
    asm volatile("st.release.gpu.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}

__device__ __forceinline__ uint32_t ld_relaxed_u32(const uint32_t* p) {
    uint32_t r;
    asm volatile("ld.relaxed.gpu.global.u32 %0, [%1];" : "=r"(r) : "l"(p) : "memory");
    return r;
}
__device__ __forceinline__ void st_relaxed_u32(uint32_t* p, uint32_t v) {
    asm volatile("st.relaxed.gpu.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}

// set FLAG bits on a u16 column from concurrent threads (two reads share one 32-bit word)
__device__ __forceinline__ void atomic_or_u16(uint16_t* col, uint64_t i, uint16_t bits) {
    uint32_t* w = reinterpret_cast<uint32_t*>(col) + (i >> 1);
    atomicOr(w, (uint32_t)bits << ((i & 1) * 16));
}

__host__ __device__ __forceinline__ int bits_for(uint64_t maxval) {  // number of bits to represent values 0..maxval
    int b = 0;
    while (maxval) { b++; maxval >>= 1; }
    return b;
}

// byte-lexicographic compare of two QNAMEs (Go string <, sam/sam-types.go:439-446)
__device__ __forceinline__ int qname_compare(const uint8_t* q, uint64_t a0, uint64_t a1, uint64_t b0, uint64_t b1) {
    uint64_t la = a1 - a0, lb = b1 - b0, m = la < lb ? la : lb;
    for (uint64_t k = 0; k < m; k++) {
        int d = (int)q[a0 + k] - (int)q[b0 + k];
        if (d) return d;
    }
    return la < lb ? -1 : (la > lb ? 1 : 0);
}

struct DeviceRanges {            // filled by the adapt kernel, read back by the host to size the sort keys
    int32_t pos_max, upos_min, upos_max, score_max, lseq_max, qname_max;
    uint32_t qual_present[4];    // bit q set if QUAL value q (0..127) occurs
    uint32_t n_entering, n_true_pairs;
};
