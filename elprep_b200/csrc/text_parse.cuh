// text_parse.cuh -- pieces shared by the device parsers of text inputs: SAM alignment lines (sam_ingest.cu) and .elsites files
// (known_sites.cu).
//   sam_count_kernel / sam_lines_kernel   the line finder: '\n' count per 64-byte chunk, exclusive scan (host), line starts
//   parse_dec                             strconv.ParseInt / ParseUint, base 10
//   name_entry, refid_of                  lookups in the context's dictionary of "*" and the @SQ SN names (NameDict, ctx.h), and its
//                                         upload (name_dict_upload)
#pragma once
#include <algorithm>
#include <map>
#include <string>
#include <vector>
#include "ctx.h"

namespace {

constexpr int SAM_CHUNK = 64;   // text bytes per thread of the line finder; the text is padded to a multiple of it plus 64 zero bytes

// ---- line finder ----
__device__ __forceinline__ uint32_t nl_mask(uint32_t w) { return __vcmpeq4(w, 0x0a0a0a0au); }   // 0xff in every '\n' byte

__global__ void __launch_bounds__(256) sam_count_kernel(const uint8_t* __restrict__ t, uint64_t n_chunks, uint32_t* __restrict__ cnt) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_chunks) return;
    const uint4* q = reinterpret_cast<const uint4*>(t + i * SAM_CHUNK);
    uint32_t k = 0;
#pragma unroll
    for (int j = 0; j < SAM_CHUNK / 16; j++) { const uint4 v = q[j]; k += __popc(nl_mask(v.x)) + __popc(nl_mask(v.y)) + __popc(nl_mask(v.z)) + __popc(nl_mask(v.w)); }
    cnt[i] = k >> 3;
}
// ls[j + 1] = the byte after the j-th '\n'
__global__ void __launch_bounds__(256) sam_lines_kernel(const uint8_t* __restrict__ t, uint64_t n_chunks, const uint64_t* __restrict__ off, uint64_t* __restrict__ ls) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_chunks) return;
    const uint4* q = reinterpret_cast<const uint4*>(t + i * SAM_CHUNK);
    uint64_t o = off[i] + 1;
#pragma unroll
    for (int j = 0; j < SAM_CHUNK / 16; j++) {
        const uint4 v = q[j];
        const uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
        for (int h = 0; h < 4; h++)
            for (uint32_t m = nl_mask(w[h]) & 0x01010101u; m; m &= m - 1)
                ls[o++] = i * SAM_CHUNK + 16 * j + 4 * h + ((__ffs(m) - 1) >> 3) + 1;
    }
}

// strconv.ParseInt (sgn) / ParseUint (!sgn), base 10, accepted only inside [lo, hi] (every range used here lies in [-2^31, 2^32-1])
__device__ bool parse_dec(const uint8_t* p, uint64_t n, bool sgn, int64_t lo, int64_t hi, int64_t* v) {
    uint64_t i = 0; bool neg = false;
    if (sgn && n && (p[0] == '+' || p[0] == '-')) { neg = p[0] == '-'; i = 1; }
    if (i >= n) return false;
    uint64_t m = 0;
    for (; i < n; i++) {
        const uint32_t d = (uint32_t)p[i] - '0';
        if (d > 9) return false;
        if (m < (1ull << 40)) m = m * 10 + d;   // saturates far above any accepted range
    }
    const int64_t x = neg ? -(int64_t)m : (int64_t)m;
    if (x < lo || x > hi) return false;
    *v = x;
    return true;
}

// the entry whose name is s[0, n), or -1
__device__ int name_entry(const NameDict& D, const uint8_t* s, uint64_t n) {
    int lo = 0, hi = D.n - 1;
    while (lo <= hi) {
        const int mid = (lo + hi) >> 1;
        const uint8_t* q = D.names + D.off[mid];
        const uint64_t qn = D.off[mid + 1] - D.off[mid];
        int cmp = 0;
        for (uint64_t j = 0; j < qn && j < n && !cmp; j++) cmp = (int)q[j] - (int)s[j];
        if (!cmp) cmp = qn < n ? -1 : (qn > n ? 1 : 0);
        if (!cmp) return mid;
        if (cmp < 0) lo = mid + 1; else hi = mid - 1;
    }
    return -1;
}
// dictTable of formatBamAlignment / AddREFID: "*" -> -1, @SQ SN -> index (the last of equal names wins), anything else -> -1
__device__ __forceinline__ int32_t refid_of(const NameDict& D, const uint8_t* s, uint64_t n) {
    const int e = name_entry(D, s, n);
    return e < 0 ? -1 : D.id[e];
}

// the dictionary of the names src (index = refid) into D, uploaded with blocking copies on first use
int name_dict_build(elp_ctx* c, NameDictBufs& D, const std::vector<std::string>& src) {
    if (D.n) return E_OK;
    std::map<std::string, std::vector<int32_t>> dict;
    dict["*"];
    for (int i = 0; i < (int)src.size(); i++) dict[src[i]].push_back(i);
    std::vector<uint8_t> names; std::vector<uint32_t> off(1, 0), all_off(1, 0); std::vector<int32_t> id, all;
    for (auto& kv : dict) {
        names.insert(names.end(), kv.first.begin(), kv.first.end()); off.push_back((uint32_t)names.size());
        id.push_back(kv.second.empty() ? -1 : kv.second.back());
        if (kv.first != "*") all.insert(all.end(), kv.second.begin(), kv.second.end());
        all_off.push_back((uint32_t)all.size());
    }
    CUDA_TRY(c, D.names.fit(std::max<size_t>(names.size(), 1)));
    CUDA_TRY(c, D.off.fit(off.size()));
    CUDA_TRY(c, D.id.fit(id.size()));
    CUDA_TRY(c, D.all_off.fit(all_off.size()));
    CUDA_TRY(c, D.all.fit(std::max<size_t>(all.size(), 1)));
    CUDA_TRY(c, cudaMemcpy(D.names.p, names.data(), names.size(), cudaMemcpyHostToDevice));
    CUDA_TRY(c, cudaMemcpy(D.off.p, off.data(), off.size() * 4, cudaMemcpyHostToDevice));
    CUDA_TRY(c, cudaMemcpy(D.id.p, id.data(), id.size() * 4, cudaMemcpyHostToDevice));
    CUDA_TRY(c, cudaMemcpy(D.all_off.p, all_off.data(), all_off.size() * 4, cudaMemcpyHostToDevice));
    if (!all.empty()) CUDA_TRY(c, cudaMemcpy(D.all.p, all.data(), all.size() * 4, cudaMemcpyHostToDevice));
    D.n = (int)id.size();
    return E_OK;
}
// the dictionary of the context's elp_config.contig_names (c->names)
int name_dict_upload(elp_ctx* c) { return name_dict_build(c, c->names, c->contig_names); }

}  // namespace
