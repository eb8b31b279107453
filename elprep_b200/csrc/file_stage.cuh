// file_stage.cuh -- a file streamed to the device through two page-locked chunks, shared by the loaders of side inputs: .elsites files
// (known_sites.cu) and the reference (reference_load.cu).
//   h[b], d[b]   page-locked and device halves of chunk b; the host fills h[b] while the kernels of the other chunk run
//   copy         the upload stream: h[b] -> d[b] waits for `used[b]` (the kernels that read d[b] are done) and records `up[b]`
// stage_read_lines fills a chunk with whole lines: the partial line after the last '\n' is carried, on the host, into the next chunk.
#pragma once
#include <cerrno>
#include <cstdio>
#include <cstring>
#include <vector>
#include "ctx.h"
#include "text_parse.cuh"

struct FileStage {
    uint64_t chunk = 0, hcap = 0, dcap = 0;                      // file bytes per step; capacities of h[b] and d[b]
    HBuf<uint8_t> h[2];
    DBuf<uint8_t> d[2];
    cudaEvent_t up[2] = {nullptr, nullptr};                      // the upload out of h[b] has landed in d[b] (copy stream)
    cudaEvent_t used[2] = {nullptr, nullptr};                    // the kernels that read d[b] are done (compute stream)
    cudaStream_t copy = nullptr;
    FileStage() = default;
    FileStage(const FileStage&) = delete;
    ~FileStage() {   // the chunks are freed after the last upload out of them
        if (copy) cudaStreamSynchronize(copy);
        for (int b = 0; b < 2; b++) { if (up[b]) cudaEventDestroy(up[b]); if (used[b]) cudaEventDestroy(used[b]); }
        if (copy) cudaStreamDestroy(copy);
    }
};

// a chunk of whole lines at the front of h[b]: m bytes; last: the file ends with it; long_tail: the carried line is already too long
struct LineChunk { int b = 0; uint64_t m = 0; bool last = false, long_tail = false; };

namespace {

// the stream, the events, and both chunks of hcap host and dcap device bytes (kept when the sizes are unchanged)
inline int stage_init(elp_ctx* c, FileStage& S, uint64_t chunk, uint64_t hcap, uint64_t dcap, const char* who) {
    if (!S.copy) {
        CUDA_TRY(c, cudaStreamCreateWithFlags(&S.copy, cudaStreamNonBlocking));
        for (int b = 0; b < 2; b++) { CUDA_TRY(c, cudaEventCreateWithFlags(&S.up[b], cudaEventDisableTiming)); CUDA_TRY(c, cudaEventCreateWithFlags(&S.used[b], cudaEventDisableTiming)); }
    }
    if (S.chunk == chunk && S.hcap == hcap && S.dcap == dcap) return E_OK;
    CUDA_TRY(c, cudaStreamSynchronize(S.copy));
    for (int b = 0; b < 2; b++) { S.h[b].release(); S.d[b].release(); }
    S.chunk = S.hcap = S.dcap = 0;
    for (int b = 0; b < 2; b++) {
        if (S.h[b].fit(hcap) != cudaSuccess || S.d[b].fit(dcap) != cudaSuccess) {
            cudaGetLastError();
            return c->fail(E_NOMEM, "%s: staging allocation of 2 x %llu bytes failed", who, (unsigned long long)hcap);
        }
    }
    S.chunk = chunk; S.hcap = hcap; S.dcap = dcap;
    return E_OK;
}

// device bytes for n text bytes at the line finder's granularity, with the 64 zero bytes behind
inline uint64_t stage_padded(uint64_t n) { return (n + SAM_CHUNK - 1) / SAM_CHUNK * SAM_CHUNK + SAM_CHUNK; }

// h[b] may be refilled: the last upload out of it has read it
inline int stage_wait_host(elp_ctx* c, FileStage& S, int b) {
    CUDA_TRY(c, cudaEventSynchronize(S.up[b]));
    return E_OK;
}

// h[b][0, n) -> d[b][at, at + n) on the copy stream, zeros behind up to stage_padded(at + n)
inline int stage_upload(elp_ctx* c, FileStage& S, int b, uint64_t n, uint64_t at) {
    if (!n) return E_OK;
    const uint64_t padded = stage_padded(at + n);
    CUDA_TRY(c, cudaStreamWaitEvent(S.copy, S.used[b], 0));
    CUDA_TRY(c, cudaMemcpyAsync(S.d[b].p + at, S.h[b].p, n, cudaMemcpyHostToDevice, S.copy));
    CUDA_TRY(c, cudaMemsetAsync(S.d[b].p + at + n, 0, padded - at - n, S.copy));
    CUDA_TRY(c, cudaEventRecord(S.up[b], S.copy));
    return E_OK;
}

// the carried bytes and the next chunk of the file into h[b]; lines of max_line bytes or more cannot be carried
inline int stage_read_lines(elp_ctx* c, FileStage& S, FILE* f, const char* path, const char* who, uint64_t max_line, std::vector<uint8_t>& carry, int b, LineChunk* ch) {
    if (const int rc = stage_wait_host(c, S, b)) return rc;
    uint8_t* h = S.h[b].p;
    const uint64_t nc = carry.size();
    if (nc) memcpy(h, carry.data(), nc);
    const size_t got = fread(h + nc, 1, S.chunk, f);
    if (got < S.chunk && ferror(f)) return c->fail(E_INVAL, "%s: cannot read %s: %s", who, path, strerror(errno));
    const uint64_t n = nc + got;
    ch->b = b; ch->last = got < S.chunk;
    if (ch->last) ch->m = n;   // the last line may lack its '\n'
    else {
        const void* q = got ? memrchr(h + nc, '\n', got) : nullptr;
        ch->m = q ? (uint64_t)(static_cast<const uint8_t*>(q) - h) + 1 : 0;
    }
    carry.assign(h + ch->m, h + n);
    ch->long_tail = !ch->last && carry.size() >= max_line;
    return E_OK;
}

}  // namespace
