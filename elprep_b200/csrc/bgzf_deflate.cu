// bgzf_deflate.cu -- BGZF blocks written on the device (elp_fetch_bgzf, elp_debug_deflate; SURVEY.md §8f row 2, the writer of
// utils/bgzf/bgzf-files.go:324-431).
//
// The bytes of a call (prefix and formatted records in bam_raw, or the uploaded bytes of elp_debug_deflate) are cut into blocks of 0xff00
// bytes, the last one partial, as elp_bgzf_deflate cuts them.  The blocks go through in rounds of ROUND blocks, so the device memory a call
// adds does not grow with its bytes (DESIGN.md §3d):
//   bgzf_deflate   one CTA per block: the encoder of deflate.cuh into the block's slot (word-aligned), the BGZF size of every block
//   bgzf_deflate_crc  one warp per block: per-lane CRC-32 of a 1/32 slice of the input, folded with the x^(2^k) shift table (as bgzf_inflate's)
//   scan           exclusive_scan_u32_to_u64 of the BGZF sizes: every block's offset in the round's output, and the round's bytes
//   bgzf_compact   one CTA per block: the 18-byte header (BSIZE at byte 16), the DEFLATE bytes of the slot, CRC-32 and ISIZE, contiguous
// and the compacted round goes to the host in one copy, on a second stream while the next round computes.  The EOF marker follows on request.
#include <algorithm>
#include <cstring>
#include "ctx.h"
#include "deflate.cuh"
#include "../../include/elprep_b200.h"

namespace {

constexpr uint64_t BLK_IN = 0xff00;           // input bytes per BGZF block (elp_bgzf_deflate's)
constexpr int BGZF_HDR = 18, BGZF_TRL = 8;
constexpr unsigned DFL_THREADS = 256;         // the CTA team
constexpr uint64_t ROUND = 512;               // blocks per round
constexpr uint64_t SLOT = 65536;              // bytes per slot: >= dfl::stored_bytes(0xff00), a multiple of the word
constexpr uint64_t SCRATCH = 65536;           // per-position entries of a block's chain and match arrays
static_assert(dfl::stored_bytes((uint32_t)BLK_IN) <= SLOT, "a block's stream fits its slot");
const uint8_t EOF_MARKER[28] = {0x1f, 0x8b, 0x08, 0x04, 0, 0, 0, 0, 0x00, 0xff, 0x06, 0x00, 0x42, 0x43, 0x02, 0x00, 0x1b, 0x00, 0x03, 0x00, 0, 0, 0, 0, 0, 0, 0, 0};
__constant__ uint8_t BGZF_HEADER[16] = {0x1f, 0x8b, 0x08, 0x04, 0, 0, 0, 0, 0x00, 0xff, 0x06, 0x00, 0x42, 0x43, 0x02, 0x00};   // bgzf-files.go:336-340, BSIZE follows

// the chain team: one warp, lanes grouped by hash with __match_any_sync
struct ChainWarp {
    static constexpr unsigned size = 32;
    unsigned lane;
    __device__ void sync() const { __syncwarp(); }
    __device__ uint32_t same(uint32_t h) const { return __match_any_sync(FULL_MASK, h); }
    __device__ uint32_t lt() const { return lanemask_lt(); }
};
// the encoder's team: one CTA; its first warp builds the hash chain
struct CtaTeam {
    static constexpr unsigned size = DFL_THREADS;
    unsigned lane;
    __device__ void sync() const { __syncthreads(); }
    __device__ bool any(bool b) const { return __syncthreads_or(b) != 0; }
    __device__ void or32(uint32_t* p, uint32_t v) const { if (v) atomicOr(p, v); }
    __device__ void add32(uint32_t* p, uint32_t v) const { atomicAdd(p, v); }
    __device__ bool chain_lane() const { return lane < 32; }
    __device__ ChainWarp chain() const { return ChainWarp{lane & 31}; }
};

__device__ __forceinline__ uint32_t block_len(uint64_t n, uint64_t b) { return (uint32_t)min(BLK_IN, n - b * BLK_IN); }

__global__ void __launch_bounds__(DFL_THREADS) bgzf_deflate_kernel(const uint8_t* __restrict__ in, uint64_t n, uint64_t b0, uint8_t* __restrict__ slots,
                                                                   uint32_t* __restrict__ bsize, uint16_t* __restrict__ prev, uint32_t* __restrict__ match) {
    extern __shared__ __align__(16) uint8_t smem[];
    dfl::EncShared& S = *reinterpret_cast<dfl::EncShared*>(smem);
    const uint64_t i = blockIdx.x;
    const uint32_t len = block_len(n, b0 + i);
    const uint32_t c = dfl::deflate_block(CtaTeam{threadIdx.x}, S, dfl::EncScratch{prev + i * SCRATCH, match + i * SCRATCH}, in + (b0 + i) * BLK_IN, len,
                                          reinterpret_cast<uint32_t*>(slots + i * SLOT));
    if (threadIdx.x == 0) bsize[i] = (uint32_t)BGZF_HDR + c + (uint32_t)BGZF_TRL;
}

struct X2n { uint32_t v[32]; };
__global__ void __launch_bounds__(256) bgzf_deflate_crc_kernel(const uint8_t* __restrict__ in, uint64_t n, uint64_t b0, uint64_t nb, uint32_t* __restrict__ crc, X2n x2n) {
    __shared__ uint32_t ctab[256];
    ctab[threadIdx.x] = dfl::crc_table_entry(threadIdx.x);
    __syncthreads();
    const uint64_t i = (uint64_t)blockIdx.x * 8 + (threadIdx.x >> 5);
    if (i >= nb) return;
    const uint32_t v = dfl::warp_crc(ctab, x2n.v, in + (b0 + i) * BLK_IN, block_len(n, b0 + i), threadIdx.x & 31);
    if ((threadIdx.x & 31) == 0) crc[i] = v;
}

__global__ void __launch_bounds__(256) bgzf_compact_kernel(const uint8_t* __restrict__ slots, const uint32_t* __restrict__ bsize, const uint64_t* __restrict__ off,
                                                           const uint32_t* __restrict__ crc, uint64_t n, uint64_t b0, uint8_t* __restrict__ out) {
    const uint64_t i = blockIdx.x;
    const uint32_t bs = bsize[i], clen = bs - BGZF_HDR - BGZF_TRL, isize = block_len(n, b0 + i), cr = crc[i];
    const uint8_t* s = slots + i * SLOT;
    uint8_t* o = out + off[i];
    for (uint32_t t = threadIdx.x; t < bs; t += blockDim.x) {
        uint8_t v;
        if (t < BGZF_HDR) v = t == 16 ? (uint8_t)(bs - 1) : t == 17 ? (uint8_t)((bs - 1) >> 8) : BGZF_HEADER[t & 15];
        else if (t < BGZF_HDR + clen) v = s[t - BGZF_HDR];
        else { const uint32_t k = t - BGZF_HDR - clen; v = (uint8_t)((k < 4 ? cr : isize) >> (8 * (k & 3))); }
        o[t] = v;
    }
}

}  // namespace

// device scratch of the writer: bounded by ROUND, whatever the bytes of a call (DESIGN.md §3d)
struct DeflateState {
    DBuf<uint8_t> in, slots, rout[2];          // elp_debug_deflate's upload; block slots; compacted rounds (two: one computes, one downloads)
    DBuf<uint16_t> prev;
    DBuf<uint32_t> match, bsize[2], crc[2];
    DBuf<uint64_t> off[2];
    HBuf<uint64_t> h_total;                    // the bytes of the last two rounds
    cudaStream_t down = nullptr;
    cudaEvent_t done[2] = {nullptr, nullptr};
    X2n x2n;
    ~DeflateState() {
        for (int k = 0; k < 2; k++) if (done[k]) cudaEventDestroy(done[k]);
        if (down) cudaStreamDestroy(down);
    }
};

void free_state(DeflateState* D) { delete D; }

static int deflate_state(elp_ctx* c) {
    if (c->bgzf_out) return E_OK;
    c->bgzf_out.reset(new DeflateState());
    DeflateState& D = *c->bgzf_out;
    dfl::x2n_table(D.x2n.v);
    CUDA_TRY(c, D.h_total.fit(2));
    CUDA_TRY(c, cudaStreamCreateWithFlags(&D.down, cudaStreamNonBlocking));
    for (int k = 0; k < 2; k++) CUDA_TRY(c, cudaEventCreateWithFlags(&D.done[k], cudaEventDisableTiming));
    CUDA_TRY(c, cudaFuncSetAttribute(bgzf_deflate_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(dfl::EncShared)));
    return E_OK;
}

// in[0, n) on the device -> BGZF blocks (and the EOF marker when write_eof) at out; the caller checked capacity against elp_bgzf_deflate_bound(n)
int bgzf_deflate_run(elp_ctx* c, const uint8_t* in, uint64_t n, int write_eof, uint8_t* out, uint64_t* out_n) {
    TRY(deflate_state(c));
    DeflateState& D = *c->bgzf_out;
    cudaStream_t s = c->stream;
    const uint64_t nb = (n + BLK_IN - 1) / BLK_IN, r = std::min(nb, ROUND);
    if (nb) {
        TRY(grow(c, D.slots, r * SLOT)); TRY(grow(c, D.prev, r * SCRATCH)); TRY(grow(c, D.match, r * SCRATCH));
        for (int k = 0; k < 2; k++) {
            TRY(grow(c, D.rout[k], r * SLOT)); TRY(grow(c, D.bsize[k], r + 8)); TRY(grow(c, D.crc[k], r + 8)); TRY(grow(c, D.off[k], r + 2));
        }
    }
    uint64_t w = 0;
    int pend = -1;                                       // the round whose output is still on the device
    size_t pend_ev[2] = {0, 0};                          // (its bgzf_deflate and bgzf_compact entries among the pending timing events)
    auto download = [&](int k) -> int {                  // wait for round k, copy its bytes out
        CUDA_TRY(c, cudaEventSynchronize(D.done[k]));
        const uint64_t bytes = D.h_total.p[k];
        if (c->profile) { c->pending[pend_ev[0]].alg_bytes += (double)bytes; c->pending[pend_ev[1]].alg_bytes += 2.0 * (double)bytes; }
        CUDA_TRY(c, cudaMemcpyAsync(out + w, D.rout[k].p, bytes, cudaMemcpyDeviceToHost, D.down));
        CUDA_TRY(c, cudaStreamSynchronize(D.down));
        w += bytes;
        return E_OK;
    };
    for (uint64_t b0 = 0, round = 0; b0 < nb; b0 += ROUND, round++) {
        const int k = (int)(round & 1);
        const uint64_t m = std::min(ROUND, nb - b0), in_bytes = std::min(n, (b0 + m) * BLK_IN) - b0 * BLK_IN;
        const size_t ev = c->pending.size();
        c->begin("bgzf_deflate", (double)in_bytes);              // (+ the output bytes, once known)
        bgzf_deflate_kernel<<<(unsigned)m, DFL_THREADS, sizeof(dfl::EncShared), s>>>(in, n, b0, D.slots.p, D.bsize[k].p, D.prev.p, D.match.p);
        c->end(); LAUNCH_CHECK(c);
        c->begin("bgzf_deflate_crc", (double)in_bytes);
        bgzf_deflate_crc_kernel<<<nblk(m, 8), 256, 0, s>>>(in, n, b0, m, D.crc[k].p, D.x2n);
        c->end(); LAUNCH_CHECK(c);
        TRY(exclusive_scan_u32_to_u64(c, D.bsize[k].p, D.off[k].p, m));
        const size_t ev_compact = c->pending.size();
        c->begin("bgzf_compact", 0);                             // (2 x the output bytes, once known)
        bgzf_compact_kernel<<<(unsigned)m, 256, 0, s>>>(D.slots.p, D.bsize[k].p, D.off[k].p, D.crc[k].p, n, b0, D.rout[k].p);
        c->end(); LAUNCH_CHECK(c);
        CUDA_TRY(c, cudaMemcpyAsync(&D.h_total.p[k], D.off[k].p + m, 8, cudaMemcpyDeviceToHost, s));
        CUDA_TRY(c, cudaEventRecord(D.done[k], s));
        if (pend >= 0) TRY(download(pend));              // (the previous round downloads while this one computes)
        pend = k; pend_ev[0] = ev; pend_ev[1] = ev_compact;
    }
    if (pend >= 0) TRY(download(pend));
    if (write_eof) { std::memcpy(out + w, EOF_MARKER, 28); w += 28; }
    *out_n = w;
    return E_OK;
}

extern "C" int elp_debug_deflate(elp_ctx* c, const uint8_t* data, uint64_t n, int write_eof, uint8_t* out, uint64_t capacity, uint64_t* out_n) {
    if (!c || (!data && n) || !out || !out_n) return ELP_EINVAL;
    cudaSetDevice(c->device);
    std::lock_guard<std::mutex> lk(c->append_mu);
    const uint64_t need = elp_bgzf_deflate_bound(n);
    if (capacity < need) return c->fail(E_INVAL, "elp_debug_deflate: output buffer too small (%llu < elp_bgzf_deflate_bound = %llu)", (unsigned long long)capacity, (unsigned long long)need);
    TRY(deflate_state(c));
    DeflateState& D = *c->bgzf_out;
    TRY(grow(c, D.in, n + 64));
    if (n) CUDA_TRY(c, cudaMemcpyAsync(D.in.p, data, n, cudaMemcpyHostToDevice, c->stream));
    return bgzf_deflate_run(c, D.in.p, n, write_eof, out, out_n);
}
