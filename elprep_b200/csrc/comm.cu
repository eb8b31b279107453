// comm.cu -- several GPUs of one box behind the C ABI (SURVEY.md 8e; the reference's model is `elprep sfm`: cmd/sfm.go:605-805,
// sam/split-merge.go:178-311).  One context per GPU, reads partitioned by contig group; what crosses GPUs:
//   * BQSR: ONE ncclAllReduce(sum, int64) of the dense covariate tables (LoadAndCombineBQSRTables, filters/print-bqsr.go:310-329);
//   * duplicate marking: pairs whose mates lie in different groups -- the reference's *spread* reads (split-merge.go:286-293).  The mate
//     that does not live on the pair's owner (the rank owning the smaller REFID: every candidate of a duplicate signature has the same
//     (refid1, refid2), so they all meet there) travels as a 128-byte record (hash, refid, unclipped position, score, FLAG, read group,
//     QNAME) through grouped ncclSend / ncclRecv and is appended to the owner's columns as a GHOST read: it takes part in the mate join and
//     the pair signature sort like any local read, never in fragment marking, the coordinate sort or the output.  After pair marking the
//     0x400 bits of the ghosts go back the same way and are ORed into the FLAG of the real reads;
//   * duplication metrics: allreduce of the counters and histograms (mergeDuplicatesCtrMaps, mark-optical-duplicates.go:451-466).
// NCCL is resolved at run time (dlopen of libnccl.so.2 -- the copy the process already has, e.g. torch's, or the system's), so the library
// itself has no link-time dependency on it and single-GPU users never load it.
#include <dlfcn.h>
#include <nccl.h>
#include <algorithm>
#include <climits>
#include "../../include/elprep_b200.h"
#include "ctx.h"

namespace {

struct NcclApi {
    ncclResult_t (*GetUniqueId)(ncclUniqueId*);
    ncclResult_t (*CommInitRank)(ncclComm_t*, int, ncclUniqueId, int);
    ncclResult_t (*CommDestroy)(ncclComm_t);
    ncclResult_t (*AllReduce)(const void*, void*, size_t, ncclDataType_t, ncclRedOp_t, ncclComm_t, cudaStream_t);
    ncclResult_t (*AllGather)(const void*, void*, size_t, ncclDataType_t, ncclComm_t, cudaStream_t);
    ncclResult_t (*Send)(const void*, size_t, ncclDataType_t, int, ncclComm_t, cudaStream_t);
    ncclResult_t (*Recv)(void*, size_t, ncclDataType_t, int, ncclComm_t, cudaStream_t);
    ncclResult_t (*GroupStart)();
    ncclResult_t (*GroupEnd)();
    const char* (*GetErrorString)(ncclResult_t);
};
NcclApi* nccl_api(std::string* err) {
    static NcclApi api; static int state = 0; static std::string why; static std::mutex mu;
    std::lock_guard<std::mutex> lk(mu);
    if (state == 0) {
        void* h = dlopen("libnccl.so.2", RTLD_NOW | RTLD_GLOBAL);
        if (!h) h = dlopen("libnccl.so", RTLD_NOW | RTLD_GLOBAL);
        if (!h) { why = std::string("cannot load libnccl.so.2: ") + dlerror(); state = -1; }
        else {
            bool ok = true;
            auto sym = [&](const char* n) { void* p = dlsym(h, n); if (!p) { ok = false; why = std::string("libnccl lacks ") + n; } return p; };
            api.GetUniqueId = (decltype(api.GetUniqueId))sym("ncclGetUniqueId"); api.CommInitRank = (decltype(api.CommInitRank))sym("ncclCommInitRank");
            api.CommDestroy = (decltype(api.CommDestroy))sym("ncclCommDestroy"); api.AllReduce = (decltype(api.AllReduce))sym("ncclAllReduce");
            api.AllGather = (decltype(api.AllGather))sym("ncclAllGather"); api.Send = (decltype(api.Send))sym("ncclSend"); api.Recv = (decltype(api.Recv))sym("ncclRecv");
            api.GroupStart = (decltype(api.GroupStart))sym("ncclGroupStart"); api.GroupEnd = (decltype(api.GroupEnd))sym("ncclGroupEnd");
            api.GetErrorString = (decltype(api.GetErrorString))sym("ncclGetErrorString");
            state = ok ? 1 : -1;
        }
    }
    if (state < 0) { if (err) *err = why; return nullptr; }
    return &api;
}
#define NCCL_TRY(c, api, call) do { ncclResult_t r__ = (call); if (r__ != ncclSuccess) return (c)->fail(E_CUDA, "NCCL error at %s:%d: %s", __FILE__, __LINE__, (api)->GetErrorString(r__)); } while (0)

constexpr int SP_REC = 128, SP_NAME = 92;   // bytes per spread record / of its QNAME

// destination rank of a read's spread record, or -1: true pair entering duplicate marking (mark-duplicates.go:182-184, 436) whose mate maps to a
// contig of another rank; the pair is classified by the owner of the smaller REFID
__device__ __forceinline__ int spread_dest(uint16_t f, int32_t refid, int32_t nref, const int32_t* __restrict__ owner, int n_contigs, int me) {
    if ((f & (F_UNMAPPED | F_SECONDARY | F_SUPPLEMENTARY)) != 0 || (f & (F_MULTIPLE | F_NEXTUNMAPPED)) != F_MULTIPLE) return -1;
    if (refid < 0 || nref < 0 || refid >= n_contigs || nref >= n_contigs) return -1;
    const int o1 = owner[refid], o2 = owner[nref];
    if (o1 == o2) return -1;
    const int dst = owner[min(refid, nref)];
    return dst == me ? -1 : dst;
}
// cnt[0, world): records to every rank; cnt[world]: the reads among them whose QNAME a record cannot hold; cnt[world + 1]: n (at most
// 2^32 - 1).  The count exchange gathers all of it, so every rank learns of a refusal before anything is shipped.
__global__ void __launch_bounds__(256) spread_count_kernel(uint64_t n, const uint16_t* __restrict__ flag, const int32_t* __restrict__ refid, const int32_t* __restrict__ nref,
                                                            const uint64_t* __restrict__ qname_off, const int32_t* __restrict__ owner, int n_contigs, int me, int world,
                                                            uint32_t* __restrict__ cnt) {
    extern __shared__ uint32_t sh[];
    for (int i = threadIdx.x; i < world; i += blockDim.x) sh[i] = 0;
    __syncthreads();
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i == 0) cnt[world + 1] = (uint32_t)min(n, (uint64_t)UINT32_MAX);
    if (i < n) {
        const int d = spread_dest(flag[i], refid[i], nref[i], owner, n_contigs, me);
        if (d >= 0) { atomicAdd(&sh[d], 1u); if (qname_off[i + 1] - qname_off[i] > SP_NAME) atomicAdd(&cnt[world], 1u); }
    }
    __syncthreads();
    for (int k = threadIdx.x; k < world; k += blockDim.x) if (sh[k]) atomicAdd(&cnt[k], sh[k]);
}
struct FillArgs {
    uint64_t n; const uint16_t* flag; const int32_t *refid, *nref, *rg, *upos, *score; const uint64_t* qhash; const uint64_t* qname_off; const uint8_t* qname;
    const int32_t* owner; int n_contigs, me;
    const uint32_t* base;     // [world] first record of each destination
    uint32_t* cursor;         // [world]
    uint4* recs; uint32_t* sent_idx; uint32_t* err;
};
__global__ void __launch_bounds__(256) spread_fill_kernel(FillArgs A) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= A.n) return;
    const uint16_t f = A.flag[i];
    const int d = spread_dest(f, A.refid[i], A.nref[i], A.owner, A.n_contigs, A.me);
    if (d < 0) return;
    const uint32_t at = A.base[d] + atomicAdd(&A.cursor[d], 1u);
    const uint64_t n0 = A.qname_off[i], n1 = A.qname_off[i + 1];
    if (n1 - n0 > SP_NAME) { atomicOr(A.err, DERR_SPREAD_NAME); return; }
    A.sent_idx[at] = (uint32_t)i;
    const uint64_t h = A.qhash[i];
    uint32_t w[32];
    w[0] = (uint32_t)h; w[1] = (uint32_t)(h >> 32); w[2] = (uint32_t)A.refid[i]; w[3] = (uint32_t)A.upos[i];
    w[4] = (uint32_t)A.score[i]; w[5] = f; w[6] = (uint32_t)A.rg[i]; w[7] = (uint32_t)i;
    w[8] = (uint32_t)(n1 - n0);
    for (int k = 9; k < 32; k++) w[k] = 0;
    for (uint64_t b = 0; b < n1 - n0; b++) w[9 + (b >> 2)] |= (uint32_t)A.qname[n0 + b] << (8 * (b & 3));
    uint4* out = A.recs + 8 * (uint64_t)at;
    for (int k = 0; k < 8; k++) out[k] = make_uint4(w[4 * k], w[4 * k + 1], w[4 * k + 2], w[4 * k + 3]);
}
__global__ void __launch_bounds__(256) ghost_lens_kernel(uint64_t g, const uint4* __restrict__ recs, uint32_t* __restrict__ lens) {
    const uint64_t k = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (k < g) lens[k] = min(recs[8 * k + 2].x, (uint32_t)SP_NAME);   // the arena holds SP_NAME bytes per ghost, whatever a record says
}
struct GhostArgs {
    uint64_t n, g; const uint4* recs;
    uint16_t* flag; int32_t *refid, *rg, *upos, *score; uint64_t* qhash; const uint64_t* qname_off; uint8_t* qname;
};
// ghost k becomes read n + k of the columns duplicate marking looks at (qname_off[n .. n+g] was written by the scan of the name lengths)
__global__ void __launch_bounds__(256) ghost_append_kernel(GhostArgs A) {
    const uint64_t k = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= A.g) return;
    const uint4* r = A.recs + 8 * k;
    const uint4 a = r[0], b = r[1];
    const uint64_t i = A.n + k;
    A.qhash[i] = ((uint64_t)a.y << 32) | a.x; A.refid[i] = (int32_t)a.z; A.upos[i] = (int32_t)a.w;
    A.score[i] = (int32_t)b.x; A.flag[i] = (uint16_t)(b.y & ~(uint32_t)F_DUPLICATE); A.rg[i] = (int32_t)b.z;
    const uint32_t* w = reinterpret_cast<const uint32_t*>(r + 2);
    const uint32_t len = min(w[0], (uint32_t)SP_NAME);
    const uint64_t o = A.qname_off[i];
    for (uint32_t t = 0; t < len; t++) A.qname[o + t] = (uint8_t)(w[1 + (t >> 2)] >> (8 * (t & 3)));
}
__global__ void __launch_bounds__(256) ghost_reply_kernel(uint64_t n, uint64_t g, const uint16_t* __restrict__ flag, uint8_t* __restrict__ reply) {
    const uint64_t k = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (k < g) reply[k] = (flag[n + k] & F_DUPLICATE) ? 1 : 0;
}
__global__ void __launch_bounds__(256) spread_apply_kernel(uint64_t m, const uint32_t* __restrict__ sent_idx, const uint8_t* __restrict__ reply, uint16_t* __restrict__ flag) {
    const uint64_t k = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (k < m && reply[k]) atomic_or_u16(flag, sent_idx[k], F_DUPLICATE);
}

// the word a rank contributes to a max-allreduce of error states: -code << 16 | rank of a failed rank (the max picks one failure when several
// ranks fail), INT_MIN when the rank is fine
int32_t status_word(const elp_ctx* c, int rc) { return rc ? (int32_t)(((uint32_t)-rc << 16) | (uint32_t)c->rank) : INT_MIN; }
int peer_failure(elp_ctx* c, int32_t w) {
    const int code = -(w >> 16), r = w & 0xffff;
    return c->fail(code, "duplicate marking failed with code %d on rank %d", code, r);
}
// every rank returns together: local_rc (with its own text) on the failing rank, the code of a failed peer on the others, else E_OK
int comm_agree(elp_ctx* c, NcclApi* N, int local_rc) {
    int32_t w = status_word(c, local_rc);
    CUDA_TRY(c, c->scan_tmp.reserve(16, c->stream));
    CUDA_TRY(c, cudaMemcpyAsync(c->scan_tmp.p, &w, 4, cudaMemcpyHostToDevice, c->stream));
    NCCL_TRY(c, N, N->AllReduce(c->scan_tmp.p, c->scan_tmp.p, 1, ncclInt32, ncclMax, (ncclComm_t)c->comm, c->stream));
    CUDA_TRY(c, cudaMemcpyAsync(&w, c->scan_tmp.p, 4, cudaMemcpyDeviceToHost, c->stream));
    CUDA_TRY(c, cudaStreamSynchronize(c->stream));
    if (local_rc) return local_rc;
    return w != INT_MIN ? peer_failure(c, w) : E_OK;
}

}  // namespace

// ---- called by phase_markdup (markdup.cu) ----
// Errors are agreed at three points, each in a collective every rank makes: the range allreduce (errors of adapt), the count all-gather
// (the limits of the exchange) and one status allreduce on each side of the record exchange (allocations, the ghost append).  So a rank
// that fails makes every rank return before the next collective, and before any FLAG changes.  Not agreed: a sticky CUDA error (a device
// fault), after which the rank cannot make the collective at all.
// value ranges that size the sort keys must agree on every rank (a ghost's unclipped position or score may lie outside the local range).
// local_rc is this rank's error so far (adapt, invalid QUAL, negative POS); it rides along in the same allreduce, so that all ranks return an error
// together, before any record is exchanged, instead of leaving the others waiting in a collective the failing rank never reaches.
int comm_allreduce_ranges(elp_ctx* c, int local_rc) {
    if (!c->comm) return local_rc;
    NcclApi* N = nccl_api(&c->err); if (!N) return E_CUDA;
    int32_t h[5] = {c->h_ranges.n_entering ? -c->h_ranges.upos_min : INT_MIN, c->h_ranges.n_entering ? c->h_ranges.upos_max : INT_MIN, c->h_ranges.score_max, (int32_t)std::min<uint32_t>(c->h_ranges.n_entering, 1u),
                    status_word(c, local_rc)};
    CUDA_TRY(c, c->scan_tmp.reserve(16, c->stream));
    { int rcu = upload_small(c, c->scan_tmp.p, h, 20); if (rcu) return rcu; }
    NCCL_TRY(c, N, N->AllReduce(c->scan_tmp.p, c->scan_tmp.p, 5, ncclInt32, ncclMax, (ncclComm_t)c->comm, c->stream));
    CUDA_TRY(c, cudaMemcpyAsync(h, c->scan_tmp.p, 20, cudaMemcpyDeviceToHost, c->stream));
    CUDA_TRY(c, cudaStreamSynchronize(c->stream));
    if (local_rc) return local_rc;   // (keeps its own text)
    if (h[4] != INT_MIN) return peer_failure(c, h[4]);
    if (h[3]) { c->h_ranges.upos_min = -h[0]; c->h_ranges.upos_max = h[1]; c->h_ranges.score_max = h[2]; c->any_rank_entering = true; } else c->any_rank_entering = false;
    return E_OK;
}

// ships the visiting mates to the owners of their pairs and appends what arrives as ghost reads n .. n + n_ghost - 1
int spread_exchange_begin(elp_ctx* c) {
    c->n_ghost = 0; c->sp_sent_total = 0;
    if (!c->comm || c->world < 2 || !c->d_owner.p) return E_OK;
    NcclApi* N = nccl_api(&c->err); if (!N) return E_CUDA;
    const uint64_t n = c->n; const int W = c->world; cudaStream_t s = c->stream;
    // per rank, W + 2 words are gathered: the records to every rank, the reads among them with a QNAME too long for a record, and the
    // number of reads.  Every rank checks the limits of every rank on the same numbers, so all refuse together, before anything is shipped.
    const size_t P = (size_t)W + 2;
    CUDA_TRY(c, c->scan_tmp.reserve(P * (W + 1) + 2 * W + 16, s));
    uint32_t* d_cnt = c->scan_tmp.p; uint32_t* d_all = d_cnt + P; uint32_t* d_base = d_all + P * W; uint32_t* d_cur = d_base + W;
    CUDA_TRY(c, cudaMemsetAsync(d_cnt, 0, (P * (W + 1) + 2 * W) * 4, s));
    if (n) { c->begin("spread_count", (double)n * 10); spread_count_kernel<<<nblk(n, 256), 256, W * 4, s>>>(n, c->flag.p, c->refid.p, c->nref.p, c->qname_off.p, c->d_owner.p, c->n_contigs, c->rank, W, d_cnt); c->end(); LAUNCH_CHECK(c); }
    NCCL_TRY(c, N, N->AllGather(d_cnt, d_all, P, ncclUint32, (ncclComm_t)c->comm, s));
    std::vector<uint32_t> all(P * W);
    CUDA_TRY(c, cudaMemcpyAsync(all.data(), d_all, all.size() * 4, cudaMemcpyDeviceToHost, s));
    CUDA_TRY(c, cudaStreamSynchronize(s));
    for (int r = 0; r < W; r++) {
        const std::string on = r == c->rank ? "" : " on rank " + std::to_string(r);
        if (all[r * P + W]) return c->fail(E_LIMIT, "cross-group pair exchange: QNAME longer than %d bytes%s", SP_NAME, on.c_str());
        uint64_t recv = 0;
        for (int q = 0; q < W; q++) recv += all[q * P + r];
        if (all[r * P + W + 1] + recv >= (1ull << 32)) return c->fail(E_LIMIT, "more than 2^32-1 reads + visiting mates in one context%s", on.c_str());
    }
    c->sp_send.assign(W, 0); c->sp_recv.assign(W, 0);
    std::vector<uint32_t> base(W, 0);
    uint64_t tot_send = 0, tot_recv = 0;
    for (int r = 0; r < W; r++) { c->sp_send[r] = all[(size_t)c->rank * P + r]; c->sp_recv[r] = all[(size_t)r * P + c->rank]; base[r] = (uint32_t)tot_send; tot_send += c->sp_send[r]; tot_recv += c->sp_recv[r]; }
    c->sp_sent_total = tot_send; c->n_ghost = tot_recv;
    const uint64_t g = tot_recv;
    // everything the record exchange, the ghost columns and the reply exchange need is allocated, and the records filled, before the
    // outcome is agreed: an allocation that fails on one rank makes every rank return before the record exchange
    int rc = [&]() -> int {
        CUDA_TRY(c, c->sp_sendbuf.reserve(8 * tot_send + 8, s)); CUDA_TRY(c, c->sp_recvbuf.reserve(8 * tot_recv + 8, s)); CUDA_TRY(c, c->sp_sent_idx.reserve(tot_send + 4, s));
        if (g) {   // the columns duplicate marking reads get g more entries
            const uint64_t nt = n + g;
            CUDA_TRY(c, c->flag.reserve(nt + 2, s, n)); CUDA_TRY(c, c->refid.reserve(nt + 1, s, n)); CUDA_TRY(c, c->rg.reserve(nt + 1, s, n)); CUDA_TRY(c, c->upos.reserve(nt + 1, s, n));
            CUDA_TRY(c, c->score.reserve(nt + 1, s, n)); CUDA_TRY(c, c->qhash.reserve(nt + 1, s, n)); CUDA_TRY(c, c->qname_off.reserve(nt + 2, s, n + 1));
            CUDA_TRY(c, c->qname.reserve(c->n_qname + g * SP_NAME + 64, s, c->n_qname));
            CUDA_TRY(c, c->vals_a.reserve(g + 8, s));
        }
        CUDA_TRY(c, c->bytes_tmp.reserve(((g + 15) & ~(uint64_t)15) + tot_send + 64, s));   // the replies of spread_exchange_end
        if (tot_send) {
            { int rcu = upload_small(c, d_base, base.data(), (size_t)W * 4); if (rcu) return rcu; }
            FillArgs A{};
            A.n = n; A.flag = c->flag.p; A.refid = c->refid.p; A.nref = c->nref.p; A.rg = c->rg.p; A.upos = c->upos.p; A.score = c->score.p; A.qhash = c->qhash.p; A.qname_off = c->qname_off.p; A.qname = c->qname.p;
            A.owner = c->d_owner.p; A.n_contigs = c->n_contigs; A.me = c->rank; A.base = d_base; A.cursor = d_cur; A.recs = c->sp_sendbuf.p; A.sent_idx = c->sp_sent_idx.p; A.err = c->d_err.p;
            c->begin("spread_fill", (double)n * 10 + (double)tot_send * 200); spread_fill_kernel<<<nblk(n, 256), 256, 0, s>>>(A); c->end(); LAUNCH_CHECK(c);
        }
        return E_OK;
    }();
    rc = comm_agree(c, N, rc);
    if (rc) { c->n_ghost = 0; c->sp_sent_total = 0; return rc; }
    // one grouped exchange: NVLink / NVSwitch peer traffic, ~1 % of the reads x 128 B
    NCCL_TRY(c, N, N->GroupStart());
    { uint64_t so = 0, ro = 0;
      for (int r = 0; r < W; r++) {
          if (c->sp_send[r]) NCCL_TRY(c, N, N->Send(c->sp_sendbuf.p + 8 * so, (size_t)c->sp_send[r] * SP_REC, ncclChar, r, (ncclComm_t)c->comm, s));
          if (c->sp_recv[r]) NCCL_TRY(c, N, N->Recv(c->sp_recvbuf.p + 8 * ro, (size_t)c->sp_recv[r] * SP_REC, ncclChar, r, (ncclComm_t)c->comm, s));
          so += c->sp_send[r]; ro += c->sp_recv[r];
      } }
    NCCL_TRY(c, N, N->GroupEnd());
    // the ghost append is agreed too, so that no rank starts marking (or waits in the reply exchange) when another cannot
    rc = [&]() -> int {
        if (g) {
            c->begin("ghost_append", (double)g * 300);
            ghost_lens_kernel<<<nblk(g, 256), 256, 0, s>>>(g, c->sp_recvbuf.p, c->vals_a.p);
            c->end(); LAUNCH_CHECK(c);
            int r2 = exclusive_scan_u64_from_u32(c, c->vals_a.p, c->qname_off.p + n, g, c->n_qname);
            if (r2) return r2;
            GhostArgs G{};
            G.n = n; G.g = g; G.recs = c->sp_recvbuf.p; G.flag = c->flag.p; G.refid = c->refid.p; G.rg = c->rg.p; G.upos = c->upos.p; G.score = c->score.p; G.qhash = c->qhash.p;
            G.qname_off = c->qname_off.p; G.qname = c->qname.p;
            c->launches++; ghost_append_kernel<<<nblk(g, 256), 256, 0, s>>>(G); LAUNCH_CHECK(c);
        }
        return check_device_errors(c);
    }();
    rc = comm_agree(c, N, rc);
    if (rc) { c->n_ghost = 0; c->sp_sent_total = 0; }
    return rc;
}

// returns the 0x400 bits of the ghosts to the ranks the reads live on
int spread_exchange_end(elp_ctx* c) {
    if (!c->comm || c->world < 2 || !c->d_owner.p) return E_OK;
    NcclApi* N = nccl_api(&c->err); if (!N) return E_CUDA;
    const int W = c->world; cudaStream_t s = c->stream;
    const uint64_t g = c->n_ghost, m = c->sp_sent_total;
    CUDA_TRY(c, c->bytes_tmp.reserve(g + m + 64, s));
    uint8_t* reply_out = c->bytes_tmp.p; uint8_t* reply_in = c->bytes_tmp.p + ((g + 15) & ~(uint64_t)15);
    CUDA_TRY(c, c->bytes_tmp.reserve(((g + 15) & ~(uint64_t)15) + m + 64, s));
    reply_out = c->bytes_tmp.p; reply_in = c->bytes_tmp.p + ((g + 15) & ~(uint64_t)15);
    if (g) { c->launches++; ghost_reply_kernel<<<nblk(g, 256), 256, 0, s>>>(c->n, g, c->flag.p, reply_out); LAUNCH_CHECK(c); }
    NCCL_TRY(c, N, N->GroupStart());
    { uint64_t so = 0, ro = 0;
      for (int r = 0; r < W; r++) {   // the directions of spread_exchange_begin, reversed
          if (c->sp_recv[r]) NCCL_TRY(c, N, N->Send(reply_out + ro, c->sp_recv[r], ncclChar, r, (ncclComm_t)c->comm, s));
          if (c->sp_send[r]) NCCL_TRY(c, N, N->Recv(reply_in + so, c->sp_send[r], ncclChar, r, (ncclComm_t)c->comm, s));
          so += c->sp_send[r]; ro += c->sp_recv[r];
      } }
    NCCL_TRY(c, N, N->GroupEnd());
    if (m) { c->launches++; spread_apply_kernel<<<nblk(m, 256), 256, 0, s>>>(m, c->sp_sent_idx.p, reply_in, c->flag.p); LAUNCH_CHECK(c); }
    c->n_ghost = 0;
    return E_OK;
}

extern "C" {

int elp_comm_unique_id(uint8_t id[128]) {
    NcclApi* N = nccl_api(nullptr);
    if (!N || !id) return ELP_EINVAL;
    ncclUniqueId u;
    if (N->GetUniqueId(&u) != ncclSuccess) return ELP_ECUDA;
    memcpy(id, u.internal, 128);
    return ELP_OK;
}

int elp_comm_init(elp_ctx* c, const uint8_t id[128], int rank, int world) {
    if (!c || !id || world < 1 || rank < 0 || rank >= world) return ELP_EINVAL;
    cudaSetDevice(c->device);
    NcclApi* N = nccl_api(&c->err);
    if (!N) return ELP_ECUDA;
    if (c->comm) { N->CommDestroy((ncclComm_t)c->comm); c->comm = nullptr; }
    ncclUniqueId u; memcpy(u.internal, id, 128);
    ncclComm_t comm;
    NCCL_TRY(c, N, N->CommInitRank(&comm, world, u, rank));
    c->comm = comm; c->rank = rank; c->world = world;
    return ELP_OK;
}

int elp_comm_destroy(elp_ctx* c) {
    if (!c) return ELP_EINVAL;
    if (c->comm) { cudaSetDevice(c->device); cudaStreamSynchronize(c->stream); NcclApi* N = nccl_api(nullptr); if (N) N->CommDestroy((ncclComm_t)c->comm); c->comm = nullptr; }
    return ELP_OK;
}

int elp_comm_set_partition(elp_ctx* c, const int32_t* contig_owner) {
    if (!c || !contig_owner) return ELP_EINVAL;
    cudaSetDevice(c->device);
    for (int i = 0; i < c->n_contigs; i++) if (contig_owner[i] < 0 || contig_owner[i] >= std::max(1, c->world)) return c->fail(E_INVAL, "elp_comm_set_partition: owner %d of contig %d is not a rank", contig_owner[i], i);
    CUDA_TRY(c, c->d_owner.fit(std::max(1, c->n_contigs)));
    CUDA_TRY(c, cudaMemcpy(c->d_owner.p, contig_owner, (size_t)c->n_contigs * 4, cudaMemcpyHostToDevice));
    return ELP_OK;
}

int elp_bqsr_tables_allreduce(elp_ctx* c) {
    if (!c) return ELP_EINVAL;
    cudaSetDevice(c->device);
    if (!c->comm) return c->fail(E_STATE, "elp_bqsr_tables_allreduce without elp_comm_init");
    if (!c->gathered) return c->fail(E_STATE, "elp_bqsr_tables_allreduce before elp_bqsr_gather");
    NcclApi* N = nccl_api(&c->err); if (!N) return ELP_ECUDA;
    c->begin("nccl_allreduce_tables", (double)c->geom.cells() * 16);
    ncclResult_t r = N->AllReduce(c->d_tables.p, c->d_tables.p, c->geom.cells() * 2, ncclInt64, ncclSum, (ncclComm_t)c->comm, c->stream);
    c->end();
    if (r != ncclSuccess) return c->fail(E_CUDA, "ncclAllReduce: %s", N->GetErrorString(r));
    c->finalized = false;
    return ELP_OK;
}

int elp_optical_allreduce(elp_ctx* c) {
    if (!c) return ELP_EINVAL;
    cudaSetDevice(c->device);
    if (!c->comm) return c->fail(E_STATE, "elp_optical_allreduce without elp_comm_init");
    if (!c->opt_valid) return c->fail(E_STATE, "elp_optical_allreduce before elp_sort_markdup(.., ELP_MARKDUP_OPTICAL)");
    NcclApi* N = nccl_api(&c->err); if (!N) return ELP_ECUDA;
    const size_t slots = c->opt.size(), per = 7 + 3 * OPT_HBINS;
    // dense part: counters and histogram keys < OPT_HBINS summed; larger keys (duplicate sets of > 1023 reads) gathered as (slot*4+which, key, count)
    // triples, padded to the largest number of triples of any rank, which is gathered first
    std::vector<int64_t> h(slots * per, 0), ovf;
    for (size_t sl = 0; sl < slots; sl++) {
        for (int k = 0; k < 7; k++) h[sl * per + k] = c->opt[sl].ctr[k];
        for (int w = 0; w < 3; w++) for (auto& kv : c->opt[sl].hist[w]) {
            if (kv.first >= 0 && kv.first < OPT_HBINS) h[sl * per + 7 + w * OPT_HBINS + kv.first] = kv.second;
            else { ovf.push_back((int64_t)(sl * 4 + w)); ovf.push_back(kv.first); ovf.push_back(kv.second); }
        }
    }
    const size_t W = (size_t)c->world;
    CUDA_TRY(c, c->keys_a.reserve(h.size() + W + 8, c->stream));
    int64_t* d = reinterpret_cast<int64_t*>(c->keys_a.p); int64_t* d_no = d + h.size(); int64_t* d_nos = d_no + 1;
    const int64_t no = (int64_t)(ovf.size() / 3);
    CUDA_TRY(c, cudaMemcpyAsync(d, h.data(), h.size() * 8, cudaMemcpyHostToDevice, c->stream));
    CUDA_TRY(c, cudaMemcpyAsync(d_no, &no, 8, cudaMemcpyHostToDevice, c->stream));
    NCCL_TRY(c, N, N->AllReduce(d, d, h.size(), ncclInt64, ncclSum, (ncclComm_t)c->comm, c->stream));
    NCCL_TRY(c, N, N->AllGather(d_no, d_nos, 1, ncclInt64, (ncclComm_t)c->comm, c->stream));
    std::vector<int64_t> nos(W);
    CUDA_TRY(c, cudaMemcpyAsync(h.data(), d, h.size() * 8, cudaMemcpyDeviceToHost, c->stream));
    CUDA_TRY(c, cudaMemcpyAsync(nos.data(), d_nos, W * 8, cudaMemcpyDeviceToHost, c->stream));
    CUDA_TRY(c, cudaStreamSynchronize(c->stream));
    const size_t mx = (size_t)*std::max_element(nos.begin(), nos.end());
    std::vector<int64_t> all(3 * mx * W);
    if (mx) {
        ovf.resize(3 * mx, -1);
        CUDA_TRY(c, c->keys_a.reserve(3 * mx * (W + 1) + 8, c->stream));
        int64_t* d_ovf = reinterpret_cast<int64_t*>(c->keys_a.p); int64_t* d_all = d_ovf + 3 * mx;
        CUDA_TRY(c, cudaMemcpyAsync(d_ovf, ovf.data(), ovf.size() * 8, cudaMemcpyHostToDevice, c->stream));
        NCCL_TRY(c, N, N->AllGather(d_ovf, d_all, 3 * mx, ncclInt64, (ncclComm_t)c->comm, c->stream));
        CUDA_TRY(c, cudaMemcpyAsync(all.data(), d_all, all.size() * 8, cudaMemcpyDeviceToHost, c->stream));
        CUDA_TRY(c, cudaStreamSynchronize(c->stream));
    }
    for (size_t sl = 0; sl < slots; sl++) {
        DupCounters& dc = c->opt[sl];
        for (int k = 0; k < 7; k++) dc.ctr[k] = h[sl * per + k];
        for (int w = 0; w < 3; w++) { dc.hist[w].clear(); for (int k = 0; k < OPT_HBINS; k++) if (h[sl * per + 7 + w * OPT_HBINS + k]) dc.hist[w][k] = h[sl * per + 7 + w * OPT_HBINS + k]; }
    }
    for (size_t k = 0; k < mx * W; k++) if (all[3 * k] >= 0) c->opt[(size_t)(all[3 * k] >> 2)].hist[all[3 * k] & 3][all[3 * k + 1]] += all[3 * k + 2];
    return ELP_OK;
}

}  // extern "C"
