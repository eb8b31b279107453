// nccl_loopback.cpp -- an in-process stand-in for libnccl.so.2, for testing the library's several-GPU path on one GPU.
//
// Ranks are threads of one process; every rank uses the same device.  It implements exactly the NCCL calls the library resolves
// (elprep_b200/csrc/comm.cu, nccl_api) with the types of the system nccl.h.  Every collective:
//   1. synchronizes the caller's stream, so the kernels before the call have finished;
//   2. meets all ranks of the communicator at a host rendezvous;
//   3. moves the data on the caller's stream: device-to-device copies (all-gather, send / receive), or a host reduction over host
//      copies (all-reduce: sum of int64 and max of int32, the only two the library uses), and synchronizes that stream, so that the
//      data has landed before any rank goes on and a peer may reuse its send buffer;
//   4. meets all ranks again and returns.
// Send / receive inside a group are recorded and run at ncclGroupEnd, which every rank reaches (stricter ordering than NCCL's; the
// library's stream-ordered use allows it).
//
// Three checks of its own, each failing the call with an ncclResult_t error, a text from ncclGetErrorString, and a count in
// loopback_stats():
//   * every rendezvous waits a bounded time (LOOPBACK_NCCL_TIMEOUT seconds, default 60): a rank that never arrives fails the call on
//     the ranks that did, naming the missing rank and the call.  Nothing ever waits on the GPU, so a mismatched call sequence ends as a
//     failed call, never as a hung device.  After that the communicator is broken: every later call on it fails at once;
//   * every rank must make the same call (operation, count, type, reduction) at the same point of its call sequence;
//   * within a group, the bytes rank a sends to rank b must equal the bytes b receives from a, for every pair of ranks.
//
// -DLOOPBACK_HOST_ONLY builds it without CUDA calls (copies are memcpy, stream syncs do nothing), for testing it on a machine
// without a GPU.
#include <nccl.h>

#include <algorithm>
#include <atomic>
#include <chrono>
#include <condition_variable>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <map>
#include <memory>
#include <mutex>
#include <string>
#include <vector>

#define EXPORT extern "C" __attribute__((visibility("default")))

namespace {

enum Op { OP_INIT, OP_ALLREDUCE, OP_ALLGATHER, OP_GROUP, OP_SEND, OP_RECV, N_OPS };
const char* const OP_NAME[N_OPS] = {"ncclCommInitRank", "ncclAllReduce", "ncclAllGather", "ncclGroupEnd", "ncclSend", "ncclRecv"};

size_t type_size(ncclDataType_t t) {
    switch (t) {
        case ncclInt8: case ncclUint8: return 1;
        case ncclFloat16: case ncclBfloat16: return 2;
        case ncclInt32: case ncclUint32: case ncclFloat32: return 4;
        case ncclInt64: case ncclUint64: case ncclFloat64: return 8;
        default: return 0;
    }
}

// queued on the caller's stream; the data has arrived only after stream_sync(s), which every collective calls before its second rendezvous
bool copy_bytes(void* dst, const void* src, size_t n, cudaStream_t s) {
    if (!n || dst == src) return true;
#ifdef LOOPBACK_HOST_ONLY
    (void)s;
    memcpy(dst, src, n);
    return true;
#else
    return cudaMemcpyAsync(dst, src, n, cudaMemcpyDefault, s) == cudaSuccess;
#endif
}
bool stream_sync(cudaStream_t s) {
#ifdef LOOPBACK_HOST_ONLY
    (void)s;
    return true;
#else
    return cudaStreamSynchronize(s) == cudaSuccess;
#endif
}

struct P2P { bool send; int peer; size_t bytes; const void* sbuf; void* rbuf; };

// what one rank posts for the call in progress
struct Post {
    int op = -1; uint64_t seq = 0; size_t count = 0; int dtype = -1; int redop = -1;
    const void* sbuf = nullptr; void* rbuf = nullptr;
    std::vector<uint8_t> host;   // all-reduce: the rank's input, copied to the host
    std::vector<P2P> p2p;        // group: the recorded sends and receives
};

struct Group {
    int world = 0;
    std::mutex mu; std::condition_variable cv;
    uint64_t gen = 0; int arrived = 0;
    std::vector<bool> here;
    std::vector<Post> post;
    std::vector<uint64_t> seq;   // calls made per rank
    bool broken = false; std::string why;
};

struct Stats {
    std::atomic<long long> calls[N_OPS], bytes[N_OPS];
    std::atomic<long long> timeouts, mismatches, p2p_mismatches, other_failures;
};
Stats g_stats;
std::mutex g_reg_mu;
std::map<std::string, std::shared_ptr<Group>> g_reg;
std::atomic<uint64_t> g_next_id{1};

thread_local std::string t_err;
thread_local int t_group_depth = 0;
thread_local std::vector<P2P> t_p2p;
thread_local struct ncclComm* t_p2p_comm = nullptr;
thread_local cudaStream_t t_p2p_stream = nullptr;
thread_local struct ncclComm* t_last_comm = nullptr;   // the communicator this thread (this rank) last used

double timeout_s() {
    const char* e = getenv("LOOPBACK_NCCL_TIMEOUT");
    const double v = e ? atof(e) : 0;
    return v > 0 ? v : 60.0;
}

ncclResult_t failure(ncclResult_t r, std::atomic<long long>& counter, const std::string& msg) {
    counter++;
    t_err = msg;
    return r;
}

}  // namespace

struct ncclComm { std::shared_ptr<Group> g; int rank; };

namespace {

std::string call_name(int op, uint64_t seq, int rank) {
    return std::string(OP_NAME[op]) + " (call " + std::to_string(seq) + " of rank " + std::to_string(rank) + ")";
}

// Meets all ranks of g.  false: timeout or a broken communicator (t_err says which).  Called with lk held.
bool rendezvous(Group& g, std::unique_lock<std::mutex>& lk, int rank, const std::string& what) {
    if (g.broken) { failure(ncclInvalidUsage, g_stats.other_failures, g.why); return false; }
    const uint64_t my = g.gen;
    g.here[rank] = true;
    if (++g.arrived == g.world) {
        g.arrived = 0; g.gen++;
        std::fill(g.here.begin(), g.here.end(), false);
        g.cv.notify_all();
        return true;
    }
    const auto limit = std::chrono::duration<double>(timeout_s());
    if (g.cv.wait_for(lk, limit, [&] { return g.gen != my || g.broken; }) && g.gen != my) return true;
    if (!g.broken) {
        std::string missing;
        for (int r = 0; r < g.world; r++) if (!g.here[r]) missing += (missing.empty() ? "" : ", ") + std::to_string(r);
        char buf[64]; snprintf(buf, sizeof buf, "%g", timeout_s());
        g.broken = true;
        g.why = "loopback NCCL: rank " + missing + " never arrived at " + what + " within " + buf + " s";
        g.cv.notify_all();
        failure(ncclSystemError, g_stats.timeouts, g.why);
    } else {
        failure(ncclInvalidUsage, g_stats.other_failures, g.why);
    }
    return false;
}

bool same_call(const Post& a, const Post& b) { return a.op == b.op && a.seq == b.seq && a.count == b.count && a.dtype == b.dtype && a.redop == b.redop; }

std::string describe(const Post& p) {
    return std::string(OP_NAME[p.op]) + " #" + std::to_string(p.seq) + " count " + std::to_string(p.count) + " type " + std::to_string(p.dtype) +
           " op " + std::to_string(p.redop);
}

// one collective: post, rendezvous, check the calls agree, move the data (move(g) under no lock; it returns once its copies have
// landed), rendezvous
template <class Move>
ncclResult_t collective(ncclComm* c, Post p, const cudaStream_t* s, Move move) {
    if (!c) return failure(ncclInvalidArgument, g_stats.other_failures, "loopback NCCL: null communicator");
    t_last_comm = c;
    if (s && !stream_sync(*s)) return failure(ncclUnhandledCudaError, g_stats.other_failures, "loopback NCCL: cudaStreamSynchronize failed");
    Group& g = *c->g;
    std::unique_lock<std::mutex> lk(g.mu);
    p.seq = ++g.seq[c->rank];
    const std::string what = call_name(p.op, p.seq, c->rank);
    g.post[c->rank] = std::move(p);
    if (!rendezvous(g, lk, c->rank, what)) return ncclSystemError;
    // every rank runs the same checks on the same posts, so all of them fail or none
    std::string bad;
    for (int r = 1; r < g.world && bad.empty(); r++)
        if (!same_call(g.post[0], g.post[r])) bad = "loopback NCCL: ranks disagree on the call: rank 0 " + describe(g.post[0]) + ", rank " + std::to_string(r) + " " + describe(g.post[r]);
    if (bad.empty() && g.post[0].op == OP_GROUP) {
        for (int a = 0; a < g.world && bad.empty(); a++)
            for (int b = 0; b < g.world && bad.empty(); b++) {
                size_t sent = 0, recvd = 0;
                for (auto& x : g.post[a].p2p) if (x.send && x.peer == b) sent += x.bytes;
                for (auto& x : g.post[b].p2p) if (!x.send && x.peer == a) recvd += x.bytes;
                if (sent != recvd) bad = "loopback NCCL: rank " + std::to_string(a) + " sends " + std::to_string(sent) + " bytes to rank " + std::to_string(b) +
                                         ", which receives " + std::to_string(recvd) + " from it";
            }
        if (!bad.empty()) g_stats.p2p_mismatches++;
    } else if (!bad.empty()) {
        g_stats.mismatches++;
    }
    bool moved = true;
    if (bad.empty()) { lk.unlock(); moved = move(g); lk.lock(); }
    if (!rendezvous(g, lk, c->rank, what + ", leaving")) return ncclSystemError;
    if (!bad.empty()) { g.broken = true; g.why = bad; t_err = bad; return ncclInvalidUsage; }   // the call sequences have parted: later calls fail at once
    if (!moved) return failure(ncclUnhandledCudaError, g_stats.other_failures, "loopback NCCL: a copy failed in " + what);
    return ncclSuccess;
}

}  // namespace

EXPORT ncclResult_t ncclGetUniqueId(ncclUniqueId* id) {
    if (!id) return ncclInvalidArgument;
    memset(id->internal, 0, sizeof id->internal);
    snprintf(id->internal, sizeof id->internal, "loopback-%llu", (unsigned long long)g_next_id++);
    return ncclSuccess;
}

EXPORT ncclResult_t ncclCommInitRank(ncclComm_t* comm, int nranks, ncclUniqueId id, int rank) {
    if (!comm || nranks < 1 || rank < 0 || rank >= nranks) return failure(ncclInvalidArgument, g_stats.other_failures, "loopback NCCL: bad ncclCommInitRank arguments");
    std::shared_ptr<Group> g;
    {
        std::lock_guard<std::mutex> lk(g_reg_mu);
        auto& slot = g_reg[std::string(id.internal, strnlen(id.internal, sizeof id.internal))];
        if (!slot) {
            slot = std::make_shared<Group>();
            slot->world = nranks; slot->here.assign(nranks, false); slot->post.resize(nranks); slot->seq.assign(nranks, 0);
        }
        g = slot;
    }
    if (g->world != nranks) return failure(ncclInvalidUsage, g_stats.mismatches, "loopback NCCL: ncclCommInitRank with " + std::to_string(nranks) + " ranks, the id has " + std::to_string(g->world));
    auto* c = new ncclComm{g, rank};
    Post p; p.op = OP_INIT; p.count = (size_t)nranks;
    g_stats.calls[OP_INIT]++;
    ncclResult_t r = collective(c, std::move(p), nullptr, [](Group&) { return true; });
    if (r != ncclSuccess) t_last_comm = nullptr;
    if (r != ncclSuccess) { delete c; return r; }
    *comm = c;
    return ncclSuccess;
}

EXPORT ncclResult_t ncclCommDestroy(ncclComm_t comm) {
    if (t_last_comm == comm) t_last_comm = nullptr;
    delete comm;
    return ncclSuccess;
}

EXPORT ncclResult_t ncclAllReduce(const void* sendbuff, void* recvbuff, size_t count, ncclDataType_t datatype, ncclRedOp_t op, ncclComm_t comm, cudaStream_t stream) {
    if (t_group_depth) return failure(ncclInvalidUsage, g_stats.other_failures, "loopback NCCL: ncclAllReduce inside a group");
    g_stats.calls[OP_ALLREDUCE]++;
    const bool sum64 = op == ncclSum && (datatype == ncclInt64 || datatype == ncclUint64), max32 = op == ncclMax && datatype == ncclInt32;
    if (!sum64 && !max32) return failure(ncclInvalidArgument, g_stats.other_failures, "loopback NCCL: only sum of int64 and max of int32 are implemented");
    if (!stream_sync(stream)) return failure(ncclUnhandledCudaError, g_stats.other_failures, "loopback NCCL: cudaStreamSynchronize failed");
    const size_t bytes = count * type_size(datatype);   // (the input is copied to the host before the rendezvous: send and receive buffer may be one)
    Post p; p.op = OP_ALLREDUCE; p.count = count; p.dtype = datatype; p.redop = op; p.sbuf = sendbuff; p.rbuf = recvbuff;
    p.host.resize(bytes);
    if (!copy_bytes(p.host.data(), sendbuff, bytes, stream) || !stream_sync(stream)) return failure(ncclUnhandledCudaError, g_stats.other_failures, "loopback NCCL: copy of the all-reduce input failed");
    const int me = comm ? comm->rank : 0;
    return collective(comm, std::move(p), nullptr, [&](Group& g) {
        std::vector<uint8_t> out(bytes);
        if (sum64) {
            int64_t* o = reinterpret_cast<int64_t*>(out.data());
            for (size_t k = 0; k < count; k++) {
                uint64_t s = 0;   // two's complement wrap, as NCCL's
                for (int r = 0; r < g.world; r++) s += reinterpret_cast<const uint64_t*>(g.post[r].host.data())[k];
                o[k] = (int64_t)s;
            }
        } else {
            int32_t* o = reinterpret_cast<int32_t*>(out.data());
            for (size_t k = 0; k < count; k++) {
                int32_t m = reinterpret_cast<const int32_t*>(g.post[0].host.data())[k];
                for (int r = 1; r < g.world; r++) m = std::max(m, reinterpret_cast<const int32_t*>(g.post[r].host.data())[k]);
                o[k] = m;
            }
        }
        g_stats.bytes[OP_ALLREDUCE] += (long long)bytes;
        return copy_bytes(g.post[me].rbuf, out.data(), bytes, stream) && stream_sync(stream);   // (before `out` goes away)
    });
}

EXPORT ncclResult_t ncclAllGather(const void* sendbuff, void* recvbuff, size_t sendcount, ncclDataType_t datatype, ncclComm_t comm, cudaStream_t stream) {
    if (t_group_depth) return failure(ncclInvalidUsage, g_stats.other_failures, "loopback NCCL: ncclAllGather inside a group");
    g_stats.calls[OP_ALLGATHER]++;
    const size_t bytes = sendcount * type_size(datatype);
    if (!type_size(datatype)) return failure(ncclInvalidArgument, g_stats.other_failures, "loopback NCCL: unknown data type");
    Post p; p.op = OP_ALLGATHER; p.count = sendcount; p.dtype = datatype; p.sbuf = sendbuff; p.rbuf = recvbuff;
    const int me = comm ? comm->rank : 0;
    return collective(comm, std::move(p), &stream, [&](Group& g) {
        bool ok = true;
        for (int r = 0; r < g.world; r++) ok = copy_bytes(static_cast<uint8_t*>(g.post[me].rbuf) + (size_t)r * bytes, g.post[r].sbuf, bytes, stream) && ok;
        g_stats.bytes[OP_ALLGATHER] += (long long)(bytes * g.world);
        return stream_sync(stream) && ok;
    });
}

EXPORT ncclResult_t ncclGroupStart() {
    if (t_group_depth++ == 0) { t_p2p.clear(); t_p2p_comm = nullptr; t_p2p_stream = nullptr; }
    return ncclSuccess;
}

namespace {
ncclResult_t record_p2p(bool send, const void* sbuf, void* rbuf, size_t count, ncclDataType_t datatype, int peer, ncclComm_t comm, cudaStream_t stream) {
    g_stats.calls[send ? OP_SEND : OP_RECV]++;
    if (!comm || peer < 0 || peer >= comm->g->world || !type_size(datatype)) return failure(ncclInvalidArgument, g_stats.other_failures, "loopback NCCL: bad send / receive arguments");
    if (t_group_depth && t_p2p_comm && (t_p2p_comm != comm || t_p2p_stream != stream))
        return failure(ncclInvalidUsage, g_stats.other_failures, "loopback NCCL: one group over several communicators or streams");
    t_p2p_comm = comm; t_p2p_stream = stream;
    t_p2p.push_back(P2P{send, peer, count * type_size(datatype), sbuf, rbuf});
    return ncclSuccess;
}
ncclResult_t run_group() {
    std::vector<P2P> ops; ops.swap(t_p2p);
    // A group with nothing in it still meets the other ranks on the communicator this rank last used: every rank must reach every group
    // end (stricter than NCCL, where an empty group does nothing), so a rank that skips an exchange is caught even when it had nothing to move.
    const bool empty = t_p2p_comm == nullptr;
    ncclComm* comm = empty ? t_last_comm : t_p2p_comm;
    cudaStream_t stream = t_p2p_stream;
    t_p2p_comm = nullptr; t_p2p_stream = nullptr;
    if (!comm) return ncclSuccess;
    Post p; p.op = OP_GROUP; p.p2p = ops;
    const int me = comm->rank;
    return collective(comm, std::move(p), empty ? nullptr : &stream, [&](Group& g) {
        bool ok = true;
        // the k-th receive of rank me from a peer takes the k-th send of that peer to rank me
        std::vector<size_t> taken(g.world, 0);
        for (auto& x : g.post[me].p2p) {
            if (x.send) continue;
            size_t k = 0, want = taken[x.peer]++;
            for (auto& y : g.post[x.peer].p2p) {
                if (!y.send || y.peer != me) continue;
                if (k++ == want) {
                    if (y.bytes != x.bytes) return false;
                    ok = copy_bytes(x.rbuf, y.sbuf, x.bytes, stream) && ok;
                    g_stats.bytes[OP_SEND] += (long long)x.bytes;
                    break;
                }
            }
        }
        return (empty || stream_sync(stream)) && ok;
    });
}
}  // namespace

EXPORT ncclResult_t ncclSend(const void* sendbuff, size_t count, ncclDataType_t datatype, int peer, ncclComm_t comm, cudaStream_t stream) {
    ncclResult_t r = record_p2p(true, sendbuff, nullptr, count, datatype, peer, comm, stream);
    return (r != ncclSuccess || t_group_depth) ? r : run_group();
}

EXPORT ncclResult_t ncclRecv(void* recvbuff, size_t count, ncclDataType_t datatype, int peer, ncclComm_t comm, cudaStream_t stream) {
    ncclResult_t r = record_p2p(false, nullptr, recvbuff, count, datatype, peer, comm, stream);
    return (r != ncclSuccess || t_group_depth) ? r : run_group();
}

EXPORT ncclResult_t ncclGroupEnd() {
    if (t_group_depth == 0) return failure(ncclInvalidUsage, g_stats.other_failures, "loopback NCCL: ncclGroupEnd without ncclGroupStart");
    if (--t_group_depth) return ncclSuccess;
    g_stats.calls[OP_GROUP]++;
    return run_group();
}

EXPORT const char* ncclGetErrorString(ncclResult_t result) {
    if (result != ncclSuccess && !t_err.empty()) return t_err.c_str();
    switch (result) {
        case ncclSuccess: return "no error";
        case ncclSystemError: return "loopback NCCL: system error";
        case ncclInvalidArgument: return "loopback NCCL: invalid argument";
        case ncclInvalidUsage: return "loopback NCCL: invalid usage";
        default: return "loopback NCCL: error";
    }
}

// {"calls": {op: n}, "bytes": {op: n}, "timeouts": n, "mismatches": n, "p2p_mismatches": n, "other_failures": n}
EXPORT const char* loopback_stats() {
    static thread_local std::string s;
    s = "{\"calls\": {";
    for (int k = 0; k < N_OPS; k++) s += std::string(k ? ", " : "") + "\"" + OP_NAME[k] + "\": " + std::to_string(g_stats.calls[k].load());
    s += "}, \"bytes\": {";
    for (int k = 0; k < N_OPS; k++) s += std::string(k ? ", " : "") + "\"" + OP_NAME[k] + "\": " + std::to_string(g_stats.bytes[k].load());
    s += "}, \"timeouts\": " + std::to_string(g_stats.timeouts.load()) + ", \"mismatches\": " + std::to_string(g_stats.mismatches.load()) +
         ", \"p2p_mismatches\": " + std::to_string(g_stats.p2p_mismatches.load()) + ", \"other_failures\": " + std::to_string(g_stats.other_failures.load()) + "}";
    return s.c_str();
}

EXPORT void loopback_reset_stats() {
    for (int k = 0; k < N_OPS; k++) { g_stats.calls[k] = 0; g_stats.bytes[k] = 0; }
    g_stats.timeouts = 0; g_stats.mismatches = 0; g_stats.p2p_mismatches = 0; g_stats.other_failures = 0;
}
