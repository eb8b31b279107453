// Drives the NCCL stand-in (nccl_loopback.cpp, built with -DLOOPBACK_HOST_ONLY) from threads, one per rank, and prints one line per
// case: "<case> ok" or "<case> FAIL <why>".  tests/test_nccl_loopback_cpu.py runs it and pins every line.
#include <nccl.h>

#include <chrono>
#include <climits>
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <functional>
#include <string>
#include <thread>
#include <vector>

extern "C" const char* loopback_stats();
extern "C" void loopback_reset_stats();

namespace {

int g_failures = 0;

void report(const char* name, const std::string& why) {
    if (why.empty()) printf("%s ok\n", name);
    else { printf("%s FAIL %s\n", name, why.c_str()); g_failures++; }
    fflush(stdout);
}

// runs body(rank, comm) on `world` threads over one fresh communicator; collects the first complaint of any rank
std::string run_ranks(int world, const std::function<std::string(int, ncclComm_t)>& body) {
    ncclUniqueId id;
    if (ncclGetUniqueId(&id) != ncclSuccess) return "ncclGetUniqueId failed";
    std::vector<std::string> why(world);
    std::vector<std::thread> th;
    for (int r = 0; r < world; r++)
        th.emplace_back([&, r] {
            ncclComm_t c = nullptr;
            ncclResult_t rc = ncclCommInitRank(&c, world, id, r);
            if (rc != ncclSuccess) { why[r] = std::string("init: ") + ncclGetErrorString(rc); return; }
            why[r] = body(r, c);
            ncclCommDestroy(c);
        });
    for (auto& t : th) t.join();
    for (int r = 0; r < world; r++) if (!why[r].empty()) return "rank " + std::to_string(r) + ": " + why[r];
    return "";
}

bool contains(const char* s, const char* part) { return s && strstr(s, part) != nullptr; }

}  // namespace

int main() {
    const cudaStream_t s = nullptr;

    // sum of int64, in place, with values that wrap and negative ones
    report("allreduce_sum_int64", run_ranks(3, [&](int r, ncclComm_t c) -> std::string {
        std::vector<int64_t> v = {r + 1, -5 * r, INT64_MAX / 2 + r, (int64_t)1 << 40};
        if (ncclAllReduce(v.data(), v.data(), v.size(), ncclInt64, ncclSum, c, s) != ncclSuccess) return "call failed";
        const std::vector<int64_t> want = {6, -15, (int64_t)((uint64_t)(INT64_MAX / 2) * 3 + 3), (int64_t)3 << 40};
        return v == want ? "" : "wrong sum";
    }));

    // max of int32 into a separate buffer, with INT_MIN as "no value"
    report("allreduce_max_int32", run_ranks(4, [&](int r, ncclComm_t c) -> std::string {
        std::vector<int32_t> in = {r == 2 ? 7 : INT_MIN, -r, INT_MIN, r * 1000}, out(4, 0);
        if (ncclAllReduce(in.data(), out.data(), 4, ncclInt32, ncclMax, c, s) != ncclSuccess) return "call failed";
        return out == std::vector<int32_t>{7, 0, INT_MIN, 3000} ? "" : "wrong max";
    }));

    report("allreduce_other_ops_refused", run_ranks(2, [&](int, ncclComm_t c) -> std::string {
        int32_t x = 1;
        ncclResult_t rc = ncclAllReduce(&x, &x, 1, ncclInt32, ncclSum, c, s);
        return rc == ncclInvalidArgument && contains(ncclGetErrorString(rc), "only sum of int64 and max of int32") ? "" : "not refused";
    }));

    report("allgather_uint32", run_ranks(4, [&](int r, ncclComm_t c) -> std::string {
        std::vector<uint32_t> in = {(uint32_t)r, (uint32_t)(10 * r), 0xffffffffu - r}, out(12, 0);
        if (ncclAllGather(in.data(), out.data(), 3, ncclUint32, c, s) != ncclSuccess) return "call failed";
        for (int q = 0; q < 4; q++)
            if (out[3 * q] != (uint32_t)q || out[3 * q + 1] != (uint32_t)(10 * q) || out[3 * q + 2] != 0xffffffffu - q) return "wrong gather";
        return "";
    }));

    // grouped send / receive: rank a sends (a + 1) * (b + 1) % 4 bytes to rank b (zero for some pairs, never posted), in the order
    // comm.cu posts them (send to r, then receive from r, for r = 0 .. world - 1), and two messages to the same peer keep their order
    report("grouped_send_recv", run_ranks(4, [&](int r, ncclComm_t c) -> std::string {
        auto len = [](int a, int b) { return (size_t)(((a + 1) * (b + 1)) % 4); };
        std::vector<std::vector<uint8_t>> sendb(4), recvb(4), recv2(4);
        std::vector<uint8_t> second = {(uint8_t)(0xa0 + r)}, got2(4 * 1, 0);
        ncclGroupStart();
        for (int q = 0; q < 4; q++) {
            sendb[q].assign(len(r, q), (uint8_t)(16 * r + q));
            recvb[q].assign(len(q, r), 0);
            if (!sendb[q].empty()) ncclSend(sendb[q].data(), sendb[q].size(), ncclChar, q, c, s);
            if (!recvb[q].empty()) ncclRecv(recvb[q].data(), recvb[q].size(), ncclChar, q, c, s);
        }
        const int nxt = (r + 1) % 4, prv = (r + 3) % 4;
        ncclSend(second.data(), 1, ncclChar, nxt, c, s);
        ncclRecv(&got2[0], 1, ncclChar, prv, c, s);
        if (ncclGroupEnd() != ncclSuccess) return std::string("group failed: ") + ncclGetErrorString(ncclSystemError);
        for (int q = 0; q < 4; q++)
            for (uint8_t b : recvb[q]) if (b != (uint8_t)(16 * q + r)) return "wrong bytes from rank " + std::to_string(q);
        return got2[0] == (uint8_t)(0xa0 + prv) ? "" : "second message out of order";
    }));

    // a rank with nothing to move still reaches the group end; the other two exchange
    report("empty_group_on_one_rank", run_ranks(3, [&](int r, ncclComm_t c) -> std::string {
        uint64_t mine = 100 + r, got = 0;
        int32_t sync = 0;
        if (ncclAllReduce(&sync, &sync, 1, ncclInt32, ncclMax, c, s) != ncclSuccess) return "setup failed";
        ncclGroupStart();
        if (r < 2) { ncclSend(&mine, 8, ncclChar, 1 - r, c, s); ncclRecv(&got, 8, ncclChar, 1 - r, c, s); }
        if (ncclGroupEnd() != ncclSuccess) return "group failed";
        return r == 2 || got == (uint64_t)(101 - r) ? "" : "wrong exchange";
    }));

    // ranks that make different calls all fail, with a text naming both calls; the communicator is unusable afterwards
    loopback_reset_stats();
    report("mismatched_operation", run_ranks(2, [&](int r, ncclComm_t c) -> std::string {
        int64_t a[2] = {0, 0}, b[4];
        ncclResult_t rc = r == 0 ? ncclAllReduce(a, a, 2, ncclInt64, ncclSum, c, s) : ncclAllGather(a, b, 2, ncclInt64, c, s);
        const char* e = ncclGetErrorString(rc);
        if (rc != ncclInvalidUsage || !contains(e, "ranks disagree") || !contains(e, "ncclAllReduce") || !contains(e, "ncclAllGather")) return std::string("wrong refusal: ") + e;
        rc = ncclAllReduce(a, a, 2, ncclInt64, ncclSum, c, s);
        return rc != ncclSuccess && contains(ncclGetErrorString(rc), "ranks disagree") ? "" : "the communicator still works";
    }));
    report("mismatch_counted", contains(loopback_stats(), "\"mismatches\": 2") ? "" : loopback_stats());

    report("mismatched_count", run_ranks(3, [&](int r, ncclComm_t c) -> std::string {
        int64_t a[3] = {0, 0, 0};
        ncclResult_t rc = ncclAllReduce(a, a, r == 1 ? 3 : 2, ncclInt64, ncclSum, c, s);
        return rc == ncclInvalidUsage && contains(ncclGetErrorString(rc), "count 3") ? "" : "not refused";
    }));

    report("mismatched_type", run_ranks(2, [&](int r, ncclComm_t c) -> std::string {
        uint32_t a[2] = {0, 0}, b[4];
        ncclResult_t rc = ncclAllGather(a, b, r ? 1 : 2, r ? ncclInt64 : ncclUint32, c, s);
        return rc == ncclInvalidUsage ? "" : "not refused";
    }));

    // rank 0 sends 8 bytes to rank 1, which expects 16: both fail, nothing is copied
    loopback_reset_stats();
    report("send_recv_byte_mismatch", run_ranks(2, [&](int r, ncclComm_t c) -> std::string {
        uint8_t buf[16];
        memset(buf, r ? 0x11 : 0x22, sizeof buf);
        ncclGroupStart();
        if (r == 0) ncclSend(buf, 8, ncclChar, 1, c, s);
        else ncclRecv(buf, 16, ncclChar, 0, c, s);
        ncclResult_t rc = ncclGroupEnd();
        const char* e = ncclGetErrorString(rc);
        if (rc != ncclInvalidUsage || !contains(e, "rank 0 sends 8 bytes to rank 1, which receives 16")) return std::string("wrong refusal: ") + e;
        return buf[0] == (r ? 0x11 : 0x22) ? "" : "bytes were copied";
    }));
    report("p2p_mismatch_counted", contains(loopback_stats(), "\"p2p_mismatches\": 2") ? "" : loopback_stats());

    // rank 1 skips the all-reduce: rank 0 fails after the timeout (LOOPBACK_NCCL_TIMEOUT, 1 s here) with a text naming rank 1 and the call;
    // rank 1's next call fails at once
    loopback_reset_stats();
    report("timeout_names_the_missing_rank", run_ranks(2, [&](int r, ncclComm_t c) -> std::string {
        int64_t a = 1;
        if (r == 1) {
            std::this_thread::sleep_for(std::chrono::milliseconds(2500));
            const auto t0 = std::chrono::steady_clock::now();
            ncclResult_t rc = ncclAllGather(&a, &a, 1, ncclInt64, c, s);
            const double dt = std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
            return rc != ncclSuccess && dt < 0.5 && contains(ncclGetErrorString(rc), "never arrived") ? "" : "a late rank still waited";
        }
        const auto t0 = std::chrono::steady_clock::now();
        ncclResult_t rc = ncclAllReduce(&a, &a, 1, ncclInt64, ncclSum, c, s);
        const double dt = std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
        const char* e = ncclGetErrorString(rc);
        if (rc != ncclSystemError || !contains(e, "rank 1 never arrived at ncclAllReduce (call 2 of rank 0) within 1 s")) return std::string("wrong text: ") + e;
        return dt >= 0.9 && dt < 2.0 ? "" : "waited " + std::to_string(dt) + " s";
    }));
    report("timeout_counted", contains(loopback_stats(), "\"timeouts\": 1") ? "" : loopback_stats());

    // the counters of a clean run
    loopback_reset_stats();
    run_ranks(2, [&](int r, ncclComm_t c) -> std::string {
        int64_t a[3] = {1, 2, 3}; uint32_t g[6] = {0, 0, 1, 2, 3, 4}; uint8_t x = (uint8_t)r, y = 0;
        ncclAllReduce(a, a, 3, ncclInt64, ncclSum, c, s);
        ncclAllGather(g, g + 2, 2, ncclUint32, c, s);
        ncclGroupStart(); ncclSend(&x, 1, ncclChar, 1 - r, c, s); ncclRecv(&y, 1, ncclChar, 1 - r, c, s); ncclGroupEnd();
        return "";
    });
    const char* want = "{\"calls\": {\"ncclCommInitRank\": 2, \"ncclAllReduce\": 2, \"ncclAllGather\": 2, \"ncclGroupEnd\": 2, \"ncclSend\": 2, \"ncclRecv\": 2}, "
                       "\"bytes\": {\"ncclCommInitRank\": 0, \"ncclAllReduce\": 48, \"ncclAllGather\": 32, \"ncclGroupEnd\": 0, \"ncclSend\": 2, \"ncclRecv\": 0}, "
                       "\"timeouts\": 0, \"mismatches\": 0, \"p2p_mismatches\": 0, \"other_failures\": 0}";
    report("stats", strcmp(loopback_stats(), want) == 0 ? "" : loopback_stats());

    return g_failures ? 1 : 0;
}
