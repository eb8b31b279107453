// CPU check of the team code of the DEFLATE decoder and encoder: elprep_b200/csrc/inflate.cuh and deflate.cuh, compiled here as host C++
// for host teams of K lanes, each lane a std::thread, against the team of one lane (Serial, SerialEnc) that inflate_check.cpp and
// deflate_check.cpp compare with zlib.  The team of one runs none of the code that exists because of the team: the lane-split table builds
// and copies of the decoder and the syncs that order them; the encoder's hash-chain groups, guess-and-repair parse, per-segment bit offsets
// and the ORs of two segments into one output word.  Here every lane of a call must return the same value as every other lane and as the
// team of one, with the same output bytes, whatever K is; built with -fsanitize=thread, no access may race.
//
// HostTeam<K> has the members the two headers use, with the device's semantics:
//   sync()           a std::barrier of the K lanes (__syncthreads, __syncwarp)
//   any(b)           __syncthreads_or: each lane ORs b into a flag, a barrier, every lane reads the flag, a barrier; two flag slots used in
//                    turn, so the slot lane 0 clears after the second barrier is not the one the next call ORs into
//   or32, add32      atomicOr, atomicAdd: std::atomic_ref
//   chain()          the chain team of min(K, 32) lanes (lanes chain_lane()), with its own barrier: same(h) publishes h, waits, builds the
//                    mask of the lanes with an equal h and waits again (__match_any_sync); lt() = (1 << lane) - 1 (lanemask_lt)
//
//   team_check full   the decoder at K = 2, 7, 32 on the crafted and edge streams of inflate_corpus.hpp and every 10th zlib stream; the
//                     encoder at K = 2, 3, 7, 32, 33, 255, 256 on every input of deflate_corpus.hpp up to 5500 bytes and the long edge inputs
//                     of the repair rounds, the segment offsets and the hash3 collisions (the chain team's barriers make long inputs slow)
//   team_check tsan   the subset for a ThreadSanitizer build: the decoder at K = 32 on the crafted streams and every 30th zlib stream, the
//                     encoder at K = 7 and 256 on the edge inputs up to 5500 bytes, the 0xff00-byte run and one segment-offset input
// Both print the counts and OK.  The encoder's corpus must contain an input that needs no repair round at K = 256, one that needs at least
// 200, and one with a parse segment whose entry lies at or past its end (it gets no tokens).
#include <atomic>
#include <barrier>
#include <cstdio>
#include <cstring>
#include <memory>
#include <random>
#include <string>
#include <thread>
#include <vector>
#include "inflate.cuh"
#include "deflate.cuh"
#include "inflate_corpus.hpp"
#include "deflate_corpus.hpp"

static int failures = 0;
static void fail(const std::string& what) { if (failures < 20) std::printf("FAIL %s\n", what.c_str()); failures++; }

template <unsigned N>
struct ChainShared {
    std::barrier<> bar{N};
    uint32_t h[N];
};

template <unsigned N>
struct HostChain {
    static constexpr unsigned size = N;
    unsigned lane;
    ChainShared<N>* sh;
    void sync() const { sh->bar.arrive_and_wait(); }
    uint32_t same(uint32_t h) const {
        sh->h[lane] = h;
        sync();
        uint32_t m = 0;
        for (unsigned k = 0; k < N; k++) m |= (uint32_t)(sh->h[k] == h) << k;
        sync();
        return m;
    }
    uint32_t lt() const { return (1u << lane) - 1u; }
};

template <unsigned K>
struct TeamShared {
    static constexpr unsigned CH = K < 32 ? K : 32;
    std::barrier<> bar{K};
    uint32_t flag[2] = {0, 0};
    unsigned any_calls = 0;                     // (lane 0's count)
    ChainShared<CH> chain;
};

template <unsigned K>
struct HostTeam {
    static constexpr unsigned size = K;
    unsigned lane;
    TeamShared<K>* sh;
    mutable unsigned turn = 0;
    void sync() const { sh->bar.arrive_and_wait(); }
    bool any(bool b) const {
        std::atomic_ref<uint32_t> f(sh->flag[turn++ & 1]);
        if (b) f.fetch_or(1u);
        sync();
        const bool r = f.load() != 0;
        sync();
        if (lane == 0) { f.store(0u); sh->any_calls++; }
        return r;
    }
    void or32(uint32_t* p, uint32_t v) const { std::atomic_ref<uint32_t>(*p).fetch_or(v); }
    void add32(uint32_t* p, uint32_t v) const { std::atomic_ref<uint32_t>(*p).fetch_add(v); }
    bool chain_lane() const { return lane < TeamShared<K>::CH; }
    HostChain<TeamShared<K>::CH> chain() const { return {lane, &sh->chain}; }
};

// fn(team) on K threads; -> every lane's return value
template <unsigned K, class Fn>
static std::vector<uint32_t> run_team(TeamShared<K>& sh, Fn fn) {
    std::vector<uint32_t> r(K);
    std::vector<std::thread> th;
    th.reserve(K);
    for (unsigned l = 0; l < K; l++) th.emplace_back([&, l] { const HostTeam<K> t{l, &sh}; r[l] = fn(t); });
    for (auto& t : th) t.join();
    return r;
}

template <class V>
static bool all_equal(const V& r) { for (auto x : r) if (x != r[0]) return false; return true; }

// ---- decoder ----
struct DecStats { int streams = 0, accepted = 0; };

template <unsigned K>
static void decode_team(const std::string& name, const corpus::Bytes& in, uint32_t isize, uint32_t want_st, const corpus::Bytes& want, DecStats& st) {
    auto sh = std::make_unique<TeamShared<K>>();
    auto T = std::make_unique<dfl::Tables>();
    corpus::Bytes out(isize ? isize : 1, 0);
    const auto r = run_team<K>(*sh, [&](const HostTeam<K>& t) { return dfl::inflate_stream(t, *T, in.data(), (uint32_t)in.size(), out.data(), isize); });
    st.streams++;
    st.accepted += r[0] == dfl::OK;
    const std::string at = "decoder K " + std::to_string(K) + " " + name + " (isize " + std::to_string(isize) + ")";
    if (!all_equal(r)) fail(at + ": the lanes return different statuses");
    else if (r[0] != want_st) fail(at + ": status " + dfl::status_text(r[0]) + ", the team of one: " + dfl::status_text(want_st));
    else if (out != want) fail(at + ": output bytes differ from the team of one");
}

template <unsigned... Ks>
static void decoder(bool subset) {
    std::mt19937_64 rng(12345);
    DecStats st[sizeof...(Ks)];
    int n_zlib = 0;
    corpus::for_each_stream(rng, [&](corpus::InfKind kind, const std::string& name, const corpus::Bytes& in, uint32_t isize) {
        const bool zlib_pick = kind == corpus::ZLIB && n_zlib++ % (subset ? 30 : 10) == 0;
        if (!(kind == corpus::CRAFTED || zlib_pick || (!subset && kind == corpus::EDGE))) return;
        auto T = std::make_unique<dfl::Tables>();
        corpus::Bytes want(isize ? isize : 1, 0);
        const uint32_t want_st = dfl::inflate_stream(dfl::Serial{}, *T, in.data(), (uint32_t)in.size(), want.data(), isize);
        int k = 0;
        (decode_team<Ks>(name, in, isize, want_st, want, st[k++]), ...);
    });
    int k = 0;
    ((std::printf("decoder K %u: %d streams (%d accepted)\n", Ks, st[k].streams, st[k].accepted), k++), ...);
}

// ---- encoder ----
struct EncOut { corpus::Bytes bytes; std::vector<uint32_t> match; };

static EncOut encode_serial(const corpus::Bytes& d) {
    auto S = std::make_unique<dfl::EncShared>();
    std::vector<uint16_t> prev(65536);
    EncOut o{{}, std::vector<uint32_t>(65536)};
    std::vector<uint32_t> w((dfl::stored_bytes((uint32_t)d.size()) + 3) / 4, 0xa5a5a5a5u);
    const uint32_t n = dfl::deflate_block(dfl::SerialEnc{}, *S, dfl::EncScratch{prev.data(), o.match.data()}, d.data(), (uint32_t)d.size(), w.data());
    o.bytes.assign(reinterpret_cast<uint8_t*>(w.data()), reinterpret_cast<uint8_t*>(w.data()) + n);
    return o;
}

struct EncStats {
    int inputs = 0, no_repair = 0, empty_segments = 0;
    unsigned most_rounds = 0;
    std::string no_repair_name, most_name, empty_name;
};

// parse segments (Team::size of them, deflate_block's split) whose entry in the serial parse over match[] lies at or past their end
static int segments_past_end(const std::vector<uint32_t>& match, uint32_t n, unsigned K) {
    const uint32_t seg = (n + K - 1) / K;
    int c = 0;
    uint32_t p = 0;
    for (unsigned k = 0; k < K; k++) {
        const uint32_t s0 = k * seg < n ? k * seg : n, s1 = s0 + seg < n ? s0 + seg : n;
        if (s0 >= n) break;
        c += p >= s1;
        while (p < s1) p = dfl::next_pos(match.data(), p, n);
    }
    return c;
}

template <unsigned K>
static void encode_team(const std::string& name, const corpus::Bytes& d, const EncOut& want, EncStats& st) {
    auto sh = std::make_unique<TeamShared<K>>();
    auto S = std::make_unique<dfl::EncShared>();
    std::vector<uint16_t> prev(65536);
    std::vector<uint32_t> match(65536);
    std::vector<uint32_t> w((dfl::stored_bytes((uint32_t)d.size()) + 3) / 4, 0xa5a5a5a5u);
    const auto r = run_team<K>(*sh, [&](const HostTeam<K>& t) {
        return dfl::deflate_block(t, *S, dfl::EncScratch{prev.data(), match.data()}, d.data(), (uint32_t)d.size(), w.data());
    });
    st.inputs++;
    const std::string at = "encoder K " + std::to_string(K) + " " + name + " (n " + std::to_string(d.size()) + ")";
    if (!all_equal(r)) { fail(at + ": the lanes return different lengths"); return; }
    const corpus::Bytes got(reinterpret_cast<uint8_t*>(w.data()), reinterpret_cast<uint8_t*>(w.data()) + r[0]);
    if (got != want.bytes) fail(at + ": bytes differ from the team of one (" + std::to_string(got.size()) + " vs " + std::to_string(want.bytes.size()) + " bytes)");
    if (!std::equal(match.begin(), match.begin() + d.size(), want.match.begin())) fail(at + ": match[] differs from the team of one");
    const unsigned rounds = sh->any_calls - 1;             // the last any() finds every segment right
    if (rounds == 0 && st.no_repair++ == 0) st.no_repair_name = name;
    if (rounds > st.most_rounds || st.most_name.empty()) { st.most_rounds = rounds; st.most_name = name; }
    const int e = segments_past_end(match, (uint32_t)d.size(), K);
    if (e && st.empty_segments == 0) st.empty_name = name;
    st.empty_segments += e;
}

template <unsigned... Ks>
static void encoder(bool subset) {
    std::mt19937_64 rng(20261017);
    EncStats st[sizeof...(Ks)];
    corpus::for_each_input(rng, [&](corpus::DefKind kind, const std::string& name, const corpus::Bytes& d) {
        // (the chain team's two barriers per 32 positions cost most: of the long inputs, the ones that make the team's edge cases)
        const bool big = d.size() > 5500, edge_big = name == "edge run n 65280" || name.find("offsets") != std::string::npos || name == "edge hash3 collisions";
        const bool pick = subset ? kind == corpus::TEAM_EDGE && (!big || name == "edge run n 65280" || name.find("offsets 2") != std::string::npos)
                                 : !big || edge_big;
        if (!pick) return;
        const EncOut want = encode_serial(d);
        int k = 0;
        (encode_team<Ks>(name, d, want, st[k++]), ...);
    });
    int k = 0;
    ((std::printf("encoder K %u: %d inputs; %d without a repair round (%s); most repair rounds %u (%s); %d segments with the entry at or past "
                  "their end (first in %s)\n", Ks, st[k].inputs, st[k].no_repair, st[k].no_repair_name.c_str(), st[k].most_rounds, st[k].most_name.c_str(),
                  st[k].empty_segments, st[k].empty_name.c_str()), k++), ...);
    const EncStats& s256 = st[sizeof...(Ks) - 1];                 // (the largest team last)
    if (s256.no_repair == 0) fail("the encoder corpus has no input without a repair round at the largest team");
    if (s256.most_rounds < 200) fail("the encoder corpus has no input with 200 repair rounds at the largest team");
    if (s256.empty_segments == 0) fail("the encoder corpus has no parse segment whose entry lies at or past its end at the largest team");
}

int main(int argc, char** argv) {
    const bool full = argc == 2 && !std::strcmp(argv[1], "full"), tsan = argc == 2 && !std::strcmp(argv[1], "tsan");
    if (!full && !tsan) { std::fprintf(stderr, "usage: team_check full|tsan\n"); return 2; }
    if (full) { decoder<2, 7, 32>(false); encoder<2, 3, 7, 32, 33, 255, 256>(false); }
    else { decoder<32>(true); encoder<7, 256>(true); }
    std::printf("%d failures\n", failures);
    if (failures) return 1;
    std::printf("OK\n");
    return 0;
}
