// pool.hpp -- the host thread pool of the library's host-side steps (BGZF blocks in bgzf.cpp, float texts in sam_format.cu):
// f(i) for i < n on up to `threads` threads, handing out indices 16 at a time.
#pragma once
#include <algorithm>
#include <atomic>
#include <cstddef>
#include <thread>
#include <vector>

template <class F> void pool_for(size_t n, int threads, F f) {
    threads = std::max(1, std::min<int>(threads, (int)std::max<size_t>(n, 1)));
    if (threads == 1) { for (size_t i = 0; i < n; i++) f(i); return; }
    std::atomic<size_t> next{0};
    std::vector<std::thread> th;
    for (int t = 0; t < threads; t++) th.emplace_back([&]() { for (;;) { const size_t i = next.fetch_add(16); if (i >= n) break; for (size_t k = i; k < std::min(n, i + 16); k++) f(k); } });
    for (auto& x : th) x.join();
}
