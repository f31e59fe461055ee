// A team of host threads for kernel 13's builders (pyaudioanalysis_b200/csrc/forest.cuh): run_team(n, body) runs
// body(forest::Team) on n std::threads, thread t as tid t, all meeting at one barrier at every Team::sync() as a CTA's
// threads meet at __syncthreads().  A team of one runs on the calling thread with no barrier.  Used by
// tests/forest_host.cu, tests/forest_regression_host.cu and tests/boosting_host.cu.
#pragma once
#include <atomic>
#include <thread>
#include <vector>

#include "forest.cuh"

namespace team_host {

// Sense-counting spin barrier: the last thread to arrive resets the count and starts the next generation; the others
// yield until it does.  The acquire / release pairs order every write before the barrier ahead of every read after it
// (and make them visible to ThreadSanitizer).
struct Barrier {
    explicit Barrier(int n) : n(n) {}
    const int n;
    std::atomic<int> count{0};
    std::atomic<unsigned> gen{0};
    void arrive()
    {
        const unsigned g = gen.load(std::memory_order_acquire);
        if (count.fetch_add(1, std::memory_order_acq_rel) == n - 1) {
            count.store(0, std::memory_order_relaxed);
            gen.fetch_add(1, std::memory_order_acq_rel);
            return;
        }
        while (gen.load(std::memory_order_acquire) == g) std::this_thread::yield();
    }
    static void wait(void *self) { static_cast<Barrier *>(self)->arrive(); }
};

template <class Body>
void run_team(int n, const Body &body)
{
    using b200aa::forest::Team;
    if (n <= 1) {
        body(Team{0, 1});
        return;
    }
    Barrier bar(n);
    std::vector<std::thread> th;
    for (int t = 1; t < n; ++t) th.emplace_back([&, t] { body(Team{t, n, &Barrier::wait, &bar}); });
    body(Team{0, n, &Barrier::wait, &bar});
    for (auto &x : th) x.join();
}

}  // namespace team_host
