// CPU exercise of csrc/slots.h (the work-slot ring of a plan) with a fake event that remembers which launch recorded it.
// Built and run by tests/test_slots_cpu.py (g++ -pthread, no GPU).
//   usage: slots_host a|b|c|d  -> one JSON line; exit status 1 when an invariant was broken
//
// Every launch L on a fake stream: acquire -> (hold) -> done.  The checks, at every acquire of slot s by L:
//   * no other launch holds s between its acquire and its done (two unfinished launches never share a slot);
//   * L's stream waits on the record of the launch that last finished with s, and on nothing when s is new.
// The ring calls the fake operations with its mutex held; each thread owns its streams, so no fake state is shared
// outside that mutex.
#include <atomic>
#include <chrono>
#include <cstdio>
#include <cstring>
#include <random>
#include <string>
#include <thread>
#include <vector>
#include "../pyaudioanalysis_b200/csrc/slots.h"
using namespace b200aa;

struct FakeEvent {
    long launch = -1;           // the launch whose done() recorded it last
};
struct FakeStream {
    long launch = -1;           // the launch being queued on this stream
    long waited = -1;           // what that launch's acquire made the stream wait on (-1: nothing)
};
struct FakeOps {
    using Event = FakeEvent *;
    using Stream = FakeStream *;
    static int create(Event &e)
    {
        e = new FakeEvent;
        return 0;
    }
    static int record(Event e, Stream s)
    {
        e->launch = s->launch;
        return 0;
    }
    static int wait(Stream s, Event e)
    {
        s->waited = e->launch;
        return 0;
    }
    static void destroy(Event e) { delete e; }
};
using Ring = SlotRing<FakeOps>;
constexpr unsigned kSlots = Ring::kSlots;

struct Checker {
    std::atomic<long> holder[kSlots];           // launch between acquire and done on the slot, -1 none
    std::atomic<long> last[kSlots];             // last launch that finished with the slot, -1 none
    std::atomic<long> next_id{0}, launches{0}, reuses{0}, shared{0}, bad_wait{0};
    std::atomic<long> wraps{0};                 // acquisitions of slot 0 after its first (the ring came round)
    std::string first;                          // first violation (written once)
    std::atomic<bool> have_first{false};
    Checker()
    {
        for (unsigned s = 0; s < kSlots; ++s) { holder[s] = -1; last[s] = -1; }
    }
    void fail(std::atomic<long> &ctr, const char *what, long L, unsigned s, long a, long b)
    {
        ctr.fetch_add(1);
        bool no = false;
        if (have_first.compare_exchange_strong(no, true)) {
            char buf[200];
            snprintf(buf, sizeof buf, "launch %ld, slot %u: %s (%ld, %ld)", L, s, what, a, b);
            first = buf;
        }
    }
    // one acquire on st; returns the slot
    unsigned acquire(Ring &ring, FakeStream &st, long &L)
    {
        L = next_id.fetch_add(1);
        st.launch = L;
        st.waited = -1;
        unsigned s = 0;
        if (ring.acquire(&st, s) != 0 || s >= kSlots) { fail(shared, "acquire failed", L, s, 0, 0); return 0; }
        launches.fetch_add(1);
        const long prev = holder[s].exchange(L);
        if (prev != -1) fail(shared, "slot still held by", L, s, prev, -1);
        const long want = last[s].load();
        if (want != -1) reuses.fetch_add(1);
        if (want != -1 && s == 0) wraps.fetch_add(1);
        if (st.waited != want) fail(bad_wait, "waited on / last user", L, s, st.waited, want);
        return s;
    }
    void done(Ring &ring, FakeStream &st, long L, unsigned s)
    {
        long me = L;
        if (!holder[s].compare_exchange_strong(me, -1)) fail(shared, "slot taken over by", L, s, me, -1);
        last[s].store(L);
        st.launch = L;
        ring.done(&st, s);
    }
    int report(const char *scenario, const std::string &extra)
    {
        const bool ok = shared.load() == 0 && bad_wait.load() == 0;
        printf("{\"scenario\": \"%s\", \"launches\": %ld, \"reuses\": %ld, \"wraps\": %ld, \"shared\": %ld, \"bad_wait\": %ld%s, "
               "\"first\": \"%s\"}\n",
               scenario, launches.load(), reuses.load(), wraps.load(), shared.load(), bad_wait.load(), extra.c_str(), first.c_str());
        return ok ? 0 : 1;
    }
};

// (a) one thread, 1 000 launches round-robin over 4 streams
static int scenario_a()
{
    Ring ring;
    Checker ck;
    FakeStream st[4];
    for (int i = 0; i < 1000; ++i) {
        long L;
        FakeStream &s = st[i % 4];
        const unsigned slot = ck.acquire(ring, s, L);
        ck.done(ring, s, L, slot);
    }
    return ck.report("a", "");
}

// (b) one launch held between acquire and done while 200 others acquire and finish; then it finishes and 64 more run
static int scenario_b()
{
    Ring ring;
    Checker ck;
    FakeStream held_st, st[4];
    long H;
    const unsigned h = ck.acquire(ring, held_st, H);
    long got_held = 0, reused_after = 0;
    for (int i = 0; i < 200; ++i) {
        long L;
        const unsigned s = ck.acquire(ring, st[i % 4], L);
        if (s == h) ++got_held;
        ck.done(ring, st[i % 4], L, s);
    }
    ck.done(ring, held_st, H, h);
    for (int i = 0; i < 64; ++i) {
        long L;
        const unsigned s = ck.acquire(ring, st[i % 4], L);
        if (s == h) ++reused_after;
        ck.done(ring, st[i % 4], L, s);
    }
    char extra[120];
    snprintf(extra, sizeof extra, ", \"held_slot_given\": %ld, \"held_slot_reused_after\": %ld", got_held, reused_after);
    return ck.report("b", extra) | (got_held != 0) | (reused_after != 1);
}

// (c) 64 launches held; a 65th acquires from another thread and blocks until one of them is done, then gets its slot
static int scenario_c()
{
    Ring ring;
    Checker ck;
    std::vector<FakeStream> st(kSlots + 1);
    long id[kSlots];
    unsigned slot[kSlots];
    for (unsigned i = 0; i < kSlots; ++i) slot[i] = ck.acquire(ring, st[i], id[i]);
    std::atomic<bool> returned{false};
    unsigned got = ~0u;
    long L65 = -1;
    std::thread t([&] {
        got = ck.acquire(ring, st[kSlots], L65);
        returned.store(true);
    });
    std::this_thread::sleep_for(std::chrono::milliseconds(200));
    const bool blocked = !returned.load();
    const unsigned k = 37;                      // free one slot in the middle of the ring
    ck.done(ring, st[k], id[k], slot[k]);
    t.join();
    const bool right_slot = got == slot[k] && st[kSlots].waited == id[k];
    ck.done(ring, st[kSlots], L65, got);
    for (unsigned i = 0; i < kSlots; ++i)
        if (i != k) ck.done(ring, st[i], id[i], slot[i]);
    char extra[120];
    snprintf(extra, sizeof extra, ", \"blocked\": %s, \"got_freed_slot\": %s", blocked ? "true" : "false", right_slot ? "true" : "false");
    return ck.report("c", extra) | !blocked | !right_slot;
}

// (d) 8 threads, each on its own stream, with seeded random hold times between acquire and done
static int scenario_d()
{
    Ring ring;
    Checker ck;
    constexpr int kThreads = 8, kPer = 3000;
    std::vector<std::thread> th;
    for (int t = 0; t < kThreads; ++t)
        th.emplace_back([&, t] {
            std::mt19937 rng(1234 + t);
            FakeStream st;
            for (int i = 0; i < kPer; ++i) {
                long L;
                const unsigned s = ck.acquire(ring, st, L);
                const unsigned r = rng() % 1000;
                if (r < 10) std::this_thread::sleep_for(std::chrono::microseconds(1000));      // descheduled for a while
                else if (r < 100) std::this_thread::sleep_for(std::chrono::microseconds(20));
                else if (r < 500) std::this_thread::yield();
                ck.done(ring, st, L, s);
            }
        });
    for (auto &x : th) x.join();
    return ck.report("d", "");
}

int main(int argc, char **argv)
{
    const char *s = argc > 1 ? argv[1] : "";
    if (!strcmp(s, "a")) return scenario_a();
    if (!strcmp(s, "b")) return scenario_b();
    if (!strcmp(s, "c")) return scenario_c();
    if (!strcmp(s, "d")) return scenario_d();
    fprintf(stderr, "usage: slots_host a|b|c|d\n");
    return 2;
}
