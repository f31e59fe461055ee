// Ring of work-counter slots of one plan: which slot a launch of a persistent kernel gets, and which earlier launch it
// must wait for.  A slot is in flight from acquire() until done(): acquire() never hands out a slot in flight (it blocks
// while all kSlots are), and a reused slot's stream waits on the event the slot's last user recorded in done().  The
// in-flight rule is what protects a launch whose thread is descheduled between acquire and done: kSlots acquisitions by
// other threads in that gap would otherwise come round to its slot, and the new user, waiting only on the launch before
// it, would zero the slot's counter or descriptors under a kernel still running.
//
// Host code only.  The event operations are the template parameter, so that tests/slots_host.cpp can run the ring with
// a fake event that remembers which launch recorded it (tests/test_slots_cpu.py); b200aa.cu uses the CUDA events.
//   Ops::Event, Ops::Stream; int Ops::create(Event &), Ops::record(Event, Stream), Ops::wait(Stream, Event) (0 = ok, else
//   a status returned as it is); void Ops::destroy(Event).  The ring calls them with its mutex held.
#pragma once
#include <condition_variable>
#include <mutex>

namespace b200aa {

template <class Ops>
class SlotRing {
  public:
    using Event = typename Ops::Event;
    using Stream = typename Ops::Stream;
    static constexpr unsigned kSlots = 64;

    SlotRing() = default;
    SlotRing(const SlotRing &) = delete;
    SlotRing &operator=(const SlotRing &) = delete;
    ~SlotRing()
    {
        for (unsigned s = 0; s < kSlots; ++s)
            if (created_[s]) Ops::destroy(event_[s]);
    }

    // slot of one launch on stream st: the next slot not in flight, from where the last acquire stopped; st waits for
    // the last launch that used it.  Call done() once the launch is queued, also when it failed.
    int acquire(Stream st, unsigned &slot)
    {
        std::unique_lock<std::mutex> g(mu_);
        cv_.wait(g, [this] { return held_ < kSlots; });
        unsigned s = next_;
        while (in_flight_[s]) s = (s + 1) % kSlots;
        if (!created_[s]) {
            const int rc = Ops::create(event_[s]);
            if (rc) return rc;
            created_[s] = true;
        }
        if (used_[s]) {
            const int rc = Ops::wait(st, event_[s]);
            if (rc) return rc;
        }
        in_flight_[s] = true;
        ++held_;
        next_ = (s + 1) % kSlots;
        slot = s;
        return 0;
    }

    // the launch that holds `slot` is queued on st: record the slot's event there and free the slot
    int done(Stream st, unsigned slot)
    {
        int rc;
        {
            std::lock_guard<std::mutex> g(mu_);
            rc = Ops::record(event_[slot], st);
            if (!rc) used_[slot] = true;
            in_flight_[slot] = false;
            --held_;
        }
        cv_.notify_one();
        return rc;
    }

  private:
    std::mutex mu_;
    std::condition_variable cv_;
    Event event_[kSlots] = {};
    bool created_[kSlots] = {};
    bool used_[kSlots] = {};         // event_ holds the record of the slot's last user
    bool in_flight_[kSlots] = {};
    unsigned held_ = 0;              // slots in flight
    unsigned next_ = 0;
};

}  // namespace b200aa
