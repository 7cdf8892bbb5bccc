// host/rendezvous.hpp — the meeting point of the lock-step back end (svsdf_optimize_lockstep).  CUDA-free, so it is tested on the
// CPU (tests/cpp/lockstep_host_main.cpp).
//
// Every problem in flight runs its own solver on its own host thread.  Its evaluation callback does the host half of the evaluation,
// then arrives here with its slot.  A ROUND fires when every live problem (in flight and not finished) has arrived: the thread whose
// arrival completes the round runs fire(slots) for all of them — one batched device evaluation — and then releases the others.  A
// thread that goes on with another problem keeps its place (the new problem arrives with its first evaluation); a thread with no
// problem left departs, the number of live problems drops by one, and if everyone left is already waiting the departing thread fires
// their round.
//
// Each problem's evaluations are the same whichever problems share its rounds, so what a problem computes depends neither on the
// number of problems in flight nor on the order in which they are taken.
#pragma once
#include <algorithm>
#include <condition_variable>
#include <cstdint>
#include <mutex>
#include <vector>

namespace svsdf {
namespace host {

class Rendezvous {
   public:
    // live: problems in flight at the start (each will arrive before any of them can be released)
    explicit Rendezvous(int live) : live_(live) {}

    // Slot `slot` waits for its round; returns once fire() has run on a list of slots that includes it.
    template <class Fire>
    void arrive(int slot, Fire &&fire) {
        std::unique_lock<std::mutex> lk(m_);
        waiting_.push_back(slot);
        if ((int)waiting_.size() == live_) {
            run(lk, fire);
            return;
        }
        const uint64_t g = gen_;
        cv_.wait(lk, [&] { return gen_ != g; });
    }

    // A live slot leaves for good (its thread has no problem left).
    template <class Fire>
    void depart(Fire &&fire) {
        std::unique_lock<std::mutex> lk(m_);
        --live_;
        if (live_ > 0 && (int)waiting_.size() == live_) run(lk, fire);
    }

    int64_t rounds() const {
        std::lock_guard<std::mutex> lk(m_);
        return rounds_;
    }

   private:
    // Called with the lock held and every live problem waiting: nobody else can change the state until the round is released.
    template <class Fire>
    void run(std::unique_lock<std::mutex> &lk, Fire &fire) {
        std::vector<int> slots;
        slots.swap(waiting_);
        std::sort(slots.begin(), slots.end());
        lk.unlock();
        fire(slots);
        lk.lock();
        ++rounds_;
        ++gen_;
        cv_.notify_all();
    }

    mutable std::mutex m_;
    std::condition_variable cv_;
    int live_;
    std::vector<int> waiting_;
    uint64_t gen_ = 0;
    int64_t rounds_ = 0;
};

}  // namespace host
}  // namespace svsdf
