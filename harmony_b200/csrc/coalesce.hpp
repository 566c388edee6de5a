// harmony_b200/csrc/coalesce.hpp -- combines concurrent calls from different threads into shared turns (host only, no CUDA).
//
// A caller describes its call in a Request on its own stack and submits it.  If no turn is running the caller becomes the leader:
// it takes the outer lock (the library mutex that serialises device work), drains the queue within per-kind caps and runs the
// whole turn through the executor on its own thread.  Otherwise it sleeps until its request is done or leadership is handed to it.
// There is no library thread, timer or batching window: a caller that finds the combiner idle runs at once as a turn of one.
// When a turn ends with requests still queued, leadership passes to the oldest of them, so callers that return from a turn and
// submit again queue behind the running turn instead of starting turns of one beside it.
#pragma once
#include <condition_variable>
#include <cstddef>
#include <cstdint>
#include <deque>
#include <mutex>
#include <vector>

namespace hbls_coalesce {

struct Request {
    int kind = 0;              // in [0, Combiner::kMaxKinds): selects the per-turn cap; the executor interprets the rest
    bool done = false;         // guarded by the combiner's mutex
};

struct Stats { uint64_t turns = 0, requests = 0, max_turn = 0; };

// every kind counts against its own cap
struct OwnCap { int operator()(int kind) const { return kind; } };

class Combiner {
public:
    static constexpr int kMaxKinds = 8;

    // Runs r inside some turn and returns once the executor has filled in its results.
    //   outer:    locked by the leader before it drains the queue (requests that arrive while another holder has it join the turn)
    //   cap(k):   most requests of kind k in one turn (read with `outer` held; 0 counts as 1); the rest wait for the next turn
    //   exec(rq, n): runs one turn on the leader's thread with `outer` held; must complete every one of the n requests
    //   pool(k):  the kind whose cap a request of kind k counts against (kinds that share one device stage share one cap)
    template <class Outer, class Cap, class Exec, class Pool = OwnCap>
    void submit(Request& r, Outer& outer, Cap&& cap, Exec&& exec, Pool&& pool = Pool{}) {
        std::unique_lock<std::mutex> lk(mu_);
        queue_.push_back(&r);
        for (;;) {
            cv_.wait(lk, [&] { return r.done || !running_ || next_ == &r; });
            if (r.done) return;
            running_ = true; next_ = nullptr;
            lk.unlock();
            std::vector<Request*> turn;
            {
                std::lock_guard<Outer> og(outer);
                size_t caps[kMaxKinds], taken[kMaxKinds] = {};
                for (int k = 0; k < kMaxKinds; k++) { caps[k] = (size_t)cap(k); if (caps[k] == 0) caps[k] = 1; }
                lk.lock();
                std::deque<Request*> rest;
                for (Request* q : queue_) {
                    const int p = pool(q->kind);
                    if (taken[p] < caps[p]) { taken[p]++; turn.push_back(q); }
                    else rest.push_back(q);
                }
                queue_.swap(rest);
                stats_.turns++; stats_.requests += turn.size();
                if (turn.size() > stats_.max_turn) stats_.max_turn = turn.size();
                lk.unlock();
                exec(turn.data(), turn.size());
            }
            lk.lock();
            for (Request* q : turn) q->done = true;
            if (queue_.empty()) running_ = false;
            else next_ = queue_.front();
            cv_.notify_all();
        }
    }

    Stats stats() { std::lock_guard<std::mutex> lk(mu_); return stats_; }

private:
    std::mutex mu_;
    std::condition_variable cv_;
    std::deque<Request*> queue_;       // submitted, not yet taken into a turn (oldest first)
    bool running_ = false;             // a leader exists (running a turn, or named in next_ and about to)
    Request* next_ = nullptr;          // the queued request whose caller leads the next turn
    Stats stats_;
};

}  // namespace hbls_coalesce
