// tests/coalesce/coalesce_driver.cpp -- the request combiner of harmony_b200/csrc/coalesce.hpp with a fake executor, built with
// -fsanitize=thread by tests/test_coalesce.py.  Prints "all checks passed" and exits 0, or names the first failed check.
#include "../../harmony_b200/csrc/coalesce.hpp"
#include <atomic>
#include <chrono>
#include <cstdio>
#include <cstdlib>
#include <mutex>
#include <thread>
#include <vector>

using hbls_coalesce::Combiner;
using hbls_coalesce::Request;

static int failures = 0;
#define CHECK(cond, ...) do { if (!(cond)) { std::printf("FAIL %s:%d: ", __FILE__, __LINE__); std::printf(__VA_ARGS__); std::printf("\n"); failures++; } } while (0)

struct FakeReq : Request {
    int value = 0;
    int result = 0;            // value * 2 + 1, or -100 when its turn failed
    int served = 0;            // times an executor ran it
    int turn = -1;             // index of the turn that ran it
};

// executor state: only touched with the outer mutex held
struct Fake {
    std::mutex outer;
    std::vector<size_t> turn_sizes;
    std::vector<std::vector<int>> turn_kinds;       // kinds of each turn's requests
    std::vector<std::thread::id> turn_thread;
    int fail_every = 0, fail_phase = 0;              // turn t fails when fail_every && t % fail_every == fail_phase
    size_t caps[Combiner::kMaxKinds] = {1000, 1000, 1000, 1000, 1000, 1000, 1000, 1000};
    Combiner comb;

    bool turn_fails(int t) const { return fail_every && t % fail_every == fail_phase; }
    void run(FakeReq& r) {
        comb.submit(r, outer, [&](int k) { return caps[k]; }, [&](Request** rq, size_t n) {
            const int t = (int)turn_sizes.size();
            turn_sizes.push_back(n); turn_thread.push_back(std::this_thread::get_id());
            std::vector<int> kinds;
            for (size_t i = 0; i < n; i++) {
                FakeReq* q = static_cast<FakeReq*>(rq[i]);
                q->served++; q->turn = t; kinds.push_back(q->kind);
                q->result = turn_fails(t) ? -100 : q->value * 2 + 1;
            }
            turn_kinds.push_back(kinds);
        });
    }
};

// `threads` callers, `per_thread` requests each (distinct values, kinds 0..3); every request checked after all threads joined
static void stress(int threads, int per_thread, int fail_every) {
    Fake f; f.fail_every = fail_every; f.fail_phase = 1; f.caps[2] = 5;
    std::vector<std::vector<FakeReq>> reqs(threads, std::vector<FakeReq>(per_thread));
    std::vector<std::thread> th;
    for (int t = 0; t < threads; t++)
        th.emplace_back([&, t] {
            for (int i = 0; i < per_thread; i++) {
                FakeReq& r = reqs[t][i];
                r.kind = (t + i) & 3; r.value = t * per_thread + i;
                f.run(r);
                // the result is complete when submit returns
                const int want = f.turn_fails(r.turn) ? -100 : r.value * 2 + 1;
                if (r.result != want || r.served != 1) { std::printf("FAIL: request %d result %d served %d\n", r.value, r.result, r.served); std::abort(); }
            }
        });
    for (auto& x : th) x.join();
    const size_t total = (size_t)threads * per_thread;
    size_t sum = 0, max_turn = 0;
    for (size_t s : f.turn_sizes) { sum += s; if (s > max_turn) max_turn = s; }
    CHECK(sum == total, "threads %d: turn sizes add up to %zu, %zu requests", threads, sum, total);
    const hbls_coalesce::Stats st = f.comb.stats();
    CHECK(st.requests == total && st.turns == f.turn_sizes.size() && st.max_turn == max_turn,
          "threads %d: stats %llu/%llu/%llu", threads, (unsigned long long)st.turns, (unsigned long long)st.requests, (unsigned long long)st.max_turn);
    for (auto& tk : f.turn_kinds) {
        int k2 = 0; for (int k : tk) k2 += k == 2;
        CHECK(k2 <= 5, "threads %d: a turn holds %d requests of the kind capped at 5", threads, k2);
    }
    size_t failed = 0;
    for (auto& row : reqs)
        for (FakeReq& r : row) {
            CHECK(r.served == 1, "request %d served %d times", r.value, r.served);
            if (r.result == -100) { failed++; CHECK(f.turn_fails(r.turn), "request %d failed outside a failing turn", r.value); }
            else CHECK(!f.turn_fails(r.turn) && r.result == r.value * 2 + 1, "request %d result %d", r.value, r.result);
        }
    size_t want_failed = 0;
    for (size_t t = 0; t < f.turn_sizes.size(); t++) if (f.turn_fails((int)t)) want_failed += f.turn_sizes[t];
    CHECK(failed == want_failed, "threads %d: %zu requests failed, the failing turns held %zu", threads, failed, want_failed);
    if (threads == 1) CHECK(max_turn == 1, "a single caller made a turn of %zu", max_turn);
    std::printf("threads %2d: %zu requests in %zu turns (largest %zu)\n", threads, total, f.turn_sizes.size(), max_turn);
}

// a lone request is a turn of one, run by the caller itself
static void lone() {
    Fake f; FakeReq r; r.value = 20;
    f.run(r);
    CHECK(r.result == 41 && r.served == 1, "lone request result %d", r.result);
    CHECK(f.turn_sizes.size() == 1 && f.turn_sizes[0] == 1, "lone request: %zu turns", f.turn_sizes.size());
    CHECK(f.turn_thread.size() == 1 && f.turn_thread[0] == std::this_thread::get_id(), "lone request ran on another thread");
}

// ten callers queue while the outer lock is held elsewhere (a long batch call on the device); with a cap of 3 they are served
// in turns of 3, 3, 3, 1, and a failure of the second turn fails exactly its three requests
static void capped(bool fail_second) {
    Fake f; f.caps[0] = 3; f.fail_every = fail_second ? 1000 : 0; f.fail_phase = 1;
    std::vector<FakeReq> reqs(10);
    std::atomic<int> started{0};
    std::vector<std::thread> th;
    {
        std::unique_lock<std::mutex> hold(f.outer);
        for (int i = 0; i < 10; i++)
            th.emplace_back([&, i] { reqs[i].value = i; started++; f.run(reqs[i]); });
        while (started.load() < 10) std::this_thread::sleep_for(std::chrono::milliseconds(1));
        std::this_thread::sleep_for(std::chrono::milliseconds(200));     // every caller has queued by now
    }
    for (auto& x : th) x.join();
    CHECK((f.turn_sizes == std::vector<size_t>{3, 3, 3, 1}), "capped turns: %zu turns, first %zu", f.turn_sizes.size(), f.turn_sizes.empty() ? 0 : f.turn_sizes[0]);
    int failed = 0;
    for (FakeReq& r : reqs) {
        CHECK(r.served == 1, "capped: request %d served %d times", r.value, r.served);
        if (r.result == -100) { failed++; CHECK(r.turn == 1, "capped: request %d of turn %d failed", r.value, r.turn); }
        else CHECK(r.result == r.value * 2 + 1 && !(fail_second && r.turn == 1), "capped: request %d result %d", r.value, r.result);
    }
    CHECK(failed == (fail_second ? 3 : 0), "capped: %d requests failed", failed);
}

int main() {
    lone();
    capped(false);
    capped(true);
    for (int threads : {1, 2, 8, 64}) stress(threads, 4096 / threads + 500, 0);
    for (int threads : {2, 8, 64}) stress(threads, 4096 / threads + 500, 3);
    if (failures) { std::printf("%d checks failed\n", failures); return 1; }
    std::printf("all checks passed\n");
    return 0;
}
