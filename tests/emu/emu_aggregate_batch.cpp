// tests/emu/emu_aggregate_batch.cpp -- TEST HARNESS ONLY: hbls_aggregate_sigs_batch run on the host in hbls.cu's launch order
// (HB_HOST_EMU): the signature decode with the subgroup test one "thread" after the other, then the chunk table k_g2_segsum_plan as a
// CTA of a few host threads meeting at __syncthreads, the chunk sums k_g2_segsum_chunks and the per-set fold k_g2_segsum_fold as
// 32-thread CTAs (one warp each) on 32 host threads whose shuffles and votes meet at a barrier, and k_g2_serialize.  Built with
// -DHB_AGG_CHUNK shrunk to a few rows, sets of a dozen signatures span several chunks.  Never linked into libhbls.so.
#define HB_HOST_EMU 1
#include <condition_variable>
#include <cstring>
#include <cstdint>
#include <cstddef>
#include <mutex>
#include <thread>
#include <vector>
struct hb_dim3 { unsigned x, y, z; };
static thread_local hb_dim3 threadIdx = {0, 0, 0}, blockIdx = {0, 0, 0}, blockDim = {1, 1, 1}, gridDim = {1, 1, 1};
#define __global__
#define __shared__ static
#define __restrict__
#define __launch_bounds__(...)
struct uint4 { unsigned x, y, z, w; };
static inline void __syncwarp() {}
static inline unsigned __funnelshift_l(unsigned lo, unsigned hi, unsigned sh) { sh &= 31; return sh ? (hi << sh) | (lo >> (32 - sh)) : hi; }
// one CTA of blockDim.x host threads at a time: every thread of it meets at the barrier
static std::mutex emu_b_mu;
static std::condition_variable emu_b_cv;
static unsigned emu_b_arrived = 0, emu_b_gen = 0;
static void emu_barrier() {
    std::unique_lock<std::mutex> lk(emu_b_mu);
    const unsigned gen = emu_b_gen;
    if (++emu_b_arrived == blockDim.x) { emu_b_arrived = 0; emu_b_gen++; emu_b_cv.notify_all(); }
    else emu_b_cv.wait(lk, [&] { return emu_b_gen != gen; });
}
// warp primitives in a 32-thread CTA: every lane publishes its word, all meet, each reads what it needs, all meet
static uint32_t emu_w_slot[32];
static inline unsigned __ballot_sync(unsigned, bool p) {
    const unsigned lane = threadIdx.x & 31;
    emu_w_slot[lane] = p ? 1u : 0u;
    emu_barrier();
    unsigned m = 0;
    for (unsigned l = 0; l < blockDim.x && l < 32; l++) m |= emu_w_slot[l] << l;
    emu_barrier();
    return m;
}
template <class T> static inline T __shfl_down_sync(unsigned, T v, int off) {
    const unsigned lane = threadIdx.x & 31;
    emu_w_slot[lane] = (uint32_t)v;
    emu_barrier();
    const T got = (T)emu_w_slot[lane + off < 32 ? lane + off : lane];
    emu_barrier();
    return got;
}
#include "../../harmony_b200/csrc/pairing.cuh"
static inline void __syncthreads() { if (blockDim.x > 1) emu_barrier(); }
static inline unsigned atomicAdd(unsigned* p, unsigned v) { unsigned o = *p; *p += v; return o; }
static inline long long clock64() { return 0; }
#include "../../harmony_b200/csrc/kernels.cuh"
using namespace hb;

template <class F> static void run_seq(unsigned grid, unsigned block, F f) {
    gridDim = {grid, 1, 1}; blockDim = {block, 1, 1};
    for (unsigned b = 0; b < grid; b++) for (unsigned t = 0; t < block; t++) { blockIdx = {b, 0, 0}; threadIdx = {t, 0, 0}; f(); }
    gridDim = {1, 1, 1}; blockDim = {1, 1, 1}; blockIdx = {0, 0, 0}; threadIdx = {0, 0, 0};
}
template <class F> static void run_cta(unsigned grid, unsigned block, F f) {     // CTAs of `block` host threads, one after the other
    for (unsigned b = 0; b < grid; b++) {
        std::vector<std::thread> th;
        for (unsigned t = 0; t < block; t++)
            th.emplace_back([&, t] { gridDim = {grid, 1, 1}; blockDim = {block, 1, 1}; blockIdx = {b, 0, 0}; threadIdx = {t, 0, 0}; f(); });
        for (std::thread& x : th) x.join();
    }
}

extern "C" {

// the compile-time chunk size of this build (HB_AGG_CHUNK)
uint32_t emu_agg_chunk() { return HB_AGG_CHUNK; }

// B sets over n signature rows, as hbls.cu aggregate_sigs_batch_body: offsets (B + 1 values, unchecked: a bad range gives
// HB_AGG_BAD_RANGE), out96[96 j] = Serialize(sum of set j), status[j] = HB_AGG_*; plan_threads = the plan CTA's size.
// *direct (nullable) = the sets summed by their fold warp because their chunks did not fit the table.
void emu_agg_batch(size_t B, size_t n, const uint64_t* offsets, const uint8_t* sigs96, unsigned plan_threads, uint8_t* out96, uint8_t* status,
                   uint32_t* direct) {
    const size_t cap = (n + HB_AGG_CHUNK - 1) / HB_AGG_CHUNK + B;
    std::vector<g2a> pts(n ? n : 1); std::vector<uint8_t> ok(n ? n : 1), part_bad(cap, 0xee);
    std::vector<uint64_t> first(B + 1); std::vector<uint32_t> chunk_set(cap, 0xeeeeeeeeu);
    std::vector<g2> part(cap), sum(B);
    run_seq(1, (unsigned)n, [&] { k_g2_decode(n, sigs96, pts.data(), ok.data(), 1); });
    run_cta(1, plan_threads, [&] { k_g2_segsum_plan(B, n, offsets, cap, first.data(), chunk_set.data(), status); });
    run_cta((unsigned)cap, 32, [&] { k_g2_segsum_chunks(B, offsets, first.data(), chunk_set.data(), cap, pts.data(), ok.data(), part.data(), part_bad.data()); });
    run_cta((unsigned)B, 32, [&] { k_g2_segsum_fold(B, offsets, first.data(), cap, pts.data(), ok.data(), part.data(), part_bad.data(), sum.data(), status); });
    run_seq(1, (unsigned)B, [&] { k_g2_serialize(B, sum.data(), out96); });
    if (direct) {
        uint32_t d = 0;
        for (size_t j = 0; j < B; j++)
            if (offsets[j] <= offsets[j + 1] && offsets[j + 1] <= n && first[j] + (offsets[j + 1] - offsets[j] + HB_AGG_CHUNK - 1) / HB_AGG_CHUNK > cap) d++;
        *direct = d;
    }
}

}  // extern "C"
