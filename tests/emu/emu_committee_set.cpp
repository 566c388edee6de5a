// tests/emu/emu_committee_set.cpp -- TEST HARNESS ONLY: the descriptor kernels of hbls_aggregate_verify_set_device run on the host in
// hbls.cu's launch order (HB_HOST_EMU): k_set_tile_sums and k_set_items as CTAs of HB_SET_TILE host threads meeting at __syncthreads,
// one CTA after the other, k_set_tile_scan as one CTA of a chosen size, then k_set_bad_index one "thread" after the other.  Built
// with -DHB_SET_TILE shrunk to a few items, a batch of a few dozen items spans several tiles.  Never linked into libhbls.so.
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
static inline unsigned __ballot_sync(unsigned, bool p) { return p ? 1u : 0u; }      // no warp-cooperative kernel runs here
template <class T> static inline T __shfl_down_sync(unsigned, T v, int) { return v; }
#include "../../harmony_b200/csrc/pairing.cuh"
static inline void __syncthreads() { if (blockDim.x > 1) emu_barrier(); }
static inline unsigned atomicAdd(unsigned* p, unsigned v) { unsigned o = *p; *p += v; return o; }
static inline long long clock64() { return 0; }
#include "../../harmony_b200/csrc/kernels.cuh"
using namespace hb;

template <class F> static void run_cta(unsigned grid, unsigned block, F f) {     // CTAs of `block` host threads, one after the other
    for (unsigned b = 0; b < grid; b++) {
        std::vector<std::thread> th;
        for (unsigned t = 0; t < block; t++)
            th.emplace_back([&, t] { gridDim = {grid, 1, 1}; blockDim = {block, 1, 1}; blockIdx = {b, 0, 0}; threadIdx = {t, 0, 0}; f(); });
        for (std::thread& x : th) x.join();
    }
}

extern "C" {

// the compile-time tile of this build (HB_SET_TILE)
uint32_t emu_set_tile() { return HB_SET_TILE; }

// hbls.cu verify_set_body up to the verify tail, over a set of m committees of slots[0..m) slots whose tables are stand-in addresses
// (never read): committee i's table is table_base + i, the bitmaps start at bitmap_base.  scan_threads = the tile-scan CTA's size.
// -> per item: committee[j] (the set entry its descriptor names, or -1 when it names none), off[j] (its bitmap's byte offset, or
// UINT64_MAX when it has no bitmap), n[j], ok[j]; and results[j] after k_set_bad_index over the verdicts passed in it.
void emu_set_items(size_t k, const uint32_t* index, size_t m, const uint64_t* slots, unsigned scan_threads, int64_t* committee, uint64_t* off,
                   uint64_t* n, uint8_t* ok, uint8_t* results) {
    const g1a* table_base = reinterpret_cast<const g1a*>(uintptr_t(1) << 40);
    const uint8_t* bitmap_base = reinterpret_cast<const uint8_t*>(uintptr_t(1) << 44);
    std::vector<set_entry> ents(m);
    for (size_t i = 0; i < m; i++) ents[i] = set_entry{table_base + i, slots[i]};
    const size_t nt = (k + HB_SET_TILE - 1) / HB_SET_TILE;
    std::vector<uint64_t> tile_sum(nt ? nt : 1, 0xeeeeeeeeeeeeeeeeull);
    std::vector<mask_item> items(k, mask_item{table_base - 1, bitmap_base - 1, 0xeeee});
    run_cta((unsigned)nt, HB_SET_TILE, [&] { k_set_tile_sums(k, index, (uint32_t)m, ents.data(), tile_sum.data()); });
    run_cta(1, scan_threads, [&] { k_set_tile_scan(nt, tile_sum.data()); });
    run_cta((unsigned)nt, HB_SET_TILE, [&] { k_set_items(k, index, (uint32_t)m, ents.data(), tile_sum.data(), bitmap_base, items.data(), ok); });
    blockDim = {1, 1, 1};
    for (size_t j = 0; j < k; j++) { blockIdx = {(unsigned)j, 0, 0}; k_set_bad_index(k, ok, results); }
    blockIdx = {0, 0, 0};
    for (size_t j = 0; j < k; j++) {
        committee[j] = items[j].table ? (int64_t)(items[j].table - table_base) : -1;
        off[j] = items[j].bitmap ? (uint64_t)(items[j].bitmap - bitmap_base) : UINT64_MAX;
        n[j] = items[j].n;
    }
}

}  // extern "C"
