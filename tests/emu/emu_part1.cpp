// tests/emu/emu_part1.cpp -- TEST HARNESS ONLY: the kernels that serve combined herumi-API calls (k_single with a descriptor
// array, k_broadcast_hm as an index gather) run on the host with HB_HOST_EMU, one "thread" after the other, so that n requests in
// one launch can be diffed against the same requests launched one at a time.  Never linked into libhbls.so.
#define HB_HOST_EMU 1
#include <cstring>
#include <cstdint>
#include <cstddef>
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
static inline unsigned __ballot_sync(unsigned, bool p) { return p ? 1u : 0u; }
#include "../../harmony_b200/csrc/pairing.cuh"
static inline void __syncthreads() { if (blockDim.x == 2) hb::hb_emu_exchange(0); }
static inline unsigned atomicAdd(unsigned* p, unsigned v) { unsigned o = *p; *p += v; return o; }
static inline long long clock64() { return 0; }
template <class T> static inline T __shfl_down_sync(unsigned, T v, int) { return v; }
#include "../../harmony_b200/csrc/kernels.cuh"
using namespace hb;

template <class F> static void run_seq(unsigned grid, unsigned block, F f) {
    gridDim = {grid, 1, 1}; blockDim = {block, 1, 1};
    for (unsigned b = 0; b < grid; b++) for (unsigned t = 0; t < block; t++) { blockIdx = {b, 0, 0}; threadIdx = {t, 0, 0}; f(); }
    gridDim = {1, 1, 1}; blockDim = {1, 1, 1}; blockIdx = {0, 0, 0}; threadIdx = {0, 0, 0};
}

// ops[i] = {op, ia, ib, len}: operand a / b = slot ia / ib (288 bytes each, -1 = none) of `slots`.  Runs the n ops as ONE k_single
// launch (descriptor array, 32-thread blocks) and each op alone (null descriptor array, as a lone call or the mask / ballot-box
// sites launch it); results of the combined launch go to out (288 bytes per op) and rc.  0 = both forms agree, else 1 + the first
// op that differs.
extern "C" int emu_single_mix(size_t n, const int* ops, const uint8_t* slots, uint8_t* out, int* rc) {
    std::vector<uint8_t> mix(n * 288, 0), lone(n * 288, 0);
    std::vector<int> rc_mix(n, -7), rc_lone(n, -7);
    std::vector<single_desc> d(n);
    auto slot = [&](int k) -> const void* { return k < 0 ? nullptr : slots + (size_t)288 * k; };
    for (size_t i = 0; i < n; i++) d[i] = single_desc{slot(ops[4 * i + 1]), slot(ops[4 * i + 2]), mix.data() + 288 * i, ops[4 * i], (uint32_t)ops[4 * i + 3]};
    run_seq((unsigned)((n + 31) / 32), 32, [&] { k_single(n, d.data(), d[0], rc_mix.data()); });
    for (size_t i = 0; i < n; i++) {
        single_desc one = d[i]; one.out = lone.data() + 288 * i;
        run_seq(1, 32, [&] { k_single(1, (const single_desc*)nullptr, one, &rc_lone[i]); });
    }
    std::memcpy(out, mix.data(), n * 288); std::memcpy(rc, rc_mix.data(), n * sizeof(int));
    for (size_t i = 0; i < n; i++)
        if (rc_mix[i] != rc_lone[i] || std::memcmp(&mix[288 * i], &lone[288 * i], 288) != 0) return 1 + (int)i;
    return 0;
}

// k_broadcast_hm: idx != null gathers src[idx[i]] to every i; idx == null replicates entry 0 in place (same-message batches).
// 0 = both as expected, 1 = the gather differs, 2 = the broadcast differs
extern "C" int emu_hm_gather(size_t n, size_t nsrc, const uint32_t* idx) {
    std::vector<g2a> src(nsrc), hm(n); std::vector<uint8_t> src_ok(nsrc), ok(n, 0xee);
    for (size_t k = 0; k < nsrc; k++) {
        uint8_t* p = reinterpret_cast<uint8_t*>(&src[k]);
        for (size_t b = 0; b < sizeof(g2a); b++) p[b] = (uint8_t)(k * 37 + b * 11 + 1);
        src_ok[k] = (uint8_t)(k & 1);
    }
    run_seq((unsigned)((n + 255) / 256), 256, [&] { k_broadcast_hm(n, idx, src.data(), src_ok.data(), hm.data(), ok.data()); });
    for (size_t i = 0; i < n; i++)
        if (ok[i] != src_ok[idx[i]] || std::memcmp(&hm[i], &src[idx[i]], sizeof(g2a)) != 0) return 1;
    std::vector<g2a> b(n); std::vector<uint8_t> bok(n, 0xee);
    b[0] = src[nsrc - 1]; bok[0] = 1;
    run_seq((unsigned)((n + 255) / 256), 256, [&] { k_broadcast_hm(n, (const uint32_t*)nullptr, (const g2a*)b.data(), (const uint8_t*)bok.data(), b.data(), bok.data()); });
    for (size_t i = 0; i < n; i++)
        if (bok[i] != 1 || std::memcmp(&b[i], &src[nsrc - 1], sizeof(g2a)) != 0) return 2;
    return 0;
}
