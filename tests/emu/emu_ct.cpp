// tests/emu/emu_ct.cpp -- TEST HARNESS ONLY: the four secret-scalar kernels of harmony_b200/csrc/kernels.cuh (k_g1_mul_gen,
// k_sign_hash, k_sign_hm_pair, k_sign_hm_gls_pair) on the host (HB_HOST_EMU; the lane-pair kernels on two host threads), with
// HB_CT_PROBE recording a trace of the complete formulas, table reads and ladder steps each lane executes.  With the executed-work
// counters (hb_emu_cnt_mul / hb_emu_cnt_sqr) the trace must not depend on the key.  Also exports the host key helpers of
// secret_key.hpp.  Never linked into libhbls.so.
#define HB_HOST_EMU 1
#define HB_CT_PROBE_HOST 1
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
#include "../../harmony_b200/csrc/secret_key.hpp"
using namespace hb;

static thread_local std::vector<uint32_t> ct_trace;
namespace hb { void hb_ct_probe(uint32_t tag) { ct_trace.push_back(tag); } }

// what one lane executed: trace length, FNV-1a hash of the trace, Fp products, Fp squarings
struct LaneRecord { uint64_t len, hash, mul, sqr; };
static void lane_begin() { ct_trace.clear(); hb_emu_cnt_mul = 0; hb_emu_cnt_sqr = 0; }
static LaneRecord lane_end() {
    uint64_t h = 0xcbf29ce484222325ull;
    for (uint32_t t : ct_trace) { h ^= t; h *= 0x100000001b3ull; }
    return LaneRecord{ct_trace.size(), h, hb_emu_cnt_mul, hb_emu_cnt_sqr};
}

template <class F> static void run_seq1(F f) {
    gridDim = {1, 1, 1}; blockDim = {1, 1, 1}; blockIdx = {0, 0, 0}; threadIdx = {0, 0, 0};
    f();
}
template <class F> static void run_pair(F f) {                 // one CTA of two threads = one lane pair
    hb_emu_pair_reset();
    auto lane = [&](unsigned t) {
        gridDim = {1, 1, 1}; blockDim = {2, 1, 1}; blockIdx = {0, 0, 0}; threadIdx = {t, 0, 0};
        hb_emu.role = (int)t; hb_emu.seq = 0;
        f(t);
        blockDim = {1, 1, 1}; threadIdx = {0, 0, 0}; hb_emu.role = 0;
    };
    std::thread th(lane, 1u); lane(0u); th.join();
}

// Runs one kernel on one key: kernel 0 k_g1_mul_gen (out: 48-byte public key), 1 k_sign_hash, 2 k_sign_hm_pair, 3 k_sign_hm_gls_pair
// (out: 96-byte signature; H(m) of kernels 2 and 3 comes from k_hash_to_g2 beforehand, outside the record; kernel 3 takes the key's
// base-|z| digits from secret_key.hpp).  rec[0..3] / rec[4..7]: LaneRecord of lane 0 / lane 1 (zeros for thread-per-item kernels).
// Returns the kernel's ok flag (1 for kernel 0), or -2 when kernel 3 gets a key >= Z^4.
extern "C" int emu_ct_run(int kernel, const uint8_t* sk32, const uint8_t* msg, uint32_t len, uint8_t* out, uint64_t* rec) {
    LaneRecord lr[2] = {};
    uint8_t ok = 1;
    if (kernel == 0) {
        g1 p;
        run_seq1([&] { lane_begin(); k_g1_mul_gen(1, sk32, &p); lr[0] = lane_end(); });
        g1_serialize(out, p);
    } else if (kernel == 1) {
        g2 s;
        run_seq1([&] { lane_begin(); k_sign_hash(1, sk32, msg, len, &s, &ok); lr[0] = lane_end(); });
        g2_serialize(out, s);
    } else {
        g2a hm; uint8_t okh = 0;
        run_seq1([&] { k_hash_to_g2(1, msg, len, &hm, &okh); });
        uint64_t sk[4], dig[4]; std::memcpy(sk, sk32, 32);
        if (kernel == 3 && !hb_secret::sk_digits_base_z(sk, dig)) return -2;
        g2 s;
        run_pair([&](unsigned t) {
            lane_begin();
            if (kernel == 2) k_sign_hm_pair(1, sk32, &hm, &okh, 0, &s, &ok);
            else k_sign_hm_gls_pair(1, dig, &hm, &okh, 0, &s, &ok);
            lr[t] = lane_end();
        });
        g2_serialize(out, s);
    }
    for (int t = 0; t < 2; t++) { rec[4 * t] = lr[t].len; rec[4 * t + 1] = lr[t].hash; rec[4 * t + 2] = lr[t].mul; rec[4 * t + 3] = lr[t].sqr; }
    return ok;
}

// the host key helpers: digits (returns sk_digits_base_z's verdict), k < r, 32-byte equality
extern "C" int emu_ct_digits(const uint64_t* sk, uint64_t* dig) { return hb_secret::sk_digits_base_z(sk, dig) ? 1 : 0; }
extern "C" int emu_ct_lt_r(const uint64_t* k) { return hb_secret::scalar_lt_r(k) ? 1 : 0; }
extern "C" int emu_ct_eq32(const uint8_t* a, const uint8_t* b) { return hb_secret::eq32(a, b) ? 1 : 0; }
