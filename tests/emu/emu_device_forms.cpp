// tests/emu/emu_device_forms.cpp -- TEST HARNESS ONLY: runs the message-grouping and status kernels of
// harmony_b200/csrc/device_forms.cuh on the host (HB_HOST_EMU, as tests/emu/emu_kernels.cpp does for kernels.cuh): the hash-table
// insert one "thread" after the other, in either order, atomics as plain read-modify-writes; the compaction as a CTA of one thread.
// Never linked into libhbls.so; the product has no CPU path.
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
static inline unsigned __ballot_sync(unsigned, bool p) { return p ? 1u : 0u; }      // the warp-cooperative hash forms are not run here
#include "../../harmony_b200/csrc/pairing.cuh"
static inline void __syncthreads() {}                                                  // CTAs of one thread only
static inline unsigned atomicAdd(unsigned* p, unsigned v) { unsigned o = *p; *p += v; return o; }
static inline unsigned atomicCAS(unsigned* p, unsigned cmp, unsigned v) { unsigned o = *p; if (o == cmp) *p = v; return o; }
static inline unsigned atomicMin(unsigned* p, unsigned v) { unsigned o = *p; if (v < o) *p = v; return o; }
static inline long long clock64() { return 0; }
template <class T> static inline T __shfl_down_sync(unsigned, T v, int) { return v; }
#include "../../harmony_b200/csrc/device_forms.cuh"
using namespace hb;

extern "C" {

// hbls.cu launch_hash_grouped up to the hash: k_group_insert (reverse: the "threads" from the last item to the first), then
// k_group_compact, under the table hash key (k0, k1).  -> *d, grp[k], keys[48 k] (the first d rows written), rep[k] (each item's
// representative)
void emu_group(size_t k, const uint8_t* msgs, uint32_t msg_len, int reverse, uint64_t k0, uint64_t k1, unsigned* d, uint32_t* grp, uint8_t* keys,
               uint32_t* rep) {
    size_t T = 64; while (T < 2 * k) T <<= 1;
    std::vector<uint32_t> slot_item(T, HB_GRP_EMPTY), slot_rep(T, HB_GRP_EMPTY), item_slot(k), pos(k);
    gridDim = {1, 1, 1}; blockDim = {(unsigned)k, 1, 1};
    for (size_t u = 0; u < k; u++) {
        threadIdx = {(unsigned)(reverse ? k - 1 - u : u), 0, 0};
        k_group_insert(k, msgs, msg_len, (uint32_t)(T - 1), k0, k1, slot_item.data(), slot_rep.data(), item_slot.data());
    }
    blockDim = {1, 1, 1}; threadIdx = {0, 0, 0};
    k_group_compact(k, msgs, msg_len, slot_rep.data(), item_slot.data(), pos.data(), grp, keys, d);
    for (size_t i = 0; i < k; i++) rep[i] = slot_rep[item_slot[i]];
}

// the table hash of item i (SipHash-2-4 of its 48 key bytes under (k0, k1))
uint64_t emu_group_hash(const uint8_t* msgs, uint32_t msg_len, size_t i, uint64_t k0, uint64_t k1) { return grp_hash(msgs, msg_len, i, k0, k1); }

void emu_status_triples(size_t k, const uint8_t* flags, const uint8_t* results, uint8_t* status) {
    blockDim = {1, 1, 1};
    for (size_t j = 0; j < k; j++) { blockIdx = {(unsigned)j, 0, 0}; k_status_triples(k, flags, results, status); }
    blockIdx = {0, 0, 0};
}

void emu_status_headers(size_t n, size_t nslots, const uint8_t* bitmaps, size_t blen, size_t quorum, const uint8_t* flags, const uint8_t* results,
                        uint8_t* status) {
    blockDim = {1, 1, 1};
    for (size_t j = 0; j < n; j++) { blockIdx = {(unsigned)j, 0, 0}; k_status_headers(n, nslots, bitmaps, blen, quorum, flags, results, status); }
    blockIdx = {0, 0, 0};
}

}  // extern "C"
