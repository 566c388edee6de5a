// tests/emu/emu_part1_committee.cpp -- TEST HARNESS ONLY: one combined Part-1 turn of hbls.cu part1_locked with committee checks
// (hbls_aggregate_verify), resident-mask checks (hbls_mask_verify) and VerifyHash requests, run on the host with HB_HOST_EMU: the
// warp kernels (k_mask_aggregate_items, k_mask_aggregate) on 32 host threads whose shuffles meet at a barrier, the lane-pair kernels
// on two host threads, the rest one "thread" after the other.  The pairing is the lane-pair form the turn launches when coop_max is 0
// (k_pairing_verify_split + k_pairing_fixup).  Never linked into libhbls.so.
#define HB_HOST_EMU 1
#include <condition_variable>
#include <cstring>
#include <cstdint>
#include <cstddef>
#include <map>
#include <array>
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
static inline unsigned __ballot_sync(unsigned, bool p) { return p ? 1u : 0u; }      // the warp pairing k_pairing_coop is not run here
#include "../../harmony_b200/csrc/pairing.cuh"
static inline void __syncthreads() { if (blockDim.x == 2) hb::hb_emu_exchange(0); }
static inline unsigned atomicAdd(unsigned* p, unsigned v) { unsigned o = *p; *p += v; return o; }
static inline long long clock64() { return 0; }
// a warp of 32 host threads: every lane publishes its word, all meet, each reads lane + off (its own beyond the warp), all meet again
static std::mutex emu_w_mu;
static std::condition_variable emu_w_cv;
static unsigned emu_w_arrived = 0, emu_w_gen = 0;
static uint32_t emu_w_slot[32];
static void emu_w_barrier() {
    std::unique_lock<std::mutex> lk(emu_w_mu);
    const unsigned gen = emu_w_gen;
    if (++emu_w_arrived == 32) { emu_w_arrived = 0; emu_w_gen++; emu_w_cv.notify_all(); }
    else emu_w_cv.wait(lk, [&] { return emu_w_gen != gen; });
}
template <class T> static inline T __shfl_down_sync(unsigned, T v, int off) {
    const unsigned lane = threadIdx.x & 31;
    emu_w_slot[lane] = (uint32_t)v;
    emu_w_barrier();
    const T got = (T)emu_w_slot[lane + off < 32 ? lane + off : lane];
    emu_w_barrier();
    return got;
}
#include "../../harmony_b200/csrc/kernels.cuh"
using namespace hb;

template <class F> static void run_seq(unsigned grid, unsigned block, F f) {
    gridDim = {grid, 1, 1}; blockDim = {block, 1, 1};
    for (unsigned b = 0; b < grid; b++) for (unsigned t = 0; t < block; t++) { blockIdx = {b, 0, 0}; threadIdx = {t, 0, 0}; f(); }
    gridDim = {1, 1, 1}; blockDim = {1, 1, 1}; blockIdx = {0, 0, 0}; threadIdx = {0, 0, 0};
}
template <class F> static void run_pair(F f) {                 // one CTA of two threads = one lane pair, persistent over all items
    hb_emu_pair_reset();
    auto lane = [&](unsigned t) {
        gridDim = {1, 1, 1}; blockDim = {2, 1, 1}; blockIdx = {0, 0, 0}; threadIdx = {t, 0, 0};
        hb_emu.role = (int)t; hb_emu.seq = 0;
        f();
        blockDim = {1, 1, 1}; threadIdx = {0, 0, 0}; hb_emu.role = 0;
    };
    std::thread th(lane, 1u); lane(0u); th.join();
}
template <class F> static void run_warps(unsigned grid, F f) {  // 32-thread CTAs (one warp each), one after the other
    for (unsigned b = 0; b < grid; b++) {
        std::vector<std::thread> th;
        for (unsigned t = 0; t < 32; t++)
            th.emplace_back([&, t] { gridDim = {grid, 1, 1}; blockDim = {32, 1, 1}; blockIdx = {b, 0, 0}; threadIdx = {t, 0, 0}; f(); });
        for (std::thread& x : th) x.join();
    }
}

enum { RQ_VERIFY = 0, RQ_AGG = 4, RQ_MASK = 5 };               // hbls.cu request kinds

extern "C" {

// k requests of kind[i] (RQ_VERIFY / RQ_AGG / RQ_MASK) over nc committees (their keys back to back in keys48, sizes[c] keys each).
//   AGG / MASK: committee com[i] and its bitmap (the next (n + 7) / 8 bytes of `bitmaps`); MASK: the mask holds that bitmap, its
//               resident aggregate built from an empty mask as hbls_mask_set_mask builds it
//   VERIFY:     the serialized key pk48[i] (deserialized into the struct blsPublicKeyDeserialize makes)
//   all:        the serialized signature sig96[i] (VERIFY: deserialized into the struct) and message msgs[64 i], lens[i] bytes
// results[i] = the turn's verdict.  Returns 0, or -3 when a committee key or a VERIFY struct does not decode.
int emu_committee_turn(size_t nc, const uint8_t* keys48, const uint32_t* sizes, size_t k, const int* kind, const int* com,
                       const uint8_t* bitmaps, const uint8_t* pk48, const uint8_t* sig96, const uint8_t* msgs, const uint32_t* lens,
                       uint8_t* results) {
    // committee tables (hbls_committee_create)
    std::vector<std::vector<g1a>> tables(nc);
    for (size_t c = 0, off = 0; c < nc; off += sizes[c], c++) {
        tables[c].resize(sizes[c] ? sizes[c] : 1);
        std::vector<uint8_t> ok(sizes[c] ? sizes[c] : 1, 1);
        run_seq(1, sizes[c], [&] { k_g1_decode(sizes[c], keys48 + 48 * off, tables[c].data(), ok.data(), 1, 0); });
        for (uint32_t i = 0; i < sizes[c]; i++) if (!ok[i]) return -3;
    }
    std::vector<const uint8_t*> bm(k, nullptr);
    for (size_t i = 0, off = 0; i < k; i++)
        if (kind[i] != RQ_VERIFY) { bm[i] = bitmaps + off; off += (sizes[com[i]] + 7) >> 3; }
    // the turn's order: AGG, MASK, VERIFY (each kind in arrival order)
    std::vector<size_t> ver;
    for (int want : {RQ_AGG, RQ_MASK, RQ_VERIFY}) for (size_t i = 0; i < k; i++) if (kind[i] == want) ver.push_back(i);
    size_t na = 0, nser = 0;
    for (size_t i : ver) { na += kind[i] == RQ_AGG; nser += kind[i] != RQ_VERIFY; }
    const size_t nv = ver.size();
    // keys: one Jacobian array.  AGG: k_mask_aggregate_items over mask_item descriptors; MASK: the resident aggregate (k_mask_aggregate
    // of the bitmap's Add row, then k_single G1_ADD into the identity), copied in; VERIFY: the deserialized struct
    std::vector<g1> apk(nv);
    std::vector<mask_item> items(na);
    for (size_t j = 0; j < na; j++) items[j] = mask_item{tables[com[ver[j]]].data(), bm[ver[j]], (uint64_t)sizes[com[ver[j]]]};
    if (na) run_warps((unsigned)na, [&] { k_mask_aggregate_items(na, items.data(), apk.data()); });
    for (size_t j = na; j < nser; j++) {
        const size_t i = ver[j], n = sizes[com[i]];
        g1 acc, sum; memset(&acc, 0, sizeof acc); int rc = 0;
        run_warps(1, [&] { k_mask_aggregate(1, n, tables[com[i]].data(), bm[i], (n + 7) >> 3, &sum); });
        const single_desc d{&acc, &sum, &acc, OP_G1_ADD, 0u};
        run_seq(1, 1, [&] { k_single(1, (const single_desc*)nullptr, d, &rc); });
        apk[j] = acc;
    }
    std::vector<g2> vsig_struct(nv - nser);
    for (size_t j = nser; j < nv; j++) {
        const size_t i = ver[j]; int rc1 = 0, rc2 = 0;
        const single_desc dp{pk48 + 48 * i, nullptr, &apk[j], OP_G1_DES, 0u}, ds{sig96 + 96 * i, nullptr, &vsig_struct[j - nser], OP_G2_DES, 0u};
        run_seq(1, 1, [&] { k_single(1, (const single_desc*)nullptr, dp, &rc1); });
        run_seq(1, 1, [&] { k_single(1, (const single_desc*)nullptr, ds, &rc2); });
        if (rc1 != 48 || rc2 != 96) return -3;
    }
    std::vector<g1a> pkneg(nv);
    run_seq(1, (unsigned)nv, [&] { k_g1_normalize_lat(nv, apk.data(), pkneg.data(), 1); });
    // signatures: AGG / MASK decoded with the subgroup test (flags), VERIFY structs made affine (flag 1)
    std::vector<g2a> vsig(nv); std::vector<uint8_t> ok_sig(nv, 1), ser(96 * (nser ? nser : 1));
    for (size_t j = 0; j < nser; j++) memcpy(&ser[96 * j], sig96 + 96 * ver[j], 96);
    for (size_t j = 0; j < nser; j++)                                 // item per lane pair: one 2-thread CTA per item
        run_pair([&] { k_g2_decode_pair(1, ser.data() + 96 * j, vsig.data() + j, ok_sig.data() + j, 1); });
    if (nv > nser) run_seq(1, (unsigned)(nv - nser), [&] { k_g2_normalize(nv - nser, vsig_struct.data(), vsig.data() + nser); });
    // H(m): one table entry per distinct 48-byte key, hashed by lane pair, gathered to the requests by index
    std::map<std::array<uint8_t, 48>, uint32_t> seen; std::vector<std::array<uint8_t, 48>> keys; std::vector<uint32_t> idx(nv);
    for (size_t j = 0; j < nv; j++) {
        std::array<uint8_t, 48> key{}; const size_t i = ver[j];
        memcpy(key.data(), msgs + 64 * i, lens[i] > 48 ? 48 : lens[i]);
        auto it = seen.emplace(key, (uint32_t)keys.size());
        if (it.second) keys.push_back(key);
        idx[j] = it.first->second;
    }
    std::vector<uint8_t> kb(48 * keys.size()), tok(keys.size()), ok_hm(nv);
    for (size_t d = 0; d < keys.size(); d++) memcpy(&kb[48 * d], keys[d].data(), 48);
    std::vector<g2a> th(keys.size()), hm(nv);
    for (size_t d = 0; d < keys.size(); d++) run_pair([&] { k_hash_to_g2_pair(1, kb.data() + 48 * d, 48, th.data() + d, tok.data() + d); });
    run_seq(1, (unsigned)nv, [&] { k_broadcast_hm(nv, idx.data(), th.data(), tok.data(), hm.data(), ok_hm.data()); });
    // pairing: lane pair per request, rounds with an identity operand decided by the fix-up
    std::vector<uint8_t> res(nv, 0xee);
    run_pair([&] { k_pairing_verify_split(nv, vsig.data(), pkneg.data(), hm.data(), ok_hm.data(), ok_sig.data(), (const uint8_t*)nullptr, res.data(), (const int*)nullptr); });
    run_seq(1, 1, [&] { k_pairing_fixup(nv, vsig.data(), pkneg.data(), hm.data(), ok_hm.data(), ok_sig.data(), (const uint8_t*)nullptr, res.data(), (const int*)nullptr); });
    for (size_t j = 0; j < nv; j++) results[ver[j]] = res[j];
    return 0;
}

}  // extern "C"
