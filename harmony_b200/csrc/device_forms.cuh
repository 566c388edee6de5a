// harmony_b200/csrc/device_forms.cuh -- kernels of the device forms of the batch verifiers (include/hbls.h:
// hbls_verify_batch_status_device, hbls_verify_headers_device, hbls_aggregate_verify_items_device), and the status kernels their
// host forms share.  Included by hbls.cu only.
//   * message grouping: the inputs of a device form never reach the host, so items whose messages agree in the 48 zero-padded bytes
//     the map reads (hbls.cu hm_key) are found to be one message here; each distinct message is hashed to G2 once and the point
//     gathered back to its items.  The representative of a group is its lowest item index (atomicMin), and the distinct messages
//     are numbered in item order, so nothing depends on thread scheduling.
//   * statuses: the HBLS_VB_* / HBLS_HDR_* codes from the k_pack_flags bits, the only place in the library they are assigned.
#pragma once
#include "../../include/hbls.h"
#include "kernels.cuh"

namespace hb {

#define HB_GRP_EMPTY 0xffffffffu
#define HB_GRP_SCAN 1024            // threads of the compaction kernel (one CTA)

// the bytes the map reads of item i (hash_to_fp: the first min(len, 48), zero-padded)
HB_DEV uint8_t grp_byte(const uint8_t* msgs, uint32_t msg_len, size_t i, int b) {
    return (uint32_t)b < msg_len ? msgs[(size_t)msg_len * i + b] : (uint8_t)0;
}
// table slot hash: SipHash-2-4 of the 48 key bytes under a key drawn per call (hbls.cu), so that messages chosen by a sender cannot
// be made to collide in the table on purpose
HB_DEV uint64_t grp_rotl(uint64_t x, int b) { return (x << b) | (x >> (64 - b)); }
HB_DEV void grp_sipround(uint64_t& v0, uint64_t& v1, uint64_t& v2, uint64_t& v3) {
    v0 += v1; v1 = grp_rotl(v1, 13); v1 ^= v0; v0 = grp_rotl(v0, 32);
    v2 += v3; v3 = grp_rotl(v3, 16); v3 ^= v2;
    v0 += v3; v3 = grp_rotl(v3, 21); v3 ^= v0;
    v2 += v1; v1 = grp_rotl(v1, 17); v1 ^= v2; v2 = grp_rotl(v2, 32);
}
HB_DEV uint64_t grp_hash(const uint8_t* msgs, uint32_t msg_len, size_t i, uint64_t k0, uint64_t k1) {
    uint64_t v0 = k0 ^ 0x736f6d6570736575ull, v1 = k1 ^ 0x646f72616e646f6dull, v2 = k0 ^ 0x6c7967656e657261ull, v3 = k1 ^ 0x7465646279746573ull;
    for (int w = 0; w < 6; w++) {
        uint64_t m = 0;
        for (int b = 0; b < 8; b++) m |= (uint64_t)grp_byte(msgs, msg_len, i, 8 * w + b) << (8 * b);
        v3 ^= m; grp_sipround(v0, v1, v2, v3); grp_sipround(v0, v1, v2, v3); v0 ^= m;
    }
    const uint64_t last = 48ull << 56;
    v3 ^= last; grp_sipround(v0, v1, v2, v3); grp_sipround(v0, v1, v2, v3); v0 ^= last;
    v2 ^= 0xff;
    for (int r = 0; r < 4; r++) grp_sipround(v0, v1, v2, v3);
    return v0 ^ v1 ^ v2 ^ v3;
}
HB_DEV bool grp_same(const uint8_t* msgs, uint32_t msg_len, size_t i, size_t j) {
    for (int b = 0; b < 48; b++) if (grp_byte(msgs, msg_len, i, b) != grp_byte(msgs, msg_len, j, b)) return false;
    return true;
}

// open addressing over mask + 1 >= 2k slots (both arrays HB_GRP_EMPTY beforehand): item i claims the first slot of its probe
// sequence that is empty or holds its key, and lowers that slot's representative to i.  A claimed slot is never released, so
// every item of one key stops at the same slot.  (k0, k1): the call's hash key (slots, not results, depend on it).
__global__ void k_group_insert(size_t k, const uint8_t* msgs, uint32_t msg_len, uint32_t mask, uint64_t k0, uint64_t k1, uint32_t* slot_item,
                               uint32_t* slot_rep, uint32_t* item_slot) {
  for (size_t i = HB_TID; i < k; i += HB_STRIDE) {
    uint32_t s = (uint32_t)grp_hash(msgs, msg_len, i, k0, k1) & mask;
    for (;;) {
        const uint32_t prev = atomicCAS(&slot_item[s], HB_GRP_EMPTY, (uint32_t)i);
        if (prev == HB_GRP_EMPTY || grp_same(msgs, msg_len, prev, i)) { atomicMin(&slot_rep[s], (uint32_t)i); item_slot[i] = s; break; }
        s = (s + 1) & mask;
    }
  }
}

// one CTA: representatives (items whose slot names them) numbered in item order by a scan, their 48 key bytes compacted into
// keys[0..d), grp[i] = the number of item i's message, *count = d.  Any CTA size (contiguous chunks per thread).
__global__ void __launch_bounds__(HB_GRP_SCAN) k_group_compact(size_t k, const uint8_t* msgs, uint32_t msg_len, const uint32_t* slot_rep,
                                                              const uint32_t* item_slot, uint32_t* pos, uint32_t* grp, uint8_t* keys, unsigned* count) {
    __shared__ uint32_t part[HB_GRP_SCAN];
    const size_t T = blockDim.x, t = threadIdx.x, chunk = (k + T - 1) / T;
    const size_t i0 = t * chunk < k ? t * chunk : k, i1 = i0 + chunk < k ? i0 + chunk : k;
    uint32_t c = 0;
    for (size_t i = i0; i < i1; i++) c += slot_rep[item_slot[i]] == (uint32_t)i;
    part[t] = c;
    __syncthreads();
    if (t == 0) {
        uint32_t run = 0;
        for (size_t u = 0; u < T; u++) { const uint32_t v = part[u]; part[u] = run; run += v; }
        *count = run;
    }
    __syncthreads();
    uint32_t run = part[t];
    for (size_t i = i0; i < i1; i++) {
        if (slot_rep[item_slot[i]] != (uint32_t)i) continue;
        pos[i] = run;
        for (int b = 0; b < 48; b++) keys[(size_t)48 * run + b] = grp_byte(msgs, msg_len, i, b);
        run++;
    }
    __syncthreads();                                     // pos[] of every representative is written
    for (size_t i = i0; i < i1; i++) grp[i] = pos[slot_rep[item_slot[i]]];
}

// ---- hash-to-G2 of the d = *count distinct keys (48 bytes each).  d is known on the device only, so every form is launched and
// runs only in its range of d: warp per message for d <= coop_hi, lane pair per message for coop_hi < d <= pair_hi, and the
// thread-per-item map (then hbls.cu's cofactor / affine kernels over all k slots) for d > pair_hi.  The per-item bodies are those of
// k_hash_to_g2_coop, k_hash_to_g2_pair and k_hash_sw (kernels.cuh).
__global__ void __launch_bounds__(32) k_hash_keys_coop(const unsigned* count, unsigned long long coop_hi, const uint8_t* keys, g2a* out,
                                                       uint8_t* ok, int force_fallback) {
    const size_t n = *count;
    if (n > coop_hi) return;
    __shared__ uint32_t slots[VM_SMEM_WORDS];
    const int lane = threadIdx.x & 31;
    vm_load_consts(slots);
    for (size_t i = blockIdx.x; i < n; i += gridDim.x) HB_HASH_ITEM_WARP(i, keys, 48, out, ok, slots, lane, force_fallback)
}
__global__ void k_hash_keys_pair(const unsigned* count, unsigned long long coop_hi, unsigned long long pair_hi, const uint8_t* keys, g2a* out,
                                 uint8_t* ok) {
    const size_t n = *count, i = HB_TID >> 1;
    if (n <= coop_hi || n > pair_hi || i >= n) return;
    HB_HASH_ITEM_PAIR(i, keys, 48, out, ok)
}
// writes all k slots: the map for i < d when d > pair_hi, else (and beyond d) the identity with ok = 0, so that the cofactor and
// affine kernels that follow over k slots leave nothing the other forms have to undo
__global__ void __launch_bounds__(64, HB_SW_MINBLOCKS) k_hash_keys_sw(size_t k, const unsigned* count, unsigned long long pair_hi,
                                                                      const uint8_t* keys, g2a* pts, uint8_t* ok) {
    const size_t d = *count, n = d > pair_hi ? d : 0;
    for (size_t i0 = HB_TID; i0 < k; i0 += (size_t)HB_BATCH_K * HB_STRIDE) hash_sw_items(i0, n, k, keys, 48, pts, ok);
}

// ---- statuses from the k_pack_flags bits (bit0 signature decoded, bit2 key decoded) and the verdicts, for the host and device forms
// alike, in the order the reference meets the errors.
// hbls_verify_batch_status: key decode first (BytesToBLSPublicKey, consensus/view_change_msg.go:159), then signature decode
// (Sign.Deserialize, :168-179), then VerifyHash
__global__ void k_status_triples(size_t k, const uint8_t* flags, const uint8_t* results, uint8_t* status) {
    const size_t j = HB_TID; if (j >= k) return;
    const uint8_t f = flags[j];
    status[j] = !(f & 4) ? HBLS_VB_BAD_KEY_ENCODING : !(f & 1) ? HBLS_VB_BAD_SIG_ENCODING : results[j] == 1 ? HBLS_VB_OK : HBLS_VB_BAD_SIG;
}
HB_DEV uint32_t grp_popc8(uint32_t v) { v = v - ((v >> 1) & 0x55u); v = (v & 0x33u) + ((v >> 2) & 0x33u); return (v + (v >> 4)) & 0x0fu; }
// hbls_verify_headers (engine.go:630-640): signature decode (DecodeSigBitmap), then the quorum over the committee's nslots slots
// (IsQuorumAchievedByMask; padding bits of the last byte never count; quorum 0 skips the gate), then VerifyHash
__global__ void k_status_headers(size_t n, size_t nslots, const uint8_t* bitmaps, size_t blen, size_t quorum, const uint8_t* flags,
                                 const uint8_t* results, uint8_t* status) {
    const size_t j = HB_TID; if (j >= n) return;
    uint8_t st;
    if (!(flags[j] & 1)) st = HBLS_HDR_BAD_ENCODING;
    else {
        size_t set = 0;
        if (quorum) {
            const uint8_t* bm = bitmaps + j * blen;
            for (size_t b = 0; b < (nslots >> 3); b++) set += grp_popc8(bm[b]);
            if (nslots & 7) set += grp_popc8(bm[nslots >> 3] & ((1u << (nslots & 7)) - 1u));
        }
        st = quorum && set < quorum ? HBLS_HDR_NO_QUORUM : results[j] ? HBLS_HDR_OK : HBLS_HDR_BAD_SIG;
    }
    status[j] = st;
}

}  // namespace hb
