// harmony_b200/csrc/kernels.cuh -- __global__ entry points of the BLS hot path (thread-per-item throughput kernels).
//
// Data layout in HBM (all arrays of structs, Montgomery limbs, little-endian u32):
//   g1a  96 B  affine G1   (committee table rows, -apk per round)
//   g2a 192 B  affine G2   (decoded signatures, H(m))
//   g1  144 B / g2 288 B   Jacobian partial sums
//   fp12 576 B             Miller-loop outputs, 2 per verification round
// The arithmetic is integer-pipe bound (~375 MAC32 per byte touched, SURVEY 8d): HBM is idle by design; the
// launch geometry therefore only aims at filling every SM's 4 schedulers (132 SMs on an H100 SXM) with independent IMAD chains.
#pragma once
#include "pairing.cuh"
#include "vm.cuh"

namespace hb {

#ifndef HB_MINBLOCKS
#define HB_MINBLOCKS 4      // 64-thread CTAs: 4 => up to 255 regs/thread, 8 => 128
#endif
#define HB_TID ((size_t)blockIdx.x * blockDim.x + threadIdx.x)
#define HB_STRIDE ((size_t)gridDim.x * blockDim.x)      // heavy kernels are persistent grid-stride loops: resident threads are capped
                                                        // so the per-thread working set (~3 KB of Fp12 temporaries) stays in L1/L2

// ---- parity probe: canonical LE operands -> Montgomery -> product -> canonical
__global__ void k_fp_mul(size_t n, const uint8_t* a, const uint8_t* b, uint8_t* out) {
    size_t i = HB_TID; if (i >= n) return;
    fp x, y, v;
    load_words(v.l, a + 48 * i, 12); fp_from_int(x, v);
    load_words(v.l, b + 48 * i, 12); fp_from_int(y, v);
    fp_mul(x, x, y); fp_to_int(v, x); store_words(out + 48 * i, v.l, 12);
}

// ---- decode (R2/R3 of SURVEY 8a): 48/96 B -> affine point (+ optional negation), ok flag
__global__ void k_g1_decode(size_t n, const uint8_t* in, g1a* out, uint8_t* ok, int check_order, int negate) {
    size_t i = HB_TID; if (i >= n) return;
    g1 p; bool good = g1_deserialize(p, in + 48 * i, check_order != 0);
    g1a a;
    if (!good || pt_is_inf(p)) { fp_zero(a.x); fp_zero(a.y); }
    else { a.x = p.x; a.y = p.y; if (negate) fp_neg(a.y, a.y); }      // deserialize returns z == 1
    out[i] = a; ok[i] = good ? 1 : 0;
}
// triples (hbls_verify_batch): the key feeds the same pipeline as a mask aggregate, so it is kept Jacobian (z = 1; identity on failure)
__global__ void k_g1_decode_jac(size_t n, const uint8_t* in, g1* out, uint8_t* ok, int check_order) {
  for (size_t i = HB_TID; i < n; i += HB_STRIDE) {
    g1 p; bool good = g1_deserialize(p, in + 48 * i, check_order != 0);
    if (!good) pt_set_inf(p);
    out[i] = p; ok[i] = good ? 1 : 0;
  }
}
#ifndef HB_DEC_MINBLOCKS
#define HB_DEC_MINBLOCKS 8          // <= 128 registers: 512 resident threads per SM = exactly 4 waves of the benchmark's batch (bench.py --rounds)
#endif
__global__ void __launch_bounds__(64, HB_DEC_MINBLOCKS) k_g2_decode(size_t n, const uint8_t* in, g2a* out, uint8_t* ok, int check_order) {
  for (size_t i = HB_TID; i < n; i += HB_STRIDE) {
    g2 p; bool good = g2_deserialize(p, in + 96 * i, check_order != 0);
    g2a a;
    if (!good || pt_is_inf(p)) { fp2_zero(a.x); fp2_zero(a.y); }
    else { a.x = p.x; a.y = p.y; }
    out[i] = a; ok[i] = good ? 1 : 0;
  }
}

// subgroup test of already-decoded affine points, one per thread; a point outside the subgroup loses its ok flag and is zeroed.  The
// split decode stage (hbls.cu "decode_split") runs k_g2_subgroup_pair instead; this form is the reference tests compare it with.
__global__ void __launch_bounds__(64, HB_DEC_MINBLOCKS) k_g2_subgroup(size_t n, g2a* pts, uint8_t* ok) {
  for (size_t i = HB_TID; i < n; i += HB_STRIDE) {
    if (!ok[i]) continue;
    const g2a a = pts[i];
    if (aff_is_inf(a)) continue;
    g2 q; q.x = a.x; q.y = a.y; fp2_one(q.z);
    if (!g2_in_subgroup(q)) { g2a z; fp2_zero(z.x); fp2_zero(z.y); pts[i] = z; ok[i] = 0; }
  }
}

// ---- warp shuffle of a whole point
template <class T> HB_DEV void shfl_down_struct(T& dst, const T& src, int off) {
    const uint32_t* s = reinterpret_cast<const uint32_t*>(&src);
    uint32_t* d = reinterpret_cast<uint32_t*>(&dst);
    for (int w = 0; w < (int)(sizeof(T) / 4); w++) d[w] = __shfl_down_sync(0xffffffffu, s[w], off);
}

// ---- Mask.SetMask (R4): one warp per round; lane l sums table rows l, l+32, ... whose bit is set, then a
// 5-level shuffle tree folds the 32 partial sums.  Summation order is free: only Serialize normalises (A.6).
__global__ void k_mask_aggregate(size_t B, size_t n, const g1a* __restrict__ table, const uint8_t* __restrict__ bitmaps, size_t blen, g1* out) {
    size_t warp = HB_TID >> 5; int lane = threadIdx.x & 31;
    if (warp >= B) return;
    const uint8_t* bm = bitmaps + warp * blen;
    g1 acc; pt_set_inf(acc);
    for (size_t i = lane; i < n; i += 32) {
        if (bm[i >> 3] & (1u << (i & 7))) { g1a q = table[i]; pt_add_mixed(acc, acc, q); }
    }
    for (int off = 16; off >= 1; off >>= 1) {
        g1 other; shfl_down_struct(other, acc, off);
        if (lane < off) pt_add(acc, acc, other);
    }
    if (lane == 0) out[warp] = acc;
}
// multi-committee form (crosslinks / multi-shard block seal: internal/chain/engine.go:592-604, node/harmony/node_cross_link.go:69-90):
// every item names its own committee table; one warp per item
struct mask_item { const g1a* table; const uint8_t* bitmap; uint64_t n; };
__global__ void k_mask_aggregate_items(size_t B, const mask_item* __restrict__ items, g1* out) {
    size_t warp = HB_TID >> 5; int lane = threadIdx.x & 31;
    if (warp >= B) return;
    const mask_item it = items[warp];
    g1 acc; pt_set_inf(acc);
    for (size_t i = lane; i < it.n; i += 32) {
        if (it.bitmap[i >> 3] & (1u << (i & 7))) { g1a q = it.table[i]; pt_add_mixed(acc, acc, q); }
    }
    for (int off = 16; off >= 1; off >>= 1) {
        g1 other; shfl_down_struct(other, acc, off);
        if (lane < off) pt_add(acc, acc, other);
    }
    if (lane == 0) out[warp] = acc;
}
// committee set (hbls_aggregate_verify_set_device): the mask_item descriptors built on the device from a uint32 committee index per
// item.  Item j's bitmap starts at the sum of the bitmap bytes of items 0..j-1; an index >= m is a bad index, which occupies no
// bitmap bytes and gets n = 0, no table and no bitmap.  The offsets are an exclusive scan across the whole batch in three launches:
// k_set_tile_sums (one tile of HB_SET_TILE items per CTA, one item per thread), k_set_tile_scan (one CTA over the tile totals),
// k_set_items (each tile's scan again, plus its tile's offset).
#ifndef HB_SET_TILE
#define HB_SET_TILE 256                     // the host emulation shrinks it so that a few dozen items span several tiles
#endif
enum { HB_SET_BAD_INDEX = 48 };             // == HBLS_SET_BAD_INDEX
struct set_entry { const g1a* table; uint64_t n; };
HB_DEV uint64_t set_item_bytes(const uint32_t* __restrict__ index, size_t j, uint32_t m, const set_entry* __restrict__ ents) {
    const uint32_t c = index[j];
    return c < m ? (ents[c].n + 7) >> 3 : 0;
}
// inclusive scan of v over the CTA (any size up to HB_SET_TILE), *total = the CTA's sum; every thread of it calls
HB_DEV uint64_t set_cta_scan(uint64_t v, uint64_t* total) {
    __shared__ uint64_t scan[HB_SET_TILE];
    const unsigned t = threadIdx.x, T = blockDim.x;
    scan[t] = v;
    __syncthreads();
    for (unsigned off = 1; off < T; off <<= 1) {
        const uint64_t u = t >= off ? scan[t - off] : 0;
        __syncthreads();
        scan[t] += u;
        __syncthreads();
    }
    const uint64_t r = scan[t];
    *total = scan[T - 1];
    __syncthreads();                                    // the next call may overwrite scan[]
    return r;
}
// tile_sum[b] = the bitmap bytes of tile b's items
__global__ void __launch_bounds__(HB_SET_TILE) k_set_tile_sums(size_t k, const uint32_t* __restrict__ index, uint32_t m,
                                                              const set_entry* __restrict__ ents, uint64_t* tile_sum) {
    const size_t j = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    uint64_t total;
    set_cta_scan(j < k ? set_item_bytes(index, j, m, ents) : 0, &total);
    if (threadIdx.x == 0) tile_sum[blockIdx.x] = total;
}
// one CTA (any size up to HB_SET_TILE): tile_sum[0..nt) := its exclusive scan, in place
__global__ void __launch_bounds__(HB_SET_TILE) k_set_tile_scan(size_t nt, uint64_t* tile_sum) {
    const unsigned t = threadIdx.x, T = blockDim.x;
    uint64_t carry = 0;
    for (size_t b0 = 0; b0 < nt; b0 += T) {
        const size_t b = b0 + t;
        const uint64_t v = b < nt ? tile_sum[b] : 0;
        uint64_t total;
        const uint64_t incl = set_cta_scan(v, &total);
        if (b < nt) tile_sum[b] = carry + incl - v;
        carry += total;
    }
}
// items[j] = {table, bitmaps + offset, n} of item j's committee, ok_key[j] = its index is < m
__global__ void __launch_bounds__(HB_SET_TILE) k_set_items(size_t k, const uint32_t* __restrict__ index, uint32_t m,
                                                          const set_entry* __restrict__ ents, const uint64_t* __restrict__ tile_off,
                                                          const uint8_t* bitmaps, mask_item* items, uint8_t* ok_key) {
    const size_t j = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    const uint64_t own = j < k ? set_item_bytes(index, j, m, ents) : 0;
    uint64_t total;
    const uint64_t incl = set_cta_scan(own, &total);
    if (j >= k) return;
    const uint32_t c = index[j];
    const bool good = c < m;
    mask_item it{nullptr, nullptr, 0};
    if (good) { it.table = ents[c].table; it.bitmap = bitmaps + tile_off[blockIdx.x] + incl - own; it.n = ents[c].n; }
    items[j] = it; ok_key[j] = good ? 1 : 0;
}
// after the verify tail: a bad index's result is HB_SET_BAD_INDEX, whatever the decode and pairing verdicts wrote
__global__ void k_set_bad_index(size_t k, const uint8_t* __restrict__ ok_key, uint8_t* results) {
    const size_t j = HB_TID; if (j >= k) return;
    if (!ok_key[j]) results[j] = HB_SET_BAD_INDEX;
}
// large-batch form: one thread per round.  Quorum bitmaps are dense (167..250 of 250 set), so the thread sums whichever
// side is SMALLER -- the set bits, or the unset bits subtracted from the committee total (computed once at
// hbls_committee_create) -- from a compacted index list: ~44 point additions per round instead of ~206, and the
// loop trip counts of the 32 lanes are short and similar.  Group arithmetic only; Serialize normalises (SURVEY A.6).
#ifndef HB_MASK_LIST
#define HB_MASK_LIST 512                    // the host emulation shrinks both to reach every branch with committees of a few dozen keys
#endif
// The 32 lanes of a warp run as long as the lane with the most additions (167 / 200 / 250 signers of 250 = 83 / 50 / 0 additions,
// so unsorted rounds keep the multiplier busy with lanes that have finished).  `order` (nullable) = the rounds sorted by the number of additions they
// need (counting sort on the device: k_mask_count -> k_mask_scan -> k_mask_scatter), so that neighbouring lanes get equal trip counts.
#ifndef HB_MASK_BINS
#define HB_MASK_BINS 1024
#endif
__global__ void k_mask_count(size_t B, size_t n, const uint8_t* __restrict__ bitmaps, size_t blen, uint16_t* cost, unsigned* hist) {
    const size_t j = HB_TID; if (j >= B) return;
    const uint8_t* bm = bitmaps + j * blen;
    uint32_t k = 0;
    for (size_t i = 0; i < n; i++) k += (bm[i >> 3] >> (i & 7)) & 1u;
    uint32_t c = (2 * (size_t)k > n) ? (uint32_t)(n - k) : k;            // the side k_mask_aggregate_serial will sum
    if (c >= HB_MASK_BINS) c = HB_MASK_BINS - 1;
    cost[j] = (uint16_t)c; atomicAdd(&hist[c], 1u);
}
__global__ void k_mask_scan(unsigned* hist) {                             // exclusive prefix sum of the bins, one thread (1 024 adds)
    if (HB_TID != 0) return;
    unsigned acc = 0;
    for (int i = 0; i < HB_MASK_BINS; i++) { const unsigned h = hist[i]; hist[i] = acc; acc += h; }
}
__global__ void k_mask_scatter(size_t B, const uint16_t* cost, unsigned* hist, uint32_t* order) {
    const size_t j = HB_TID; if (j >= B) return;
    order[atomicAdd(&hist[cost[j]], 1u)] = (uint32_t)j;
}
__global__ void k_mask_aggregate_serial(size_t B, size_t n, const g1a* __restrict__ table, const g1* __restrict__ total,
                                        const uint8_t* __restrict__ bitmaps, size_t blen, g1* out, const uint32_t* __restrict__ order = nullptr) {
  for (size_t jt = HB_TID; jt < B; jt += HB_STRIDE) {
    const size_t j = order ? order[jt] : jt;
    const uint8_t* bm = bitmaps + j * blen;
    uint32_t k = 0;
    for (size_t i = 0; i < n; i++) k += (bm[i >> 3] >> (i & 7)) & 1u;
    const bool fits = n <= 65536;                                                             // idx[] holds 16-bit row numbers
    const bool comp = fits && (2 * (size_t)k > n) && (n - k) <= HB_MASK_LIST && total != nullptr;     // sum the unset side
    g1 acc; pt_set_inf(acc);
    if (comp || (fits && k <= HB_MASK_LIST)) {
        uint16_t idx[HB_MASK_LIST]; uint32_t cnt = 0;
        const uint32_t want = comp ? 0u : 1u;
        for (size_t i = 0; i < n; i++) if (((bm[i >> 3] >> (i & 7)) & 1u) == want) idx[cnt++] = (uint16_t)i;
        for (uint32_t t = 0; t < cnt; t++) { g1a q = table[idx[t]]; pt_add_mixed(acc, acc, q); }
        if (comp) { g1 tot = *total; pt_neg(acc, acc); pt_add(acc, tot, acc); }
    } else {
        for (size_t i = 0; i < n; i++) if ((bm[i >> 3] >> (i & 7)) & 1u) { g1a q = table[i]; pt_add_mixed(acc, acc, q); }
    }
    out[j] = acc;
  }
}
// committee total (sum of all table rows), single CTA
__global__ void __launch_bounds__(128) k_g1_sum(size_t n, const g1a* in, g1* out) {
    __shared__ g1 sm[128];
    g1 acc; pt_set_inf(acc);
    for (size_t i = threadIdx.x; i < n; i += 128) { g1a q = in[i]; pt_add_mixed(acc, acc, q); }
    sm[threadIdx.x] = acc;
    __syncthreads();
    for (int off = 64; off >= 1; off >>= 1) {
        if ((int)threadIdx.x < off) { g1 o = sm[threadIdx.x + off]; pt_add(acc, acc, o); sm[threadIdx.x] = acc; }
        __syncthreads();
    }
    if (threadIdx.x == 0) out[0] = acc;
}
__global__ void k_g1_normalize(size_t n, const g1* in, g1a* out, int negate, const int* run_if) {
    if (run_if && !*run_if) return;          // deferred form: only needed when the batched check sends rounds to the exact pass
    size_t i = HB_TID; if (i >= n) return;
    g1 p = in[i]; g1a a; pt_to_aff(a, p);
    if (negate) fp_neg(a.y, a.y);
    out[i] = a;
}
// latency path: affine -apk with the binary-GCD inverse
__global__ void k_g1_normalize_lat(size_t n, const g1* in, g1a* out, int negate) {
    size_t i = HB_TID; if (i >= n) return;
    g1 p = in[i]; g1a a;
    if (pt_is_inf(p)) { fp_zero(a.x); fp_zero(a.y); }
    else {
        fp zi, zi2; fp_inv_gcd(zi, p.z); fp_sqr(zi2, zi);
        fp_mul(a.x, p.x, zi2); fp_mul(zi2, zi2, zi); fp_mul(a.y, p.y, zi2);
        if (negate) fp_neg(a.y, a.y);
    }
    out[i] = a;
}
__global__ void k_g2_normalize(size_t n, const g2* in, g2a* out) {
    size_t i = HB_TID; if (i >= n) return;
    g2 p = in[i]; g2a a; pt_to_aff(a, p);
    out[i] = a;
}
__global__ void k_g1_serialize(size_t n, const g1* in, uint8_t* out) {
    size_t i = HB_TID; if (i >= n) return;
    g1 p = in[i]; g1_serialize(out + 48 * i, p);
}
__global__ void k_g2_serialize(size_t n, const g2* in, uint8_t* out) {
    size_t i = HB_TID; if (i >= n) return;
    g2 p = in[i]; g2_serialize(out + 96 * i, p);
}

// ---- AggregateSig (R5): single-CTA strided sum + shared-memory tree; out = 1 Jacobian point
#define HB_SUM_THREADS 128
__global__ void __launch_bounds__(HB_SUM_THREADS) k_g2_sum(size_t n, const g2a* in, g2* out) {
    __shared__ g2 sm[HB_SUM_THREADS];
    g2 acc; pt_set_inf(acc);
    for (size_t i = threadIdx.x; i < n; i += HB_SUM_THREADS) { g2a q = in[i]; pt_add_mixed(acc, acc, q); }
    sm[threadIdx.x] = acc;
    __syncthreads();
    for (int off = HB_SUM_THREADS / 2; off >= 1; off >>= 1) {
        if ((int)threadIdx.x < off) { g2 o = sm[threadIdx.x + off]; pt_add(acc, acc, o); sm[threadIdx.x] = acc; }
        __syncthreads();
    }
    if (threadIdx.x == 0) out[0] = acc;
}

// ---- B AggregateSig calls in one launch sequence (hbls_aggregate_sigs_batch): set j = decoded rows offsets[j] .. offsets[j+1]-1.
// Every set is cut into chunks of at most HB_AGG_CHUNK rows that never cross a set boundary; a warp sums a chunk (k_g2_segsum_chunks),
// then a warp per set adds its chunk partials (k_g2_segsum_fold).  Summation order is free: only Serialize normalises (A.6).
#ifndef HB_AGG_CHUNK
#define HB_AGG_CHUNK 128        // 4 rows per lane: the shuffle tree's 5 Jacobian additions then cost about what the lane's 4 mixed additions
#endif                          // do, and a 1 000-signature set still spreads over 8 warps (the host emulation shrinks it to a few rows)
#define HB_AGG_PLAN_THREADS 256
#define HB_AGG_NO_CHUNK 0xffffffffu                                    // chunk-table slot of a set that is summed by its fold warp
enum { HB_AGG_OK = 32, HB_AGG_BAD_SIG_ENCODING = 33, HB_AGG_BAD_RANGE = 34 };       // == HBLS_AGG_*
HB_DEV size_t agg_chunks(size_t len) { return (len + HB_AGG_CHUNK - 1) / HB_AGG_CHUNK; }
// the 32 lanes' Jacobian sums into lane 0 (5-level shuffle tree); *bad := some lane's flag
HB_DEV void warp_fold_g2(g2& acc, bool& bad) {
    const int lane = threadIdx.x & 31;
    for (int off = 16; off >= 1; off >>= 1) {
        g2 other; shfl_down_struct(other, acc, off);
        if (lane < off) pt_add(acc, acc, other);
    }
    bad = __ballot_sync(0xffffffffu, bad) != 0;
}
// rows b .. e-1 summed by one warp (lane l adds rows b + l, b + l + 32, ...); bad := a row of them did not decode
HB_DEV void warp_sum_rows(const g2a* __restrict__ pts, const uint8_t* __restrict__ ok, size_t b, size_t e, g2& acc, bool& bad) {
    pt_set_inf(acc); bad = false;
    for (size_t i = b + (threadIdx.x & 31); i < e; i += 32) {
        if (ok[i]) { g2a q = pts[i]; pt_add_mixed(acc, acc, q); }
        else bad = true;
    }
    warp_fold_g2(acc, bad);
}
// chunk table (one CTA, any block size): first[j] = exclusive scan of the sets' chunk counts (first[B] = total), chunk_set[c] = the
// set of chunk c for the chunks below cap; status[j] = HB_AGG_BAD_RANGE for a set whose range is reversed or ends past row n, else 0.
// Valid sets can overlap when a reversed one lies between them, so the total can exceed cap (the host's bound for disjoint sets,
// ceil(n / C) + B): a set whose chunks do not all fit marks its slots below cap HB_AGG_NO_CHUNK and is summed by its fold warp.
__global__ void __launch_bounds__(HB_AGG_PLAN_THREADS) k_g2_segsum_plan(size_t B, size_t n, const uint64_t* __restrict__ offsets, size_t cap,
                                                                       uint64_t* first, uint32_t* chunk_set, uint8_t* status) {
    __shared__ uint64_t scan[HB_AGG_PLAN_THREADS];
    const unsigned t = threadIdx.x, T = blockDim.x;
    uint64_t carry = 0;
    for (size_t j0 = 0; j0 < B; j0 += T) {
        const size_t j = j0 + t;
        bool good = false; uint64_t cnt = 0;
        if (j < B) {
            const uint64_t lo = offsets[j], hi = offsets[j + 1];
            good = lo <= hi && hi <= n;
            cnt = good ? agg_chunks(hi - lo) : 0;
        }
        scan[t] = cnt;
        __syncthreads();
        for (unsigned off = 1; off < T; off <<= 1) {                  // inclusive scan of the tile
            const uint64_t v = t >= off ? scan[t - off] : 0;
            __syncthreads();
            scan[t] += v;
            __syncthreads();
        }
        const uint64_t f = carry + scan[t] - cnt;
        if (j < B) {
            first[j] = f; status[j] = good ? 0 : HB_AGG_BAD_RANGE;
            const uint32_t mark = f + cnt <= cap ? (uint32_t)j : HB_AGG_NO_CHUNK;
            for (uint64_t c = f; c < f + cnt && c < cap; c++) chunk_set[c] = mark;
        }
        carry += scan[T - 1];
        __syncthreads();                                               // every thread has read the tile total
    }
    if (t == 0) first[B] = carry;
}
// one warp per chunk-table slot (grid: cap warps; slots at or past the total exit): part[c] = the chunk's sum, part_bad[c] = a row of
// it did not decode
__global__ void __launch_bounds__(128, 4) k_g2_segsum_chunks(size_t B, const uint64_t* __restrict__ offsets, const uint64_t* __restrict__ first,
                                                         const uint32_t* __restrict__ chunk_set, size_t cap, const g2a* __restrict__ pts,
                                                         const uint8_t* __restrict__ ok, g2* part, uint8_t* part_bad) {
    const size_t c = HB_TID >> 5;
    if (c >= cap || c >= first[B]) return;
    const uint32_t j = chunk_set[c];
    if (j == HB_AGG_NO_CHUNK) return;
    const uint64_t b = offsets[j] + (c - first[j]) * HB_AGG_CHUNK, hi = offsets[j + 1];
    g2* dst = part + c; uint8_t* dst_bad = part_bad + c;
    g2 acc; bool bad;
    warp_sum_rows(pts, ok, b, b + HB_AGG_CHUNK < hi ? b + HB_AGG_CHUNK : hi, acc, bad);
    if ((threadIdx.x & 31) == 0) { *dst = acc; *dst_bad = bad ? 1 : 0; }
}
// one warp per set: the sum of its chunk partials (or of its rows, for a set without table slots) into sum[j], the status into status[j];
// a set with a bad range or an undecodable row gets the identity
__global__ void __launch_bounds__(128) k_g2_segsum_fold(size_t B, const uint64_t* __restrict__ offsets, const uint64_t* __restrict__ first,
                                                       size_t cap, const g2a* __restrict__ pts, const uint8_t* __restrict__ ok,
                                                       const g2* __restrict__ part, const uint8_t* __restrict__ part_bad, g2* sum, uint8_t* status) {
    const size_t j = HB_TID >> 5;
    if (j >= B) return;
    const int lane = threadIdx.x & 31;
    g2 acc; pt_set_inf(acc); bool bad = false;
    if (status[j] == HB_AGG_BAD_RANGE) { if (lane == 0) sum[j] = acc; return; }
    const uint64_t lo = offsets[j], hi = offsets[j + 1], f = first[j], cnt = agg_chunks(hi - lo);
    if (f + cnt > cap) warp_sum_rows(pts, ok, lo, hi, acc, bad);
    else {
        for (uint64_t c = f + lane; c < f + cnt; c += 32) { g2 q = part[c]; pt_add(acc, acc, q); bad |= part_bad[c] != 0; }
        warp_fold_g2(acc, bad);
    }
    if (lane == 0) {
        if (bad) pt_set_inf(acc);
        sum[j] = acc; status[j] = bad ? HB_AGG_BAD_SIG_ENCODING : HB_AGG_OK;
    }
}

// ---- leader's vote queue into the ballot box (hbls_ballot_box_submit_votes; consensus/leader.go:110-345, quorum.go:164-196,354-377).
// k_ballot_admit applies the ballot rules in arrival order: vote j's fate depends on the verdicts of the votes before it, so one CTA
// walks the queue with the box's collected bitmap in shared memory.  Votes are staged into shared memory a chunk at a time (one
// coalesced load per chunk); per vote, each thread tests its bytes of the bitmap against the box and the CTA meets at ONE barrier.
// The "some signer is already collected" flag is a stamp (j + 1) in a slot that alternates with j, so it never needs clearing: a
// thread that writes vote j + 1's slot has passed vote j's barrier, hence every thread has left vote j - 1, the slot's last reader.
// Statuses follow the order in which onPrepare / onCommit meet the errors: already collected (before the signature is looked at),
// signature does not decode, VerifyHash false, accepted.  Padding bits of the last byte (slots >= n) are ignored.  Any block size
// (the host emulation runs one thread).
#define HB_BALLOT_THREADS 128
#ifndef HB_BALLOT_MAX_BYTES
#define HB_BALLOT_MAX_BYTES 2048            // collected bitmap held in shared memory: committees of up to 16 384 slots
#endif
#ifndef HB_BALLOT_STAGE
#define HB_BALLOT_STAGE 8192                // staged vote bitmaps per chunk (bytes; the host emulation shrinks both to test chunking)
#endif
static_assert(HB_BALLOT_STAGE >= HB_BALLOT_MAX_BYTES, "a chunk holds at least one vote");
#define HB_BALLOT_CHUNK 1024                // votes per chunk at most
enum { HB_BALLOT_ACCEPTED = 16, HB_BALLOT_COLLECTED = 17, HB_BALLOT_BAD_SIG_ENCODING = 18, HB_BALLOT_BAD_SIG = 19 };      // == HBLS_BALLOT_*
__global__ void __launch_bounds__(HB_BALLOT_THREADS) k_ballot_admit(size_t k, size_t n, size_t blen, const uint8_t* __restrict__ bitmaps,
                                                                   const uint8_t* __restrict__ verified, const uint8_t* __restrict__ ok_sig,
                                                                   const uint8_t* __restrict__ collected_in, uint8_t* collected_out,
                                                                   uint8_t* status, uint8_t* accept) {
    __shared__ uint8_t box[HB_BALLOT_MAX_BYTES];
    __shared__ uint8_t stage[HB_BALLOT_STAGE];
    __shared__ uint8_t verdict[HB_BALLOT_CHUNK];        // bit 0: signature decoded, bit 1: VerifyHash true
    __shared__ uint32_t hit[2];
    const uint8_t last = (n & 7) ? (uint8_t)((1u << (n & 7)) - 1u) : (uint8_t)0xff;
    for (size_t i = threadIdx.x; i < blen; i += blockDim.x) box[i] = collected_in[i] & (i + 1 == blen ? last : (uint8_t)0xff);
    if (threadIdx.x == 0) { hit[0] = 0; hit[1] = 0; }
    size_t per = HB_BALLOT_STAGE / (blen ? blen : 1);
    if (per > HB_BALLOT_CHUNK) per = HB_BALLOT_CHUNK;
    for (size_t j0 = 0; j0 < k; j0 += per) {
        const size_t m = k - j0 < per ? k - j0 : per;
        __syncthreads();                                 // the previous chunk's scan is over
        for (size_t i = threadIdx.x; i < m * blen; i += blockDim.x) stage[i] = bitmaps[j0 * blen + i];
        for (size_t i = threadIdx.x; i < m; i += blockDim.x) verdict[i] = (uint8_t)((ok_sig[j0 + i] ? 1 : 0) | (verified[j0 + i] ? 2 : 0));
        __syncthreads();
        for (size_t t = 0; t < m; t++) {
            const size_t j = j0 + t;
            const uint8_t* bm = stage + t * blen;
            for (size_t i = threadIdx.x; i < blen; i += blockDim.x)
                if (bm[i] & box[i]) hit[j & 1] = (uint32_t)(j + 1);
            __syncthreads();
            const bool dup = hit[j & 1] == (uint32_t)(j + 1);
            const uint8_t vd = verdict[t];
            const bool ok = !dup && vd == 3;
            if (ok)                                      // each thread ORs the bytes it tests: no barrier needed before the next vote
                for (size_t i = threadIdx.x; i < blen; i += blockDim.x) box[i] |= bm[i] & (i + 1 == blen ? last : (uint8_t)0xff);
            if (threadIdx.x == 0) {
                status[j] = dup ? HB_BALLOT_COLLECTED : !(vd & 1) ? HB_BALLOT_BAD_SIG_ENCODING : !(vd & 2) ? HB_BALLOT_BAD_SIG : HB_BALLOT_ACCEPTED;
                accept[j] = ok ? 1 : 0;
            }
        }
    }
    for (size_t i = threadIdx.x; i < blen; i += blockDim.x) collected_out[i] = box[i];
}
// the accepted votes' decoded signatures added into the box's running sum (single CTA; block size a power of two, any including 1)
__global__ void __launch_bounds__(HB_SUM_THREADS) k_ballot_fold(size_t k, const g2a* __restrict__ sig, const uint8_t* __restrict__ accept, g2* sum) {
    __shared__ g2 sm[HB_SUM_THREADS];
    g2 acc; pt_set_inf(acc);
    for (size_t j = threadIdx.x; j < k; j += blockDim.x) if (accept[j]) { g2a q = sig[j]; pt_add_mixed(acc, acc, q); }
    sm[threadIdx.x] = acc;
    __syncthreads();
    for (unsigned off = blockDim.x / 2; off >= 1; off >>= 1) {
        if (threadIdx.x < off) { g2 o = sm[threadIdx.x + off]; pt_add(acc, acc, o); sm[threadIdx.x] = acc; }
        __syncthreads();
    }
    if (threadIdx.x == 0) { g2 s = *sum; pt_add(s, s, acc); *sum = s; }
}

// ---- message -> G2 (hash part of R6/R7), affine output
// HB_BATCH_INV: a persistent thread shares ONE inversion among HB_BATCH_K of its items (Montgomery's trick) -- both inversions of
// hash-to-G2 and the affine conversion of the coefficient-scaling stage: one inversion costs ~400 products, the trick 3 per item.
#ifndef HB_BATCH_INV
#define HB_BATCH_INV 1
#endif
#ifndef HB_BATCH_K
#define HB_BATCH_K 8
#endif
__global__ void k_hash_to_g2(size_t n, const uint8_t* msgs, uint32_t msg_len, g2a* out, uint8_t* ok) {
#if HB_BATCH_INV
  for (size_t i0 = HB_TID; i0 < n; i0 += (size_t)HB_BATCH_K * HB_STRIDE) {
    g2 h[HB_BATCH_K]; fp2 z[HB_BATCH_K], t[HB_BATCH_K], u[HB_BATCH_K], ct[HB_BATCH_K]; bool skip[HB_BATCH_K], good[HB_BATCH_K];
    for (int k = 0; k < HB_BATCH_K; k++) {
        const size_t i = i0 + (size_t)k * HB_STRIDE;
        good[k] = false; skip[k] = true;
        if (i >= n) continue;
        fp_zero(t[k].b); hash_to_fp(t[k].a, msgs + (size_t)msg_len * i, msg_len);
        good[k] = sw_map_g2_pre(u[k], ct[k], z[k], t[k]);
        skip[k] = !good[k];
    }
    f_batch_inv<fp2, HB_BATCH_K>(z, skip);                     // the maps' (u c1 t)^-1
    for (int k = 0; k < HB_BATCH_K; k++) {
        if (skip[k]) continue;
        g2 a;
        good[k] = sw_map_g2_post(a, t[k], u[k], ct[k], z[k]);
        if (good[k]) g2_clear_cofactor(h[k], a);
        skip[k] = !good[k] || pt_is_inf(h[k]);
        if (!skip[k]) z[k] = h[k].z;
    }
    f_batch_inv<fp2, HB_BATCH_K>(z, skip);                     // -> affine
    for (int k = 0; k < HB_BATCH_K; k++) {
        const size_t i = i0 + (size_t)k * HB_STRIDE;
        if (i >= n) continue;
        g2a a;
        if (skip[k]) { fp2_zero(a.x); fp2_zero(a.y); } else pt_to_aff_zinv(a, h[k], z[k]);
        out[i] = a; ok[i] = good[k] ? 1 : 0;
    }
  }
#else
  for (size_t i = HB_TID; i < n; i += HB_STRIDE) {
    g2 h; bool good = map_to_g2(h, msgs + (size_t)msg_len * i, msg_len);
    g2a a;
    if (!good) { fp2_zero(a.x); fp2_zero(a.y); } else pt_to_aff(a, h);
    out[i] = a; ok[i] = good ? 1 : 0;
  }
#endif
}

// ---- the same hash in two kernels (large batches, hbls.cu "hash_split"): the Shallue-van de Woestijne map is Fp-only work (square-
// root exponentiation chains, Jacobi symbols, the shared inversion) with a small register and instruction-cache footprint, the
// cofactor clearing is G2 ladders over Fp2.  Separate kernels let the first run with more resident warps and keep each kernel's hot
// code small (the fused kernel stalls on instruction fetch with only 3 warps per scheduler).
#ifndef HB_SW_MINBLOCKS
#define HB_SW_MINBLOCKS 8         // x 64 threads = 512 resident threads per SM (<= 128 registers)
#endif
// thread form, one thread's HB_BATCH_K items i0 + j * HB_STRIDE: the SW maps of the items below n share one inversion; items in
// [n, k) get the identity with ok = 0
HB_DEV void hash_sw_items(size_t i0, size_t n, size_t k, const uint8_t* msgs, uint32_t msg_len, g2a* pts, uint8_t* ok) {
    fp2 z[HB_BATCH_K], t[HB_BATCH_K], u[HB_BATCH_K], ct[HB_BATCH_K]; bool skip[HB_BATCH_K];
    for (int j = 0; j < HB_BATCH_K; j++) {
        const size_t i = i0 + (size_t)j * HB_STRIDE;
        skip[j] = true;
        if (i >= n) continue;
        fp_zero(t[j].b); hash_to_fp(t[j].a, msgs + (size_t)msg_len * i, msg_len);
        skip[j] = !sw_map_g2_pre(u[j], ct[j], z[j], t[j]);
    }
    f_batch_inv<fp2, HB_BATCH_K>(z, skip);
    for (int j = 0; j < HB_BATCH_K; j++) {
        const size_t i = i0 + (size_t)j * HB_STRIDE;
        if (i >= k) continue;
        g2 a; g2a o; fp2_zero(o.x); fp2_zero(o.y);
        const bool good = !skip[j] && sw_map_g2_post(a, t[j], u[j], ct[j], z[j]);
        if (good) { o.x = a.x; o.y = a.y; }
        pts[i] = o; ok[i] = good ? 1 : 0;
    }
}
__global__ void __launch_bounds__(64, HB_SW_MINBLOCKS) k_hash_sw(size_t n, const uint8_t* msgs, uint32_t msg_len, g2a* pts, uint8_t* ok) {
    for (size_t i0 = HB_TID; i0 < n; i0 += (size_t)HB_BATCH_K * HB_STRIDE) hash_sw_items(i0, n, n, msgs, msg_len, pts, ok);
}
// cofactor clearing alone, Jacobian result (no per-thread arrays of pending items: the frame is the group law's own temporaries), and
// the shared-inversion affine conversion as its own small kernel.  hbls.cu runs the cofactor clearing as k_hash_cofactor_z1_pair + _z2_pair; this
// one-thread form is the reference tests compare k_hash_cofactor_pair with.
__global__ void k_hash_cofactor_jac(size_t n, const g2a* pts, const uint8_t* ok, g2* out) {
  for (size_t i = HB_TID; i < n; i += HB_STRIDE) {
    g2 h; pt_set_inf(h);
    if (ok[i]) { g2 a; const g2a p = pts[i]; a.x = p.x; a.y = p.y; fp2_one(a.z); g2_clear_cofactor(h, a); }
    out[i] = h;
  }
}
__global__ void k_g2_normalize_batch(size_t n, const g2* in, g2a* out) {
  for (size_t i0 = HB_TID; i0 < n; i0 += (size_t)HB_BATCH_K * HB_STRIDE) {
    fp2 z[HB_BATCH_K]; bool skip[HB_BATCH_K];
    for (int k = 0; k < HB_BATCH_K; k++) {
        const size_t i = i0 + (size_t)k * HB_STRIDE;
        skip[k] = true;
        if (i >= n) continue;
        z[k] = in[i].z; skip[k] = fp2_is_zero(z[k]);
    }
    f_batch_inv<fp2, HB_BATCH_K>(z, skip);
    for (int k = 0; k < HB_BATCH_K; k++) {
        const size_t i = i0 + (size_t)k * HB_STRIDE;
        if (i >= n) continue;
        g2a a;
        if (skip[k]) { fp2_zero(a.x); fp2_zero(a.y); } else { const g2 h = in[i]; pt_to_aff_zinv(a, h, z[k]); }
        out[i] = a;
    }
  }
}
__global__ void k_hash_cofactor(size_t n, g2a* pts, const uint8_t* ok) {
  for (size_t i0 = HB_TID; i0 < n; i0 += (size_t)HB_BATCH_K * HB_STRIDE) {
    g2 h[HB_BATCH_K]; fp2 z[HB_BATCH_K]; bool skip[HB_BATCH_K];
    for (int k = 0; k < HB_BATCH_K; k++) {
        const size_t i = i0 + (size_t)k * HB_STRIDE;
        skip[k] = true;
        if (i >= n || !ok[i]) continue;
        g2 a; const g2a p = pts[i]; a.x = p.x; a.y = p.y; fp2_one(a.z);
        g2_clear_cofactor(h[k], a);
        skip[k] = pt_is_inf(h[k]);
        if (!skip[k]) z[k] = h[k].z;
    }
    f_batch_inv<fp2, HB_BATCH_K>(z, skip);
    for (int k = 0; k < HB_BATCH_K; k++) {
        const size_t i = i0 + (size_t)k * HB_STRIDE;
        if (i >= n) continue;
        g2a a;
        if (skip[k]) { fp2_zero(a.x); fp2_zero(a.y); } else pt_to_aff_zinv(a, h[k], z[k]);
        pts[i] = a;
    }
  }
}

// ---- lane-pair forms of decode / hash for small batches (latency path, hbls.cu: B <= coop_max): one item per LANE PAIR.  The Fp-only
// chains (square roots, Jacobi symbols, the SW map) run redundantly on both lanes; the long G2 ladders -- subgroup test, cofactor
// clearing -- run on the split carrier (an Fp2 product costs one product-time per lane instead of three), inversions by binary GCD.
__global__ void k_g2_decode_pair(size_t n, const uint8_t* in, g2a* out, uint8_t* ok, int check_order) {
    const size_t i = HB_TID >> 1; if (i >= n) return;                    // a pair leaves together
    g2 p; bool good = g2_deserialize(p, in + 96 * i, false);
    if (good && check_order && !pt_is_inf(p)) {
        jac<fp2h> q; fp2h_pack(q.x, p.x); fp2h_pack(q.y, p.y); fp2h_pack(q.z, p.z);
        good = g2_in_subgroup(q);
    }
    if ((threadIdx.x & 1) == 0) {
        g2a a;
        if (!good || pt_is_inf(p)) { fp2_zero(a.x); fp2_zero(a.y); } else { a.x = p.x; a.y = p.y; }
        out[i] = a; ok[i] = good ? 1 : 0;
    }
}
// The per-item bodies of the lane-pair and warp forms of hash-to-G2, shared by the message kernels below and the key kernels of
// device_forms.cuh.  They are macros, not functions: a function boundary, even a forceinline one, changes the stack layout ptxas is
// given, and with it the registers and spills of these latency-path kernels.
// The lane-pair tail: cofactor clearing of the mapped point a on the split carrier, binary-GCD inversion, affine result into res
// (left as it is -- zero -- for the identity).
#define HB_HASH_TAIL_PAIR(res, a) {                                                                                                   \
        jac<fp2h> A, H; fp2h_pack(A.x, a.x); fp2h_pack(A.y, a.y); fp2h_pack(A.z, a.z);                                              \
        g2_clear_cofactor(H, A);                                                                                                      \
        if (!pt_is_inf(H)) {                                                                                                          \
            fp2h zi, zi2, hx, hy; fp2_inv_gcd(zi, H.z); fp2_sqr(zi2, zi);                                                            \
            fp2_mul(hx, H.x, zi2); fp2_mul(zi2, zi2, zi); fp2_mul(hy, H.y, zi2);                                                     \
            fp2h_unpack(res.x, hx); fp2h_unpack(res.y, hy);                                                                          \
        }                                                                                                                             \
    }
// lane-pair form: message i (msg_len bytes at stride msg_len) on the calling lane pair (both lanes compute the same point: the map
// is Fp-heavy), the even lane writes
#define HB_HASH_ITEM_PAIR(i, msgs, msg_len, out, ok) {                                                                                \
    fp2 t; hash_to_fp(t.a, msgs + (size_t)msg_len * i, msg_len); fp_zero(t.b);                                                       \
    g2 a; bool good = sw_map_g2<true>(a, t);                                                                                          \
    g2a res; fp2_zero(res.x); fp2_zero(res.y);                                                                                        \
    if (good) HB_HASH_TAIL_PAIR(res, a)                                                                                               \
    if ((threadIdx.x & 1) == 0) { out[i] = res; ok[i] = good ? 1 : 0; }                                                              \
}
__global__ void k_hash_to_g2_pair(size_t n, const uint8_t* msgs, uint32_t msg_len, g2a* out, uint8_t* ok) {
    const size_t i = HB_TID >> 1; if (i >= n) return;
    HB_HASH_ITEM_PAIR(i, msgs, msg_len, out, ok)
}
// ---- latency form of hash-to-G2 (vm.cuh): ONE WARP per message.  The Shallue-van de Woestijne map (Fp chains: one inversion, two
// Legendre symbols, the Fp2 square root) runs on every lane alike (warp-uniform: every lane maps the same message); the cofactor
// clearing -- two 63-doubling chains of G2, about half of a lane pair's hash time -- runs as VM step programs with the 3 independent
// products of a doubling level side by side.  Falls back to the complete lane-pair code when the generic formulas degenerate
// (force_fallback: test hook, hbls_set_param "hash_fallback").  Message i on the calling warp, whose VM slots hold the constants
// (vm_load_consts); lane 0 writes.
#define HB_HASH_ITEM_WARP(i, msgs, msg_len, out, ok, slots, lane, force_fallback) {                                                  \
        fp2 t; hash_to_fp(t.a, msgs + (size_t)msg_len * i, msg_len); fp_zero(t.b);                                                   \
        g2 a; const bool good = sw_map_g2<true>(a, t);                                                                                \
        g2a res; fp2_zero(res.x); fp2_zero(res.y);                                                                                    \
        if (good) {                                                                                                                   \
            if (lane == 0) { vm_set_fp2(slots, VM_R_Q2X, a.x); vm_set_fp2(slots, VM_R_Q2Y, a.y); }                                   \
            __syncwarp();                                                                                                             \
            if (vm_hash_cofactor(slots) && !force_fallback) {                                                                         \
                if (lane == 0) { vm_ld(res.x.a.l, slots, VM_R_HX, 0); vm_ld(res.x.b.l, slots, VM_R_HX, 1); vm_ld(res.y.a.l, slots, VM_R_HY, 0); vm_ld(res.y.b.l, slots, VM_R_HY, 1); } \
            } else if (lane < 2) HB_HASH_TAIL_PAIR(res, a)                                                                            \
        }                                                                                                                             \
        if (lane == 0) { out[i] = res; ok[i] = good ? 1 : 0; }                                                                       \
        __syncwarp();                                                                                                                 \
    }
__global__ void __launch_bounds__(32) k_hash_to_g2_coop(size_t n, const uint8_t* msgs, uint32_t msg_len, g2a* out, uint8_t* ok, int force_fallback) {
    __shared__ uint32_t slots[VM_SMEM_WORDS];
    const int lane = threadIdx.x & 31;
    vm_load_consts(slots);
    for (size_t i = blockIdx.x; i < n; i += gridDim.x) HB_HASH_ITEM_WARP(i, msgs, msg_len, out, ok, slots, lane, force_fallback)
}

// same-message batches (the leader's prepare / commit vote collection, consensus/leader.go:127-290: every vote signs
// the same block hash / commit payload): H(m) is computed once and replicated.  With an index (concurrent herumi-API calls
// combined into one turn, hbls.cu): H(m) of each distinct message once, gathered to the requests -- hm[i] = src[idx[i]].
__global__ void k_broadcast_hm(size_t n, const uint32_t* idx, const g2a* src, const uint8_t* src_ok, g2a* hm, uint8_t* ok) {
    size_t i = HB_TID; if (i >= n) return;
    if (!idx) { if (i == 0) return; hm[i] = hm[0]; ok[i] = ok[0]; }
    else { hm[i] = src[idx[i]]; ok[i] = src_ok[idx[i]]; }
}

// ---- verification (R7/R8)
// ---- lane-pair form: lanes (2k, 2k+1) co-own round j (even lane = real parts, odd lane = imaginary parts of every Fp2).
// Half the per-thread state of a thread-per-round pairing => twice the warps for the same L1/L2 footprint.  Control flow is
// data-oblivious; rounds with an identity operand (never the case for honest input) are flagged 0xFF and recomputed by
// k_pairing_fixup with the thread-per-round code.
#ifndef HB_TPB_SPLIT
#define HB_TPB_SPLIT 512
#endif
#ifndef HB_MINBLOCKS_SPLIT
#define HB_MINBLOCKS_SPLIT 1        // 1 x 512 threads x 128 regs per SM, lock-stepped per Miller / exponentiation iteration
#endif
__global__ void __launch_bounds__(HB_TPB_SPLIT, HB_MINBLOCKS_SPLIT) k_pairing_verify_split(size_t B, const g2a* sig, const g1a* pk_neg, const g2a* hm,
                                 const uint8_t* ok_a, const uint8_t* ok_b, const uint8_t* ok_c, uint8_t* results, const int* run_if) {
    if (run_if && *run_if == 0) return;                                 // fallback pass of the batched form: nothing failed
    const int role = threadIdx.x & 1;
    const size_t ppg = HB_STRIDE >> 1;                                  // pairs per grid sweep
    for (size_t it = 0; ; it++) {
        const size_t warp_first = it * ppg + ((HB_TID & ~(size_t)31) >> 1);
        if (warp_first >= B) break;                                     // warp-uniform exit
        const size_t j = it * ppg + (HB_TID >> 1);
        const bool valid = j < B;
        const size_t jj = valid ? j : B - 1;
        bool good = (!ok_a || ok_a[jj]) && (!ok_b || ok_b[jj]) && (!ok_c || ok_c[jj]);
        g1a gen, p2 = pk_neg[jj];
        fp_set(gen.x, K_G1_X); fp_set(gen.y, K_G1_Y);
        const fp* s4 = reinterpret_cast<const fp*>(&sig[jj]);           // x.a, x.b, y.a, y.b
        const fp* h4 = reinterpret_cast<const fp*>(&hm[jj]);
        fp2h q1x, q1y, q2x, q2y;
        q1x.c = s4[role]; q1y.c = s4[2 + role]; q2x.c = h4[role]; q2y.c = h4[2 + role];
        // NB: no short-circuit around fp2_is_zero(fp2h) -- it shuffles across the whole warp
        const bool z1x = fp2_is_zero(q1x), z1y = fp2_is_zero(q1y), z2x = fp2_is_zero(q2x), z2y = fp2_is_zero(q2y);
        const bool irregular = (z1x & z1y) | (z2x & z2y) | (fp_is_zero(p2.x) & fp_is_zero(p2.y));
        fp12_t<fp2h> m;
        miller_loop2<fp2h>(m, gen, q1x, q1y, p2, q2x, q2y, true, true);
        final_exp(m, m);
        const bool one = fp12_is_one(m);
        if (valid && role == 0) results[j] = irregular ? 0xFF : ((good && one) ? 1 : 0);
    }
}
// rounds with an identity operand (thread-per-round code path).  An identity public key never verifies (include/hbls.h: a
// zero key would make the zero signature "valid" for every message); an identity signature is checked like any other point.
HB_NOINLINE bool verify_irregular(const g1a& gen, const g2a& q1, const g1a& p2, const g2a& q2) {
    if (aff_is_inf(p2)) return false;
    fp12 m; miller_loop2(m, gen, q1, p2, q2); final_exp(m, m);
    return fp12_is_one(m);
}
__global__ void k_pairing_fixup(size_t B, const g2a* sig, const g1a* pk_neg, const g2a* hm,
                                const uint8_t* ok_a, const uint8_t* ok_b, const uint8_t* ok_c, uint8_t* results, const int* run_if) {
  if (run_if && *run_if == 0) return;
  for (size_t j = HB_TID; j < B; j += HB_STRIDE) {
    if (results[j] != 0xFF) continue;
    bool good = (!ok_a || ok_a[j]) && (!ok_b || ok_b[j]) && (!ok_c || ok_c[j]);
    g1a gen, p2 = pk_neg[j]; g2a q1 = sig[j], q2 = hm[j];
    fp_set(gen.x, K_G1_X); fp_set(gen.y, K_G1_Y);
    results[j] = (good && verify_irregular(gen, q1, p2, q2)) ? 1 : 0;
  }
}
// ---- latency form (vm.cuh): ONE WARP per round runs the 2-pair Miller loop + final exponentiation as step programs over
// shared-memory slots, 16 lane pairs wide.  Same inputs, flags and result protocol as k_pairing_verify_split (0xFF = a round with an
// identity operand, decided afterwards by k_pairing_fixup).  Small batches: a single round is ~10x faster than on one lane pair.
__global__ void __launch_bounds__(32) k_pairing_coop(size_t B, const g2a* sig, const g1a* pk_neg, const g2a* hm,
                                 const uint8_t* ok_a, const uint8_t* ok_b, const uint8_t* ok_c, uint8_t* results) {
    __shared__ uint32_t slots[VM_SMEM_WORDS];
    const int lane = threadIdx.x & 31;
    vm_load_consts(slots);
    for (size_t j = blockIdx.x; j < B; j += gridDim.x) {
        const bool good = (!ok_a || ok_a[j]) && (!ok_b || ok_b[j]) && (!ok_c || ok_c[j]);
        // lanes 0..7 stage one operand each: P1 = generator, Q1 = signature, P2 = -pk, Q2 = H(m)
        bool zero = true;
        if (lane < 8) {
            fp2 v; fp2_zero(v);
            const g1a pk = pk_neg[j];
            switch (lane) {
            case 0: fp_set(v.a, K_G1_X); break;
            case 1: fp_set(v.a, K_G1_Y); break;
            case 2: v = sig[j].x; break;
            case 3: v = sig[j].y; break;
            case 4: v.a = pk.x; break;
            case 5: v.a = pk.y; break;
            case 6: v = hm[j].x; break;
            default: v = hm[j].y; break;
            }
            vm_set_fp2(slots, VM_R_P1X + lane, v);
            zero = fp_is_zero(v.a) & fp_is_zero(v.b);
        }
        const unsigned zmask = __ballot_sync(0xffffffffu, zero);            // bit l: operand l is zero
        const bool irregular = ((zmask & 0x0c) == 0x0c) | ((zmask & 0x30) == 0x30) | ((zmask & 0xc0) == 0xc0);
        bool one = false;
        if (!irregular) one = vm_pairing_check(slots);                        // warp-uniform branch
        if (lane == 0) results[j] = irregular ? 0xFF : ((good && one) ? 1 : 0);
        __syncwarp();
    }
}

// ---- ONE batch split over several GPUs (SURVEY 8e, BASELINE configs[3]): every rank turns its slice into a fixed-size partial record
// { sum_j r_j sigma_j (G2) , prod_j f_{|z|, H_j}(-r_j pk_j) (Fp12, no final exponentiation) , bad count }; the records are all-gathered
// (NCCL) and every rank folds them identically: prod of the partial products x Miller(B, sum of the partial sums), ONE final
// exponentiation.  EC addition / Fp12 multiplication are not NCCL reduction operators, hence all-gather + local fold.
// A warp multiplies the Miller values of its items (w, w + W, ...) into the VM register A; bad / identity items only count.
__global__ void __launch_bounds__(32) k_rlc_partial_coop(size_t n, const g1a* pk_scaled_neg, const g2a* hm, const uint8_t* bad,
                                                         fp2* partial /* 6 per warp, tower order */, unsigned* bad_count) {
    __shared__ uint32_t slots[VM_SMEM_WORDS];
    const int lane = threadIdx.x & 31;
    vm_load_consts(slots);
    vm_run(VM_P_A_ONE, slots);
    for (size_t j = blockIdx.x; j < n; j += gridDim.x) {
        bool zero = true;
        if (lane < 4) {
            fp2 v; fp2_zero(v);
            const g1a pk = pk_scaled_neg[j];
            if (lane == 0) v.a = pk.x; else if (lane == 1) v.a = pk.y; else if (lane == 2) v = hm[j].x; else v = hm[j].y;
            vm_set_fp2(slots, VM_R_P2X + lane, v);
            zero = fp_is_zero(v.a) & fp_is_zero(v.b);
        }
        const unsigned zmask = __ballot_sync(0xffffffffu, zero);
        const bool skip = bad[j] != 0 || (zmask & 0x3) == 0x3 || (zmask & 0xc) == 0xc;
        if (skip) { if (lane == 0) atomicAdd(bad_count, 1u); __syncwarp(); continue; }
        vm_run(VM_P_ML1_INIT, slots);
        for (int i = 62; i >= 0; i--) {
            vm_run(VM_P_ML1_DBL, slots);
            if ((K_Z_ABS >> i) & 1) vm_run(VM_P_ML1_ADD, slots);
        }
        vm_run(VM_P_AMULF, slots);
    }
    if (lane < 12) vm_ld(reinterpret_cast<fp*>(&partial[6 * (size_t)blockIdx.x + (lane >> 1)])[lane & 1].l, slots, VM_R_A0 + (lane >> 1), lane & 1);
}
// product of W partial products (one warp)
__global__ void __launch_bounds__(32) k_rlc_reduce_coop(size_t W, const fp2* partial, fp2* out) {
    __shared__ uint32_t slots[VM_SMEM_WORDS];
    const int lane = threadIdx.x & 31;
    vm_load_consts(slots);
    vm_run(VM_P_A_ONE, slots);
    for (size_t w = 0; w < W; w++) {
        if (lane < 12) vm_st(slots, VM_R_F0 + (lane >> 1), lane & 1, reinterpret_cast<const fp*>(&partial[6 * w + (lane >> 1)])[lane & 1].l);
        __syncwarp();
        vm_run(VM_P_AMULF, slots);
    }
    if (lane < 12) vm_ld(reinterpret_cast<fp*>(&out[lane >> 1])[lane & 1].l, slots, VM_R_A0 + (lane >> 1), lane & 1);
}
// fold: verdict = FE( prod_p parts[p] * Miller(B, Sg) ) == 1, Sg = affine sum of the partial signature sums (not the identity)
__global__ void __launch_bounds__(32) k_rlc_fold_coop(size_t nparts, const fp2* parts, const g2a* Sg, uint8_t* result) {
    __shared__ uint32_t slots[VM_SMEM_WORDS];
    const int lane = threadIdx.x & 31;
    vm_load_consts(slots);
    vm_run(VM_P_A_ONE, slots);
    for (size_t w = 0; w < nparts; w++) {
        if (lane < 12) vm_st(slots, VM_R_F0 + (lane >> 1), lane & 1, reinterpret_cast<const fp*>(&parts[6 * w + (lane >> 1)])[lane & 1].l);
        __syncwarp();
        vm_run(VM_P_AMULF, slots);
    }
    bool zero = true;
    if (lane < 4) {
        fp2 v; fp2_zero(v);
        if (lane == 0) fp_set(v.a, K_G1_X); else if (lane == 1) fp_set(v.a, K_G1_Y); else if (lane == 2) v = Sg->x; else v = Sg->y;
        vm_set_fp2(slots, VM_R_P2X + lane, v);
        zero = fp_is_zero(v.a) & fp_is_zero(v.b);
    }
    const unsigned zmask = __ballot_sync(0xffffffffu, zero);
    if ((zmask & 0xc) == 0xc) { if (lane == 0) *result = 0; return; }       // empty / cancelling signature sum: not proven, callers fall back
    vm_run(VM_P_ML1_INIT, slots);
    for (int i = 62; i >= 0; i--) {
        vm_run(VM_P_ML1_DBL, slots);
        if ((K_Z_ABS >> i) & 1) vm_run(VM_P_ML1_ADD, slots);
    }
    vm_run(VM_P_FMULA, slots);
    const bool one = vm_final_exp_is_one(slots);
    if (lane == 0) *result = one ? 1 : 0;
}
// Jacobian G2 sum, single CTA (the partial signature sums)
__global__ void __launch_bounds__(HB_SUM_THREADS) k_g2_sum_jac(size_t n, const g2* in, g2* out) {
    __shared__ g2 sm[HB_SUM_THREADS];
    g2 acc; pt_set_inf(acc);
    for (size_t i = threadIdx.x; i < n; i += HB_SUM_THREADS) { g2 q = in[i]; pt_add(acc, acc, q); }
    sm[threadIdx.x] = acc;
    __syncthreads();
    for (int off = HB_SUM_THREADS / 2; off >= 1; off >>= 1) {
        if ((int)threadIdx.x < off) { g2 o = sm[threadIdx.x + off]; pt_add(acc, acc, o); sm[threadIdx.x] = acc; }
        __syncthreads();
    }
    if (threadIdx.x == 0) out[0] = acc;
}

// ---- latency form, split in two: the Miller value of (B, sigma) only needs the decoded signature, so it is computed on the decode
// stream while hash-to-G2 (the long pole of a single check) still runs; the second kernel adds the pair (-apk, H(m)) and the final
// exponentiation.  f1: 6 Fp2 per round (tower order); irr1[j] = 1 when the signature is the identity / did not decode.
__global__ void __launch_bounds__(32) k_miller1_coop(size_t B, const g2a* sig, const uint8_t* ok_sig, fp2* f1, uint8_t* irr1) {
    __shared__ uint32_t slots[VM_SMEM_WORDS];
    const int lane = threadIdx.x & 31;
    vm_load_consts(slots);
    for (size_t j = blockIdx.x; j < B; j += gridDim.x) {
        bool zero = true;
        if (lane < 4) {
            fp2 v; fp2_zero(v);
            if (lane == 0) fp_set(v.a, K_G1_X); else if (lane == 1) fp_set(v.a, K_G1_Y); else if (lane == 2) v = sig[j].x; else v = sig[j].y;
            vm_set_fp2(slots, VM_R_P2X + lane, v);
            zero = fp_is_zero(v.a) & fp_is_zero(v.b);
        }
        const unsigned zmask = __ballot_sync(0xffffffffu, zero);
        const bool skip = (ok_sig && !ok_sig[j]) || (zmask & 0xc) == 0xc;
        if (lane == 0) irr1[j] = skip ? 1 : 0;
        if (skip) { __syncwarp(); continue; }
        vm_run(VM_P_ML1_INIT, slots);
        for (int i = 62; i >= 0; i--) {
            vm_run(VM_P_ML1_DBL, slots);
            if ((K_Z_ABS >> i) & 1) vm_run(VM_P_ML1_ADD, slots);
        }
        if (lane < 12) vm_ld(reinterpret_cast<fp*>(&f1[6 * j + (lane >> 1)])[lane & 1].l, slots, VM_R_F0 + (lane >> 1), lane & 1);
        __syncwarp();
    }
}
// ---- latency form with H(m) already known (the library's H(m) cache, hbls.cu): BOTH Miller values are independent of each other --
// (B, sigma) waits for the signature decode, (-apk, H(m)) only for the key aggregation -- so they run on two streams and a third
// kernel multiplies them and does the final exponentiation.  P = nullptr: the generator.  irr[j] = 1: an operand is the identity /
// did not decode (the round is then decided by k_pairing_fixup, like in the other forms).
__global__ void __launch_bounds__(32) k_miller_pq_coop(size_t B, const g1a* P, const g2a* Q, const uint8_t* ok_q, fp2* f, uint8_t* irr) {
    __shared__ uint32_t slots[VM_SMEM_WORDS];
    const int lane = threadIdx.x & 31;
    vm_load_consts(slots);
    for (size_t j = blockIdx.x; j < B; j += gridDim.x) {
        bool zero = true;
        if (lane < 4) {
            fp2 v; fp2_zero(v);
            if (lane < 2) { if (P) v.a = lane == 0 ? P[j].x : P[j].y; else fp_set(v.a, lane == 0 ? K_G1_X : K_G1_Y); }
            else v = lane == 2 ? Q[j].x : Q[j].y;
            vm_set_fp2(slots, VM_R_P2X + lane, v);
            zero = fp_is_zero(v.a) & fp_is_zero(v.b);
        }
        const unsigned zmask = __ballot_sync(0xffffffffu, zero);
        const bool skip = (ok_q && !ok_q[j]) || (zmask & 0x3) == 0x3 || (zmask & 0xc) == 0xc;
        if (lane == 0) irr[j] = skip ? 1 : 0;
        if (skip) { __syncwarp(); continue; }
        vm_run(VM_P_ML1_INIT, slots);
        for (int i = 62; i >= 0; i--) {
            vm_run(VM_P_ML1_DBL, slots);
            if ((K_Z_ABS >> i) & 1) vm_run(VM_P_ML1_ADD, slots);
        }
        if (lane < 12) vm_ld(reinterpret_cast<fp*>(&f[6 * j + (lane >> 1)])[lane & 1].l, slots, VM_R_F0 + (lane >> 1), lane & 1);
        __syncwarp();
    }
}
// verdict = FE(f1 f2) == 1; ok_sub (nullable): the signature's subgroup test, run beside its Miller loop
__global__ void __launch_bounds__(32) k_fe2_coop(size_t B, const fp2* f1, const uint8_t* irr1, const fp2* f2, const uint8_t* irr2,
                             const uint8_t* ok_a, const uint8_t* ok_b, const uint8_t* ok_c, const uint8_t* ok_sub, uint8_t* results) {
    __shared__ uint32_t slots[VM_SMEM_WORDS];
    const int lane = threadIdx.x & 31;
    vm_load_consts(slots);
    for (size_t j = blockIdx.x; j < B; j += gridDim.x) {
        const bool good = (!ok_a || ok_a[j]) && (!ok_b || ok_b[j]) && (!ok_c || ok_c[j]) && (!ok_sub || ok_sub[j]);
        const bool irregular = irr1[j] != 0 || irr2[j] != 0;
        bool one = false;
        if (!irregular) {
            if (lane < 12) {
                vm_st(slots, VM_R_A0 + (lane >> 1), lane & 1, reinterpret_cast<const fp*>(&f1[6 * j + (lane >> 1)])[lane & 1].l);
                vm_st(slots, VM_R_F0 + (lane >> 1), lane & 1, reinterpret_cast<const fp*>(&f2[6 * j + (lane >> 1)])[lane & 1].l);
            }
            __syncwarp();
            vm_run(VM_P_FMULA, slots);
            one = vm_final_exp_is_one(slots);
        }
        if (lane == 0) results[j] = irregular ? 0xFF : ((good && one) ? 1 : 0);
        __syncwarp();
    }
}
// ---- large-batch G2 ladders on the lane-pair carrier: one item per lane pair, persistent, one lock-stepped CTA per SM (hbls.cu
// lockstep_cta).  The carrier halves each thread's state (frames of ~1.3 KB instead of 3-4.7 KB for one item per thread), so the
// ladders' operands stay in L1 at 512 resident threads; the Fp-level work is the same.  Sweep `it` gives lane pair q item
// it * pairs + q; a warp leaves as a whole once its first item is past n, and a CTA barrier per sweep keeps the warps of a CTA on
// the same instruction-cache lines.
template <class Body> HB_DEV void pair_sweep(size_t n, Body body) {
    const size_t ppg = HB_STRIDE >> 1;
    for (size_t it = 0; ; it++) {
        if (it * ppg + ((HB_TID & ~(size_t)31) >> 1) >= n) break;
        hb_lockstep<fp2h>();
        const size_t i = it * ppg + (HB_TID >> 1);
        if (i < n) body(i);
    }
}
// subgroup test of already-decoded affine signatures (the second half of k_g2_decode_pair; for large batches the second half of the
// split decode stage).  zero_bad: a point outside the subgroup is also zeroed in place, as k_g2_subgroup does.
__global__ void __launch_bounds__(HB_TPB_SPLIT, HB_MINBLOCKS_SPLIT) k_g2_subgroup_pair(size_t n, g2a* pts, const uint8_t* ok_in, uint8_t* ok_out,
                                                                                      int zero_bad = 0) {
    const int role = threadIdx.x & 1;
    pair_sweep(n, [&](size_t i) {
        const fp* a4 = reinterpret_cast<const fp*>(&pts[i]);
        aff<fp2h> a; a.x.c = a4[role]; a.y.c = a4[2 + role];
        const bool in = ok_in[i] != 0;
        bool good = in;
        if (good) good = g2_in_subgroup_aff(a);
        if (zero_bad && in && !good) { fp* o = reinterpret_cast<fp*>(&pts[i]); fp_zero(o[role]); fp_zero(o[2 + role]); }
        if (role == 0) ok_out[i] = good ? 1 : 0;
    });
}
// cofactor clearing of the SW map's output (k_hash_sw) into the Jacobian buffer k_g2_normalize_batch converts: k_hash_cofactor_jac
// on the lane-pair carrier, byte for byte.  hbls.cu runs k_hash_cofactor_z1_pair + _z2_pair below; this one is the reference tests compare them with.
__global__ void __launch_bounds__(HB_TPB_SPLIT, HB_MINBLOCKS_SPLIT) k_hash_cofactor_pair(size_t n, const g2a* pts, const uint8_t* ok, g2* out) {
    const int role = threadIdx.x & 1;
    pair_sweep(n, [&](size_t i) {
        jac<fp2h> h; pt_set_inf(h);
        if (ok[i]) {
            const fp* p4 = reinterpret_cast<const fp*>(&pts[i]);
            jac<fp2h> a; a.x.c = p4[role]; a.y.c = p4[2 + role]; fp2_one(a.z);
            g2_clear_cofactor(h, a);
        }
        fp* o = reinterpret_cast<fp*>(&out[i]); o[role] = h.x.c; o[2 + role] = h.y.c; o[4 + role] = h.z.c;
    });
}
// the cofactor clearing hbls.cu runs, g2_clear_cofactor_aff_z1 / _z2 on the lane-pair carrier as two kernels of one |z| ladder each
// (each the size of k_g2_subgroup_pair, instead of one kernel holding both ladders, the combination and both group laws): the first
// writes t1 = [z]P (the identity where ok is not set) into out, the second turns it into h(P) in place.  Together they give the same
// affine H(m) as k_hash_cofactor_pair after k_g2_normalize_batch.  The map's outputs are never the identity; the all-zero encoding
// with ok set gives the identity, as in k_hash_cofactor_pair.
__global__ void __launch_bounds__(HB_TPB_SPLIT, HB_MINBLOCKS_SPLIT) k_hash_cofactor_z1_pair(size_t n, const g2a* pts, const uint8_t* ok, g2* out) {
    const int role = threadIdx.x & 1;
    pair_sweep(n, [&](size_t i) {
        jac<fp2h> t1; pt_set_inf(t1);
        if (ok[i]) {
            const fp* p4 = reinterpret_cast<const fp*>(&pts[i]);
            aff<fp2h> a; a.x.c = p4[role]; a.y.c = p4[2 + role];
            g2_clear_cofactor_aff_z1(t1, a);
        }
        fp* o = reinterpret_cast<fp*>(&out[i]); o[role] = t1.x.c; o[2 + role] = t1.y.c; o[4 + role] = t1.z.c;
    });
}
__global__ void __launch_bounds__(HB_TPB_SPLIT, HB_MINBLOCKS_SPLIT) k_hash_cofactor_z2_pair(size_t n, const g2a* pts, const uint8_t* ok, g2* io) {
    const int role = threadIdx.x & 1;
    pair_sweep(n, [&](size_t i) {
        if (!ok[i]) return;
        const fp* p4 = reinterpret_cast<const fp*>(&pts[i]);
        aff<fp2h> a; a.x.c = p4[role]; a.y.c = p4[2 + role];
        fp* o = reinterpret_cast<fp*>(&io[i]);
        jac<fp2h> t1, h; t1.x.c = o[role]; t1.y.c = o[2 + role]; t1.z.c = o[4 + role];
        g2_clear_cofactor_aff_z2(h, t1, a);
        o[role] = h.x.c; o[2 + role] = h.y.c; o[4 + role] = h.z.c;
    });
}
__global__ void __launch_bounds__(32) k_pairing_coop2(size_t B, const fp2* f1, const uint8_t* irr1, const g1a* pk_neg, const g2a* hm,
                                  const uint8_t* ok_a, const uint8_t* ok_b, const uint8_t* ok_c, uint8_t* results) {
    __shared__ uint32_t slots[VM_SMEM_WORDS];
    const int lane = threadIdx.x & 31;
    vm_load_consts(slots);
    for (size_t j = blockIdx.x; j < B; j += gridDim.x) {
        const bool good = (!ok_a || ok_a[j]) && (!ok_b || ok_b[j]) && (!ok_c || ok_c[j]);
        bool zero = true;
        if (lane < 4) {
            fp2 v; fp2_zero(v);
            const g1a pk = pk_neg[j];
            if (lane == 0) v.a = pk.x; else if (lane == 1) v.a = pk.y; else if (lane == 2) v = hm[j].x; else v = hm[j].y;
            vm_set_fp2(slots, VM_R_P2X + lane, v);
            zero = fp_is_zero(v.a) & fp_is_zero(v.b);
        }
        const unsigned zmask = __ballot_sync(0xffffffffu, zero);
        const bool irregular = irr1[j] != 0 || (zmask & 0x3) == 0x3 || (zmask & 0xc) == 0xc;
        bool one = false;
        if (!irregular) {
            if (lane < 12) vm_st(slots, VM_R_A0 + (lane >> 1), lane & 1, reinterpret_cast<const fp*>(&f1[6 * j + (lane >> 1)])[lane & 1].l);
            __syncwarp();
            vm_run(VM_P_ML1_INIT, slots);
            for (int i = 62; i >= 0; i--) {
                vm_run(VM_P_ML1_DBL, slots);
                if ((K_Z_ABS >> i) & 1) vm_run(VM_P_ML1_ADD, slots);
            }
            vm_run(VM_P_FMULA, slots);
            one = vm_final_exp_is_one(slots);
        }
        if (lane == 0) results[j] = irregular ? 0xFF : ((good && one) ? 1 : 0);
        __syncwarp();
    }
}

// ------------------------------------------------------------------ random-linear-combination batch (R9 / R10 GPU form)
// prod_j [ e(B, sigma_j) e(-apk_j, H_j) ]^{r_j} == 1 with 64-bit r_j: the G rounds of a group share ONE Miller accumulator
// (pairs (-r_j apk_j, H_j) plus (B, sum_j r_j sigma_j)) and ONE final exponentiation.  The rounds of a group that fails -- or
// holds a round that did not decode -- are re-verified exactly afterwards (compacted list, k_pairing_verify_split_list), so
// results stay exact booleans (a bad round survives the batched test with probability <= 2^-63).
#ifndef HB_RLC_G
#define HB_RLC_G 4       // smallest group size (scratch is sized for it); the host picks 4 or 8 per call (hbls.cu): larger groups save
                         // final exponentiations, but the group count must still fill the SMs
#endif
#define HB_RLC_GMAX 8
// Groups are STRIDED: group g = rounds {g, g + ng, g + 2 ng, ...}; the coefficient depends only on the position k inside the
// group (c[k], fresh per call from the host's keyed ChaCha20 stream: hbls.cu rlc_draw), so the 32 consecutive rounds of a warp
// share one scalar and the double-and-add ladders run without divergence.  Sharing c[k] across groups is sound: every group's
// test passes wrongly with probability <= 2^-63 over the draw, whatever the (non-adaptive) input.
struct rlc_coeffs { uint64_t c[HB_RLC_GMAX]; };
// Blocks (hbls.cu rlc_blocks): HB_RLC_M groups share ONE final exponentiation and ONE generator pair.  Group g is member m = g / S of
// block b = g mod S, S = ceil(ng / HB_RLC_M) rounded up to a multiple of 32, so the 32 consecutive groups of a warp of the scaling
// kernels share (k, m) and their ladders stay warp-uniform.  Equal coefficients would no longer do: two bad rounds at the same
// position of two groups of one block (sigma_a + D, sigma_b - D) would cancel in the block's product.  So every (position, member)
// gets its own draw and only (0, 0) keeps 1.
#define HB_RLC_M 16
struct rlc_block_coeffs { uint64_t c[HB_RLC_GMAX][HB_RLC_M]; };
// Coefficient sources of the scaling kernels (a template parameter of each, deduced at the launch): the structs above, passed by value
// (direct calls: hbls.cu draws them on the host per call), or these pointer wrappers with the same c[k] / c[k][m] access into device
// memory (calls captured into a CUDA graph: k_rlc_draw writes them there at every replay, so no coefficient is frozen into a node).
struct rlc_coeffs_dev { const uint64_t* c; };
struct rlc_block_coeffs_dev { const uint64_t (*c)[HB_RLC_M]; };
// coefficient of round j = k ng + g: per position (S = 0: every group checked on its own), or per (position, block member)
template <class CO, class CB>
HB_DEV uint64_t rlc_coeff(const CO& co, size_t j, size_t ng, size_t S, const CB& cb) {
    const size_t k = j / ng;
    if (!S) return k ? co.c[k] : 1ull;
    const size_t m = (j - k * ng) / S;
    return (k | m) ? cb.c[k][m] : 1ull;
}
// ---- secrets of a captured call, drawn on the device.  ChaCha20 block function (RFC 8439 section 2.3) on a whole 16-word state.
HB_DEV uint32_t chacha_rotl(uint32_t v, int c) { return (v << c) | (v >> (32 - c)); }
HB_DEV void chacha_qr(uint32_t* x, int a, int b, int c, int d) {
    x[a] += x[b]; x[d] ^= x[a]; x[d] = chacha_rotl(x[d], 16); x[c] += x[d]; x[b] ^= x[c]; x[b] = chacha_rotl(x[b], 12);
    x[a] += x[b]; x[d] ^= x[a]; x[d] = chacha_rotl(x[d], 8);  x[c] += x[d]; x[b] ^= x[c]; x[b] = chacha_rotl(x[b], 7);
}
HB_DEV void chacha20_block_dev(const uint32_t st[16], uint32_t out[16]) {
    uint32_t x[16];
    for (int i = 0; i < 16; i++) x[i] = st[i];
    for (int r = 0; r < 10; r++) {
        chacha_qr(x, 0, 4, 8, 12); chacha_qr(x, 1, 5, 9, 13); chacha_qr(x, 2, 6, 10, 14); chacha_qr(x, 3, 7, 11, 15);
        chacha_qr(x, 0, 5, 10, 15); chacha_qr(x, 1, 6, 11, 12); chacha_qr(x, 2, 7, 8, 13); chacha_qr(x, 3, 4, 9, 14);
    }
    for (int i = 0; i < 16; i++) out[i] = x[i] + st[i];
}
// What k_rlc_draw writes into a captured call's scratch: keystream blocks 0 .. 17 of the call's counter, in order.  Block 0 = the
// per-position coefficients, block 1 = the message-grouping salt (device_forms.cuh k_group_insert), blocks 2 .. 17 = the
// per-(position, member) coefficients of the block form, each 64-bit value from two consecutive words as the host stream packs
// them (hbls.cu rlc_draw, rlc_draw_block, launch_hash_grouped).
struct rlc_draw_out { rlc_coeffs co; uint64_t salt[2]; uint64_t unused[6]; rlc_block_coeffs cb; };
static_assert(sizeof(rlc_draw_out) == 18 * 64, "one keystream block per 64 bytes");
// Words 12, 13 of the state are the call counter, 14 the stream's nonce word, 15 the block.  The host stream (hbls.cu chacha20_block)
// uses the same key under nonce word 0x68626c73, so no keystream block is ever used by both.
#define HB_RLC_DRAW_NONCE 0x68626c64u     /* "dlbh" */
#ifndef HB_HOST_EMU
// one warp: lane 0 takes the call's counter value (one atomicAdd on *draws, so every launch -- every graph replay -- draws anew), lane
// b < nblocks writes block b.  The key is read from device memory and never appears in a kernel parameter or a graph node.
__global__ void k_rlc_draw(const uint32_t* key, unsigned long long* draws, uint32_t nonce, uint32_t nblocks, rlc_draw_out* out) {
    const unsigned lane = threadIdx.x;
    unsigned long long call = 0;
    if (lane == 0) call = atomicAdd(draws, 1ull);
    call = __shfl_sync(0xffffffffu, call, 0);
    if (lane >= nblocks) return;
    uint32_t st[16] = {0x61707865u, 0x3320646eu, 0x79622d32u, 0x6b206574u, key[0], key[1], key[2], key[3], key[4], key[5], key[6], key[7],
                       (uint32_t)call, (uint32_t)(call >> 32), nonce, lane};
    uint32_t blk[16];
    chacha20_block_dev(st, blk);
    uint32_t* o = reinterpret_cast<uint32_t*>(out) + 16 * lane;
    for (int i = 0; i < 16; i++) o[i] = blk[i];
}
#endif
// per round: P_j = -r_j apk_j (affine), S_j = r_j sigma_j (Jacobian), bad_j
#ifndef HB_SCALE_MINBLOCKS
#define HB_SCALE_MINBLOCKS 1
#endif
template <class CO = rlc_coeffs, class CB = rlc_block_coeffs>
__global__ void __launch_bounds__(64, HB_SCALE_MINBLOCKS) k_rlc_scale(size_t B, size_t ng, const g1* apk, const g2a* sig, const g2a* hm, const uint8_t* ok_sig, const uint8_t* ok_hm,
                            const uint8_t* ok_pk, CO co, const uint64_t* per_item, g1a* pk_scaled_neg, g2* S, uint8_t* bad,
                            size_t blk_stride = 0, CB cb = {}, const unsigned* blk_gate = nullptr) {
  if (blk_gate && *blk_gate == 0) blk_stride = 0;        // the device chose the group form (k_rlc_form): per-position coefficients
  // per_item (nullable): one independent coefficient per round -- needed when ALL rounds enter one combined check (the split of a
  // single batch over several GPUs, k_rlc_partial_coop); the grouped form shares co.c[position in group] across groups, the block
  // form (blk_stride = S != 0) cb.c[position][member]
#if HB_BATCH_INV
  for (size_t j0 = HB_TID; j0 < B; j0 += (size_t)HB_BATCH_K * HB_STRIDE) {
    g1 ra[HB_BATCH_K]; fp z[HB_BATCH_K]; bool skip[HB_BATCH_K];
    for (int k = 0; k < HB_BATCH_K; k++) {
        const size_t j = j0 + (size_t)k * HB_STRIDE;
        skip[k] = true;
        if (j >= B) continue;
        // grouped form: the FIRST round of every group keeps coefficient 1 (no ladders at all: a warp-uniform branch, since the 32
        // rounds of a warp share their position).  Sound: a group holding a bad round passes only if prod_j delta_j^{s_j} = 1 with
        // some delta_j != 1; if that j is 0 alone the product is delta_0 != 1, otherwise one of the random s_j (j >= 1) must hit
        // the single value mod r that cancels the rest -- probability <= 2^-63, as before.
        const uint64_t r = per_item ? per_item[j] : rlc_coeff(co, j, ng, blk_stride, cb);
        g1 a = apk[j]; g2a sg = sig[j]; g2a h = hm[j];
        const bool b = !ok_sig[j] || !ok_hm[j] || (ok_pk && !ok_pk[j]) || pt_is_inf(a) || aff_is_inf(sg) || aff_is_inf(h);
        g2 rs;
        if (r == 1ull && !per_item) { ra[k] = a; pt_from_aff(rs, sg); } else rlc_scale_pair(ra[k], rs, a, sg, r);
        S[j] = rs; bad[j] = b ? 1 : 0;
        skip[k] = pt_is_inf(ra[k]);
        if (!skip[k]) z[k] = ra[k].z;
    }
    f_batch_inv<fp, HB_BATCH_K>(z, skip);
    for (int k = 0; k < HB_BATCH_K; k++) {
        const size_t j = j0 + (size_t)k * HB_STRIDE;
        if (j >= B) continue;
        g1a pa;
        if (skip[k]) { fp_zero(pa.x); fp_zero(pa.y); } else { pt_to_aff_zinv(pa, ra[k], z[k]); fp_neg(pa.y, pa.y); }
        pk_scaled_neg[j] = pa;
    }
  }
#else
  for (size_t j = HB_TID; j < B; j += HB_STRIDE) {
    const uint64_t r = per_item ? per_item[j] : rlc_coeff(co, j, ng, blk_stride, cb);
    g1 a = apk[j]; g2a sg = sig[j]; g2a h = hm[j];
    const bool b = !ok_sig[j] || !ok_hm[j] || (ok_pk && !ok_pk[j]) || pt_is_inf(a) || aff_is_inf(sg) || aff_is_inf(h);
    g1 ra; g2 rs;
    if (r == 1ull && !per_item) { ra = a; pt_from_aff(rs, sg); } else rlc_scale_pair(ra, rs, a, sg, r);
    g1a pa; pt_to_aff(pa, ra); fp_neg(pa.y, pa.y);
    pk_scaled_neg[j] = pa; S[j] = rs; bad[j] = b ? 1 : 0;
  }
#endif
}
// the same stage as two kernels, one ladder each (hbls.cu "scale_split"): the G1 ladder (+ shared-inversion affine conversion) and the
// G2 ladder are different code over different fields, and one kernel holding both stalls on instruction fetch
template <class CO = rlc_coeffs, class CB = rlc_block_coeffs>
__global__ void k_rlc_scale_g1(size_t B, size_t ng, const g1* apk, CO co, g1a* pk_scaled_neg, size_t blk_stride = 0, CB cb = {},
                               const unsigned* blk_gate = nullptr) {
  if (blk_gate && *blk_gate == 0) blk_stride = 0;
  for (size_t j0 = HB_TID; j0 < B; j0 += (size_t)HB_BATCH_K * HB_STRIDE) {
    g1 ra[HB_BATCH_K]; fp z[HB_BATCH_K]; bool skip[HB_BATCH_K];
    for (int k = 0; k < HB_BATCH_K; k++) {
        const size_t j = j0 + (size_t)k * HB_STRIDE;
        skip[k] = true;
        if (j >= B) continue;
        const g1 a = apk[j];
        const uint64_t r = rlc_coeff(co, j, ng, blk_stride, cb);
        if (r == 1ull) ra[k] = a; else rlc_scale_g1(ra[k], a, r);
        skip[k] = pt_is_inf(ra[k]);
        if (!skip[k]) z[k] = ra[k].z;
    }
    f_batch_inv<fp, HB_BATCH_K>(z, skip);
    for (int k = 0; k < HB_BATCH_K; k++) {
        const size_t j = j0 + (size_t)k * HB_STRIDE;
        if (j >= B) continue;
        g1a pa;
        if (skip[k]) { fp_zero(pa.x); fp_zero(pa.y); } else { pt_to_aff_zinv(pa, ra[k], z[k]); fp_neg(pa.y, pa.y); }
        pk_scaled_neg[j] = pa;
    }
  }
}
#ifndef HB_SCALE_G2_MINBLOCKS
#define HB_SCALE_G2_MINBLOCKS 1
#endif
// the G2 ladder of the stage, one round per thread: the reference for k_rlc_scale_g2_pair, which hbls.cu runs
__global__ void __launch_bounds__(64, HB_SCALE_G2_MINBLOCKS) k_rlc_scale_g2(size_t B, size_t ng, const g1* apk, const g2a* sig, const g2a* hm, const uint8_t* ok_sig, const uint8_t* ok_hm,
                               const uint8_t* ok_pk, rlc_coeffs co, g2* S, uint8_t* bad, size_t blk_stride = 0, rlc_block_coeffs cb = {},
                               const unsigned* blk_gate = nullptr) {
  if (blk_gate && *blk_gate == 0) blk_stride = 0;
  for (size_t j = HB_TID; j < B; j += HB_STRIDE) {
    const g2a sg = sig[j];
    const bool b = !ok_sig[j] || !ok_hm[j] || (ok_pk && !ok_pk[j]) || fp_is_zero(apk[j].z) || aff_is_inf(sg) || aff_is_inf(hm[j]);
    g2 rs;
    const uint64_t r = rlc_coeff(co, j, ng, blk_stride, cb);
    if (r == 1ull) pt_from_aff(rs, sg); else rlc_scale_g2(rs, sg, r);
    S[j] = rs; bad[j] = b ? 1 : 0;
  }
}
// k_rlc_scale_g2 on the lane-pair carrier (pair_sweep).  A warp's 16 pairs hold 16 consecutive rounds, which share their coefficient
// (the 32 of a warp of the thread kernel do), so the JSF digits stay warp-uniform.
template <class CO = rlc_coeffs, class CB = rlc_block_coeffs>
__global__ void __launch_bounds__(HB_TPB_SPLIT, HB_MINBLOCKS_SPLIT) k_rlc_scale_g2_pair(size_t B, size_t ng, const g1* apk, const g2a* sig, const g2a* hm,
                               const uint8_t* ok_sig, const uint8_t* ok_hm, const uint8_t* ok_pk, CO co, g2* S, uint8_t* bad,
                               size_t blk_stride = 0, CB cb = {}, const unsigned* blk_gate = nullptr) {
  if (blk_gate && *blk_gate == 0) blk_stride = 0;
  const int role = threadIdx.x & 1;
  pair_sweep(B, [&](size_t j) {
    const fp* s4 = reinterpret_cast<const fp*>(&sig[j]);
    const fp* h4 = reinterpret_cast<const fp*>(&hm[j]);
    aff<fp2h> sg, h; sg.x.c = s4[role]; sg.y.c = s4[2 + role]; h.x.c = h4[role]; h.y.c = h4[2 + role];
    const bool b = !ok_sig[j] || !ok_hm[j] || (ok_pk && !ok_pk[j]) || fp_is_zero(apk[j].z) || aff_is_inf(sg) || aff_is_inf(h);
    jac<fp2h> rs;
    const uint64_t r = rlc_coeff(co, j, ng, blk_stride, cb);
    if (r == 1ull) pt_from_aff(rs, sg); else rlc_scale_g2(rs, sg, r);
    fp* o = reinterpret_cast<fp*>(&S[j]); o[role] = rs.x.c; o[2 + role] = rs.y.c; o[4 + role] = rs.z.c;
    if (role == 0) bad[j] = b ? 1 : 0;
  });
}
// per group: affine sum of its S_j
template <int G> __global__ void k_rlc_group_sum(size_t ngroups, const g2* S, g2a* Sg) {
  for (size_t g = HB_TID; g < ngroups; g += HB_STRIDE) {
    g2 acc; pt_set_inf(acc);
    for (int k = 0; k < G; k++) { g2 t = S[(size_t)k * ngroups + g]; pt_add(acc, acc, t); }
    g2a a; pt_to_aff(a, acc); Sg[g] = a;
  }
}
// k_rlc_scale_g2_pair + k_rlc_group_sum<G> as ONE joint ladder per group (hbls.cu "scale_joint"): the pairing stage reads the rounds'
// scaled signatures only through their group sum Sg = sum_k s_k sigma_k, so a lane pair runs pt_mul_joint_naf over the group's 2G
// half-scalars (a_k on sigma_k, b_k on psi^2 sigma_k, split as in rlc_scale_g2) and its rounds share 33 doublings instead of running
// a ladder each.  The unit coefficient is (a, b) = (1, 0): one addition of sigma_k.  Writes the Jacobian Sg (k_g2_normalize_batch
// turns it affine) and the bad flag of each of the G rounds, by k_rlc_scale_g2_pair's rule.  A warp's 16 pairs hold 16 consecutive
// groups, which share every coefficient (per position, or per (position, member) with the member stride a multiple of 32), so the
// digits stay warp-uniform.
template <int G, class CO = rlc_coeffs, class CB = rlc_block_coeffs>
__global__ void __launch_bounds__(HB_TPB_SPLIT, HB_MINBLOCKS_SPLIT) k_rlc_group_scale_g2_pair(size_t ng, const g1* apk, const g2a* sig,
        const g2a* hm, const uint8_t* ok_sig, const uint8_t* ok_hm, const uint8_t* ok_pk, CO co, g2* Sg, uint8_t* bad,
        size_t blk_stride = 0, CB cb = {}, const unsigned* blk_gate = nullptr) {
  if (blk_gate && *blk_gate == 0) blk_stride = 0;
  const int role = threadIdx.x & 1;
  pair_sweep(ng, [&](size_t g) {
    uint32_t k[2 * G];
    for (int t = 0; t < G; t++) {
        const size_t j = (size_t)t * ng + g;
        const uint64_t c = rlc_coeff(co, j, ng, blk_stride, cb);
        k[2 * t] = (uint32_t)c | 1u; k[2 * t + 1] = (uint32_t)(c >> 32);
        const fp* s4 = reinterpret_cast<const fp*>(&sig[j]);
        const fp* h4 = reinterpret_cast<const fp*>(&hm[j]);
        aff<fp2h> sg, h; sg.x.c = s4[role]; sg.y.c = s4[2 + role]; h.x.c = h4[role]; h.y.c = h4[2 + role];
        const bool b = !ok_sig[j] || !ok_hm[j] || (ok_pk && !ok_pk[j]) || fp_is_zero(apk[j].z) || aff_is_inf(sg) || aff_is_inf(h);
        if (role == 0) bad[j] = b ? 1 : 0;
    }
    jac<fp2h> acc;
    pt_mul_joint_naf<fp2h, 2 * G>(acc, k, [&](int t, aff<fp2h>& q) {
        const fp* s4 = reinterpret_cast<const fp*>(&sig[(size_t)(t >> 1) * ng + g]);
        q.x.c = s4[role]; q.y.c = s4[2 + role];
        if (t & 1) { fp2_mul_fp(q.x, q.x, fp_k(K_PSI2_CX)); fp2_neg(q.y, q.y); }      // psi^2(x, y) = (N(cx) x, -y)
    });
    fp* o = reinterpret_cast<fp*>(&Sg[g]); o[role] = acc.x.c; o[2 + role] = acc.y.c; o[4 + role] = acc.z.c;
  });
}
#ifndef HB_SMEM_F
#define HB_SMEM_F 0       // 1: keep each lane's Fp12 accumulator in dynamic shared memory (experiment, not faster)
#endif
#define HB_SMEM_F_WORDS 73
// lane pair per group: (G + 1)-pair Miller loop, final exponentiation, verdict
template <int G> __global__ void __launch_bounds__(HB_TPB_SPLIT, HB_MINBLOCKS_SPLIT) k_rlc_pairing_split(size_t ngroups, const g1a* pk_scaled_neg, const g2a* hm, const g2a* Sg,
                                 const uint8_t* bad, uint8_t* group_ok) {
    const int role = threadIdx.x & 1;
    const size_t ppg = HB_STRIDE >> 1;
    __shared__ g1a gen_sh;
    if (threadIdx.x == 0) { fp_set(gen_sh.x, K_G1_X); fp_set(gen_sh.y, K_G1_Y); }
    __syncthreads();
    for (size_t it = 0; ; it++) {
        const size_t warp_first = it * ppg + ((HB_TID & ~(size_t)31) >> 1);
        if (warp_first >= ngroups) break;
        const size_t g = it * ppg + (HB_TID >> 1);
        const bool valid = g < ngroups;
        const size_t gg = valid ? g : ngroups - 1;
        const g1a* ps[G + 1]; fp2h qx[G + 1], qy[G + 1];
        bool anybad = false;
        for (int k = 0; k < G; k++) {
            const size_t j = (size_t)k * ngroups + gg;
            ps[k] = &pk_scaled_neg[j];
            const fp* h4 = reinterpret_cast<const fp*>(&hm[j]);
            qx[k].c = h4[role]; qy[k].c = h4[2 + role];
            anybad |= bad[j] != 0;
        }
        ps[G] = &gen_sh;
        const fp* s4 = reinterpret_cast<const fp*>(&Sg[gg]);
        qx[G].c = s4[role]; qy[G].c = s4[2 + role];
#if HB_SMEM_F
        // the Miller accumulator / exponentiation value of this lane in shared memory (73-word stride: conflict-free), not on the stack
        extern __shared__ uint32_t hb_dyn_smem[];
        fp12_t<fp2h>& m = *reinterpret_cast<fp12_t<fp2h>*>(hb_dyn_smem + (size_t)threadIdx.x * HB_SMEM_F_WORDS);
#else
        fp12_t<fp2h> m;
#endif
        miller_loop_multi<fp2h, G + 1>(m, ps, qx, qy);
        final_exp(m, m);
        const bool one = fp12_is_one(m);
        if (valid && role == 0) group_ok[g] = (one && !anybad) ? 1 : 0;
    }
}
// ---- the same check in TWO kernels (hbls.cu "rlc_two_phase").  The fused kernel above keeps G + 1 running points, the Fp12 accumulator
// and their temporaries per lane pair (4.5 KB of local memory per thread: 340 MB per launch, far more than L2, so it streams from DRAM).
// Here the running points live in their OWN kernel: k_rlc_lines_split walks ONE pair (P, Q) per lane pair through the 63 doubling and
// 5 addition steps and writes the 68 line functions, already evaluated at P, to HBM (3 Fp2 per step: 19.6 KB per pair, read once);
// k_rlc_accum_split keeps only the accumulator: f <- f^2 * prod_k line_k per iteration, then the final exponentiation.
// Line layout: fp index ((step * 3 + c) * npairs + p) * 2 + role, p = k * ngroups + g: a warp's 32 lanes touch 1.5 KB contiguously.
#define HB_ML_STEPS 68                 // 63 doublings + 5 additions (bits 62, 60, 57, 48, 16 of |z|)
// the lines are written once and read once: streaming (evict-first) accesses keep them from pushing the kernels' own temporaries
// (local memory, which lives in L1 / L2) out of L2.  fp = 48 bytes at 16-byte aligned offsets: three 128-bit accesses.
HB_DEV void line_store(fp* dst, const fp& v) {
#ifdef HB_HOST_EMU
    *dst = v;
#else
    uint4* d = reinterpret_cast<uint4*>(dst);
    __stcs(d, make_uint4(v.l[0], v.l[1], v.l[2], v.l[3])); __stcs(d + 1, make_uint4(v.l[4], v.l[5], v.l[6], v.l[7])); __stcs(d + 2, make_uint4(v.l[8], v.l[9], v.l[10], v.l[11]));
#endif
}
HB_DEV void line_load(fp& v, const fp* src) {
#ifdef HB_HOST_EMU
    v = *src;
#else
    const uint4* s = reinterpret_cast<const uint4*>(src);
    const uint4 a = __ldcs(s), b = __ldcs(s + 1), c = __ldcs(s + 2);
    v.l[0] = a.x; v.l[1] = a.y; v.l[2] = a.z; v.l[3] = a.w; v.l[4] = b.x; v.l[5] = b.y; v.l[6] = b.z; v.l[7] = b.w; v.l[8] = c.x; v.l[9] = c.y; v.l[10] = c.z; v.l[11] = c.w;
#endif
}
// BLK (blocks, hbls.cu rlc_blocks): only the G round pairs; the block check adds ONE pair (B, sum of the block's Sg).  A compile-time
// choice, so the group form's kernels compile as they did without blocks.
template <int G, bool BLK> HB_DEV void rlc_lines_body(size_t ngtot, size_t g0, size_t ngroups, const g1a* pk_scaled_neg, const g2a* hm,
                                                     const g2a* Sg, fp* lines, const unsigned* count) {
    // groups g0 .. g0 + ngroups - 1 of ngtot (a chunk: the line buffer is sized for hbls.cu rlc_chunk_groups()); round of (k, g) = k * ngtot + g
    // count (nullable): the number of groups is only known on the device (compacted list of the failed groups' rounds; 0: nothing to do)
    if (count) { const size_t n = *count; if (g0 >= n) return; ngtot = n; ngroups = n - g0 < ngroups ? n - g0 : ngroups; }
    const int role = threadIdx.x & 1;
    const size_t ppg = HB_STRIDE >> 1, npairs = (size_t)(BLK ? G : G + 1) * ngroups;
    for (size_t it = 0; ; it++) {
        const size_t warp_first = it * ppg + ((HB_TID & ~(size_t)31) >> 1);
        if (warp_first >= npairs) break;
        const size_t p = it * ppg + (HB_TID >> 1);
        const bool valid = p < npairs;
        const size_t pp = valid ? p : npairs - 1, k = pp / ngroups, g = pp - k * ngroups;
        g1a P; const fp* q4;
        if (BLK || k < (size_t)G) { P = pk_scaled_neg[k * ngtot + g0 + g]; q4 = reinterpret_cast<const fp*>(&hm[k * ngtot + g0 + g]); }
        else { fp_set(P.x, K_G1_X); fp_set(P.y, K_G1_Y); q4 = reinterpret_cast<const fp*>(&Sg[g0 + g]); }
        fp2h qx, qy; qx.c = q4[role]; qy.c = q4[2 + role];
        g2proj_t<fp2h> T; T.x = qx; T.y = qy; fp2_one(T.z);
        fp2h l0, l2, l3;
        size_t st = 0;
        for (int i = 62; i >= 0; i--) {
#ifndef HB_LINES_SYNC
#define HB_LINES_SYNC 1
#endif
            if (HB_LINES_SYNC) hb_lockstep<fp2h>();
            ml_dbl(T, l0, l2, l3); fp2_mul_fp(l2, l2, P.x); fp2_mul_fp(l3, l3, P.y);
            if (valid) { fp* o = lines + ((st * 3) * npairs + pp) * 2 + role; line_store(o, l0.c); line_store(o + 2 * npairs, l2.c); line_store(o + 4 * npairs, l3.c); }
            st++;
            if ((K_Z_ABS >> i) & 1) {
                ml_add(T, qx, qy, l0, l2, l3); fp2_mul_fp(l2, l2, P.x); fp2_mul_fp(l3, l3, P.y);
                if (valid) { fp* o = lines + ((st * 3) * npairs + pp) * 2 + role; line_store(o, l0.c); line_store(o + 2 * npairs, l2.c); line_store(o + 4 * npairs, l3.c); }
                st++;
            }
        }
    }
}
template <int G> __global__ void __launch_bounds__(HB_TPB_SPLIT, HB_MINBLOCKS_SPLIT) k_rlc_lines_split(size_t ngtot, size_t g0, size_t ngroups, const g1a* pk_scaled_neg, const g2a* hm,
                                 const g2a* Sg, fp* lines, const unsigned* count = nullptr) {
    rlc_lines_body<G, false>(ngtot, g0, ngroups, pk_scaled_neg, hm, Sg, lines, count);
}
template <int G> __global__ void __launch_bounds__(HB_TPB_SPLIT, HB_MINBLOCKS_SPLIT) k_rlc_lines_blk(size_t ngtot, size_t g0, size_t ngroups, const g1a* pk_scaled_neg, const g2a* hm,
                                 fp* lines, const unsigned* count = nullptr) {
    rlc_lines_body<G, true>(ngtot, g0, ngroups, pk_scaled_neg, hm, nullptr, lines, count);
}
// BLK: the G round pairs only; the group's Miller value goes to fm (6 Fp2 per group, tower order) and group_ok gets "no bad round" --
// the final exponentiation is the block check's (k_rlc_block_coop), or that of the per-group check (k_rlc_group_check_list)
template <int G, bool BLK> HB_DEV void rlc_accum_body(size_t ngtot, size_t g0, size_t ngroups, const fp* lines, const uint8_t* bad, uint8_t* group_ok,
                                                     const unsigned* count, fp2* fm) {
    if (count) { const size_t n = *count; if (g0 >= n) return; ngtot = n; ngroups = n - g0 < ngroups ? n - g0 : ngroups; }
    const int role = threadIdx.x & 1;
    constexpr int klast = BLK ? G - 1 : G;                              // last pair of a step: the generator pair, unless blocks
    const size_t ppg = HB_STRIDE >> 1, npairs = (size_t)(klast + 1) * ngroups;
    for (size_t it = 0; ; it++) {
        const size_t warp_first = it * ppg + ((HB_TID & ~(size_t)31) >> 1);
        if (warp_first >= ngroups) break;
        const size_t g = it * ppg + (HB_TID >> 1);
        const bool valid = g < ngroups;
        const size_t gg = valid ? g : ngroups - 1;
        bool anybad = false;
        for (int k = 0; k < G; k++) anybad |= bad[(size_t)k * ngtot + g0 + gg] != 0;
        fp12_t<fp2h> m; fp12_one(m);
        size_t st = 0;
#ifndef HB_LINE_PAIRS
#define HB_LINE_PAIRS 0          // 1: lines are multiplied two by two before they touch the accumulator (23 instead of 26 Fp2 products):
#endif                           // measured slower: the extra temporaries cost more than the 10 % fewer products save
#ifndef HB_ACCUM_SYNC
#define HB_ACCUM_SYNC 0          // CTA re-alignment every this many lines inside an iteration (0: only once per iteration, the fastest
                                 // measured; -1: never)
#endif
        auto mul_lines = [&](size_t step) {
            const fp* base = lines + ((step * 3) * npairs + gg) * 2 + role;
#pragma unroll 1
            for (int k = 0; k <= klast; k += HB_LINE_PAIRS ? 2 : 1) {
                if (HB_ACCUM_SYNC > 0 && G > 4 && (k % (HB_ACCUM_SYNC > 0 ? HB_ACCUM_SYNC : 1)) == 0 && k) hb_lockstep<fp2h>();
                const fp* o = base + (size_t)k * ngroups * 2;
                fp2h l0, l2, l3; line_load(l0.c, o); line_load(l2.c, o + 2 * npairs); line_load(l3.c, o + 4 * npairs);
                if (HB_LINE_PAIRS && k + 1 <= klast) {
                    const fp* o2 = o + ngroups * 2;
                    fp2h n0, n2, n3; line_load(n0.c, o2); line_load(n2.c, o2 + 2 * npairs); line_load(n3.c, o2 + 4 * npairs);
                    fp12_mul_by_two_lines(m, m, l0, l2, l3, n0, n2, n3);
                } else
                    fp12_mul_by_014(m, m, l0, l2, l3);
            }
        };
        for (int i = 62; i >= 0; i--) {
            if (HB_ACCUM_SYNC >= 0) hb_lockstep<fp2h>();
            fp12_sqr(m, m);
            mul_lines(st++);
            if ((K_Z_ABS >> i) & 1) mul_lines(st++);
        }
        if (BLK) {
            if (valid) {
                fp* o = reinterpret_cast<fp*>(fm + 6 * (g0 + g)) + role;
                const fp2h* mc = reinterpret_cast<const fp2h*>(&m);
                for (int t = 0; t < 6; t++) o[2 * t] = mc[t].c;
                if (role == 0) group_ok[g0 + g] = anybad ? 0 : 1;
            }
            continue;
        }
        final_exp(m, m);
        const bool one = fp12_is_one(m);
        if (valid && role == 0) group_ok[g0 + g] = (one && !anybad) ? 1 : 0;
    }
}
template <int G> __global__ void __launch_bounds__(HB_TPB_SPLIT, HB_MINBLOCKS_SPLIT) k_rlc_accum_split(size_t ngtot, size_t g0, size_t ngroups, const fp* lines, const uint8_t* bad, uint8_t* group_ok,
                                 const unsigned* count = nullptr) {
    rlc_accum_body<G, false>(ngtot, g0, ngroups, lines, bad, group_ok, count, nullptr);
}
template <int G> __global__ void __launch_bounds__(HB_TPB_SPLIT, HB_MINBLOCKS_SPLIT) k_rlc_accum_blk(size_t ngtot, size_t g0, size_t ngroups, const fp* lines, const uint8_t* bad, uint8_t* group_ok,
                                 fp2* fm, const unsigned* count = nullptr) {
    rlc_accum_body<G, true>(ngtot, g0, ngroups, lines, bad, group_ok, count, fm);
}
// ---- blocks of HB_RLC_M groups: one final exponentiation and one generator pair per block (hbls.cu rlc_blocks).
// Per block b: Sb = sum of the Sg of its members (groups b, b + S, ...), affine
// gate (nullable, every block kernel): the block form runs only while *gate != 0 (hbls.cu: k_rlc_form picks the form on the device)
__global__ void k_rlc_block_sum(size_t S, size_t ng, const g2a* Sg, g2a* Sb, const unsigned* gate = nullptr) {
  if (gate && *gate == 0) return;
  for (size_t b = HB_TID; b < S; b += HB_STRIDE) {
    g2 acc; pt_set_inf(acc);
    for (size_t g = b; g < ng; g += S) { const g2a q = Sg[g]; pt_add_mixed(acc, acc, q); }
    g2a a; pt_to_aff(a, acc); Sb[b] = a;
  }
}
// the block check, ONE WARP per block (vm.cuh): FE( prod_m fm[member m] * Miller(B, Sb) ) == 1 and no member holds a bad round
// (group_ok = "no bad round" from k_rlc_accum_split).  An identity Sb proves nothing: the block fails and its groups are checked alone.
__global__ void __launch_bounds__(32) k_rlc_block_coop(size_t S, size_t ng, const fp2* fm, const g2a* Sb, const uint8_t* group_ok, uint8_t* block_ok,
                                                       const unsigned* gate = nullptr) {
    if (gate && *gate == 0) return;
    __shared__ uint32_t slots[VM_SMEM_WORDS];
    const int lane = threadIdx.x & 31;
    vm_load_consts(slots);
    for (size_t b = blockIdx.x; b < S; b += gridDim.x) {
        bool clean = true;
        for (size_t g = b; g < ng; g += S) clean &= group_ok[g] != 0;
        if (!clean) { if (lane == 0) block_ok[b] = 0; __syncwarp(); continue; }      // warp-uniform
        vm_run(VM_P_A_ONE, slots);
        for (size_t g = b; g < ng; g += S) {
            if (lane < 12) vm_st(slots, VM_R_F0 + (lane >> 1), lane & 1, reinterpret_cast<const fp*>(&fm[6 * g + (lane >> 1)])[lane & 1].l);
            __syncwarp();
            vm_run(VM_P_AMULF, slots);
        }
        bool zero = true;
        if (lane < 4) {
            fp2 v; fp2_zero(v);
            if (lane == 0) fp_set(v.a, K_G1_X); else if (lane == 1) fp_set(v.a, K_G1_Y); else if (lane == 2) v = Sb[b].x; else v = Sb[b].y;
            vm_set_fp2(slots, VM_R_P2X + lane, v);
            zero = fp_is_zero(v.a) & fp_is_zero(v.b);
        }
        const unsigned zmask = __ballot_sync(0xffffffffu, zero);
        bool one = false;
        if ((zmask & 0xc) != 0xc) {
            vm_run(VM_P_ML1_INIT, slots);
            for (int i = 62; i >= 0; i--) {
                vm_run(VM_P_ML1_DBL, slots);
                if ((K_Z_ABS >> i) & 1) vm_run(VM_P_ML1_ADD, slots);
            }
            vm_run(VM_P_FMULA, slots);
            one = vm_final_exp_is_one(slots);
        }
        if (lane == 0) block_ok[b] = one ? 1 : 0;
        __syncwarp();
    }
}
// groups of the blocks that failed: compacted into list (count on the device) for k_rlc_group_check_list.  A group of a proven block
// keeps group_ok = 1; a group holding a bad round keeps 0 and needs no check of its own.
__global__ void k_rlc_block_list(size_t ng, size_t S, const uint8_t* block_ok, uint8_t* group_ok, uint32_t* list, unsigned* count,
                                 const unsigned* gate = nullptr) {
    const size_t g = HB_TID; if (g >= ng || (gate && *gate == 0)) return;
    if (block_ok[g % S] || !group_ok[g]) return;
    group_ok[g] = 0;
    list[atomicAdd(count, 1u)] = (uint32_t)g;
}
// lane pair per listed group: group_ok = FE( fm[g] * Miller(B, Sg[g]) ) == 1 -- the per-group check of k_rlc_accum_split without blocks
__global__ void __launch_bounds__(HB_TPB_SPLIT, HB_MINBLOCKS_SPLIT) k_rlc_group_check_list(const unsigned* count, const uint32_t* list, const fp2* fm,
                                                                                         const g2a* Sg, uint8_t* group_ok) {
    const size_t n = *count;
    if (n == 0) return;
    const int role = threadIdx.x & 1;
    // lane pair q of CTA c takes item q * gridDim.x + c: a list shorter than the grid still gives every CTA (one per SM) its share,
    // in its first warps, and the rest of the CTA's warps leave at once
    const size_t qpc = blockDim.x >> 1;
    __shared__ g1a gen_sh;
    if (threadIdx.x == 0) { fp_set(gen_sh.x, K_G1_X); fp_set(gen_sh.y, K_G1_Y); }
    __syncthreads();
    for (size_t it = 0; ; it++) {
        const size_t warp_first = (it * qpc + ((threadIdx.x & ~31u) >> 1)) * gridDim.x + blockIdx.x;
        if (warp_first >= n) break;
        const size_t i = (it * qpc + (threadIdx.x >> 1)) * gridDim.x + blockIdx.x;
        const bool valid = i < n;
        const size_t g = list[valid ? i : n - 1];
        const fp* s4 = reinterpret_cast<const fp*>(&Sg[g]);
        fp2h qx[1], qy[1]; qx[0].c = s4[role]; qy[0].c = s4[2 + role];
        const bool zx = fp2_is_zero(qx[0]), zy = fp2_is_zero(qy[0]);     // no short-circuit: fp2_is_zero(fp2h) shuffles across the warp
        const g1a* ps[1] = {&gen_sh};
        fp12_t<fp2h> m, f;
        miller_loop_multi<fp2h, 1>(m, ps, qx, qy);
        const fp* src = reinterpret_cast<const fp*>(fm + 6 * g) + role;
        fp2h* fc = reinterpret_cast<fp2h*>(&f);
        for (int t = 0; t < 6; t++) fc[t].c = src[2 * t];
        fp12_mul(m, m, f);
        final_exp(m, m);
        const bool one = fp12_is_one(m);
        if (valid && role == 0) group_ok[g] = (one && !(zx & zy)) ? 1 : 0;
    }
}
// which form a call that can use blocks takes.  Calls are asynchronous (the host does not know how the previous one ended), so the
// choice is made on the device: *form = 1 when the last such call had at least one failed group in 64 (k_rlc_form_update).  Then most
// blocks would fail and the per-group check of their groups -- a Miller loop and a final exponentiation per group at partial occupancy --
// costs more than the blocks save, so the groups are checked one by one.  gates[0] = ng runs the group form's kernels (their count),
// gates[1] = ng the block form's; the other is 0.  force_blocks: hbls_set_param("rlc_block", 1).
__global__ void k_rlc_form(size_t ng, int force_blocks, const int* form, unsigned* gates) {
    if (HB_TID != 0) return;
    const bool groups = !force_blocks && *form != 0;
    gates[0] = groups ? (unsigned)ng : 0u; gates[1] = groups ? 0u : (unsigned)ng;
}
__global__ void k_rlc_form_update(size_t ng, const unsigned* counts, int* form) {
    if (HB_TID != 0) return;
    *form = 64 * (size_t)counts[1] >= ng ? 1 : 0;
}
// ---- the EXACT check through the same two kernels: a "group" of ONE round = the pairs (-apk_j, H(m_j)) and (B, sigma_j), i.e.
// k_rlc_lines_split<1> / k_rlc_accum_split<1> with pk_scaled_neg = -apk (affine) and Sg = the decoded signatures.  These two small
// kernels prepare the flags (a round with an identity operand is left to k_pairing_fixup: 0xFF, as in k_pairing_verify_split)
// and publish the verdicts.  idx (nullable): the rounds are those of a compacted list (failed groups of the batched form).
__global__ void k_exact_prepare(size_t n, const uint32_t* idx, const g2a* sig, const g1a* pk_neg, const g2a* hm, const uint8_t* ok_a, const uint8_t* ok_b,
                                const uint8_t* ok_c, g1a* pk_c, g2a* hm_c, g2a* sig_c, uint8_t* bad, uint8_t* results, const unsigned* count = nullptr) {
    if (count) n = *count;
    const size_t t = HB_TID; if (t >= n) return;
    const size_t j = idx ? idx[t] : t;
    const g2a s = sig[j], h = hm[j]; const g1a p = pk_neg[j];
    const bool good = (!ok_a || ok_a[j]) && (!ok_b || ok_b[j]) && (!ok_c || ok_c[j]);
    const bool irregular = aff_is_inf(s) || aff_is_inf(h) || aff_is_inf(p);
    bad[t] = (!good || irregular) ? 1 : 0;
    if (pk_c) { pk_c[t] = p; hm_c[t] = h; sig_c[t] = s; }               // gathered copies (list form)
    results[j] = irregular ? 0xFF : 0;
}
__global__ void k_exact_publish(size_t n, const uint32_t* idx, const uint8_t* verdict, uint8_t* results, const unsigned* count = nullptr) {
    if (count) n = *count;
    const size_t t = HB_TID; if (t >= n) return;
    const size_t j = idx ? idx[t] : t;
    if (results[j] != 0xFF) results[j] = verdict[t];
}
// verdicts of the groups -> per-round results; the rounds of failed groups are compacted into `list` for the exact pass.
// counts[0] = rounds listed, counts[1] = groups that failed (hbls_last_batch_info)
__global__ void k_rlc_finish(size_t nrounds, size_t ngroups, const uint8_t* group_ok, uint8_t* results, uint32_t* list, unsigned* counts) {
    size_t j = HB_TID; if (j >= nrounds) return;
    const uint8_t ok = group_ok[j % ngroups];
    results[j] = ok;
    if (!ok) {
        list[atomicAdd(&counts[0], 1u)] = (uint32_t)j;
        if (j < ngroups) atomicAdd(&counts[1], 1u);
    }
}
__global__ void k_g1_normalize_list(const unsigned* count, const uint32_t* list, const g1* in, g1a* out, int negate) {
  const size_t n = *count;
  for (size_t i = HB_TID; i < n; i += HB_STRIDE) {
    const size_t j = list[i];
    g1 p = in[j]; g1a a; pt_to_aff(a, p);
    if (negate) fp_neg(a.y, a.y);
    out[j] = a;
  }
}
// k_pairing_verify_split over the listed rounds only (same body, indirect round index)
__global__ void __launch_bounds__(HB_TPB_SPLIT, HB_MINBLOCKS_SPLIT) k_pairing_verify_split_list(const unsigned* count, const uint32_t* list, const g2a* sig, const g1a* pk_neg,
                                 const g2a* hm, const uint8_t* ok_a, const uint8_t* ok_b, const uint8_t* ok_c, uint8_t* results) {
    const size_t B = *count;
    if (B == 0) return;
    const int role = threadIdx.x & 1;
    const size_t ppg = HB_STRIDE >> 1;
    for (size_t it = 0; ; it++) {
        const size_t warp_first = it * ppg + ((HB_TID & ~(size_t)31) >> 1);
        if (warp_first >= B) break;
        const size_t i = it * ppg + (HB_TID >> 1);
        const bool valid = i < B;
        const size_t jj = list[valid ? i : B - 1];
        bool good = (!ok_a || ok_a[jj]) && (!ok_b || ok_b[jj]) && (!ok_c || ok_c[jj]);
        g1a gen, p2 = pk_neg[jj];
        fp_set(gen.x, K_G1_X); fp_set(gen.y, K_G1_Y);
        const fp* s4 = reinterpret_cast<const fp*>(&sig[jj]);
        const fp* h4 = reinterpret_cast<const fp*>(&hm[jj]);
        fp2h q1x, q1y, q2x, q2y;
        q1x.c = s4[role]; q1y.c = s4[2 + role]; q2x.c = h4[role]; q2y.c = h4[2 + role];
        const bool z1x = fp2_is_zero(q1x), z1y = fp2_is_zero(q1y), z2x = fp2_is_zero(q2x), z2y = fp2_is_zero(q2y);
        const bool irregular = (z1x & z1y) | (z2x & z2y) | (fp_is_zero(p2.x) & fp_is_zero(p2.y));
        fp12_t<fp2h> m;
        miller_loop2<fp2h>(m, gen, q1x, q1y, p2, q2x, q2y, true, true);
        final_exp(m, m);
        const bool one = fp12_is_one(m);
        if (valid && role == 0) results[jj] = irregular ? 0xFF : ((good && one) ? 1 : 0);
    }
}
__global__ void k_pairing_fixup_list(const unsigned* count, const uint32_t* list, const g2a* sig, const g1a* pk_neg, const g2a* hm,
                                     const uint8_t* ok_a, const uint8_t* ok_b, const uint8_t* ok_c, uint8_t* results) {
  const size_t n = *count;
  for (size_t i = HB_TID; i < n; i += HB_STRIDE) {
    const size_t j = list[i];
    if (results[j] != 0xFF) continue;
    bool good = (!ok_a || ok_a[j]) && (!ok_b || ok_b[j]) && (!ok_c || ok_c[j]);
    g1a gen, p2 = pk_neg[j]; g2a q1 = sig[j], q2 = hm[j];
    fp_set(gen.x, K_G1_X); fp_set(gen.y, K_G1_Y);
    results[j] = (good && verify_irregular(gen, q1, p2, q2)) ? 1 : 0;
  }
}
// headers / items callers want to tell "signature bytes do not decode" from "pairing check failed" (engine.go:630-640 returns
// different errors): flags[j] bit0 = signature decoded, bit1 = message mapped to a point, bit2 = public key decoded
__global__ void k_pack_flags(size_t n, const uint8_t* ok_sig, const uint8_t* ok_hm, const uint8_t* ok_pk, uint8_t* flags) {
    size_t j = HB_TID; if (j >= n) return;
    flags[j] = (ok_sig[j] ? 1 : 0) | (ok_hm[j] ? 2 : 0) | ((!ok_pk || ok_pk[j]) ? 4 : 0);
}

// device self-test of the lane-pair Fp2 primitives against the single-thread ones on pseudo-random operands
__global__ void k_selftest_fp2h(uint32_t n, uint32_t seed, uint32_t* mismatches) {
    const int role = threadIdx.x & 1;
    for (uint32_t it = 0; it < n; it++) {
        uint32_t st = seed + 7919u * (uint32_t)(HB_TID >> 1) + 104729u * it;
        fp2 x, y;
        uint32_t* w[4] = {x.a.l, x.b.l, y.a.l, y.b.l};
        for (int c = 0; c < 4; c++) { for (int k = 0; k < 12; k++) { st = st * 1664525u + 1013904223u; w[c][k] = st ^ (st >> 13); } w[c][11] &= 0x0fffffffu; }
        fp2h hx, hy, hr; hx.c = role ? x.b : x.a; hy.c = role ? y.b : y.a;
        fp2 r; uint32_t bad = 0;
#define HB_CHK() do { const fp& e = role ? r.b : r.a; if (!fp_eq(e, hr.c)) bad++; } while (0)
        fp2_mul(r, x, y); fp2_mul(hr, hx, hy); HB_CHK();
        fp2_sqr(r, x); fp2_sqr(hr, hx); HB_CHK();
        fp2_mul_xi(r, x); fp2_mul_xi(hr, hx); HB_CHK();
        fp2_conj(r, y); fp2_conj(hr, hy); HB_CHK();
        fp2_add(r, x, y); fp2_add(hr, hx, hy); HB_CHK();
        fp2_sub(r, x, y); fp2_sub(hr, hx, hy); HB_CHK();
        fp2_neg(r, x); fp2_neg(hr, hx); HB_CHK();
        fp2_dbl(r, y); fp2_dbl(hr, hy); HB_CHK();
        fp2_mul_fp(r, x, y.a); fp2_mul_fp(hr, hx, y.a); HB_CHK();
        fp2_inv(r, x); fp2_inv(hr, hx); HB_CHK();
        fp2_one(r); fp2_one(hr); HB_CHK();
        fp2_const(r, K_PSI_CX); fp2_const(hr, K_PSI_CX); HB_CHK();
        if (fp2_is_zero(hx) != fp2_is_zero(x)) bad++;
        fp2 z; fp2_zero(z); fp2h hz; fp2_zero(hz); if (!fp2_is_zero(hz)) bad++;
        if (bad) atomicAdd(mismatches, bad);
    }
}

// ---- scalar multiplication batches (R6 sign, R14 GetPublicKey): constant-time ladders (curve.cuh pt_mul_ct, g2_mul_gls_ct).  Branches
// here depend on public data only: the item count, whether H(m) exists.
__global__ void k_g1_mul_gen(size_t n, const uint8_t* sk32, g1* out) {
    size_t i = HB_TID; if (i >= n) return;
    uint32_t k[8]; load_words(k, sk32 + 32 * i, 8);
    g1 g, r; g1_generator(g); pt_mul_ct(r, g, k); out[i] = r;
}
__global__ void k_sign_hash(size_t n, const uint8_t* sk32, const uint8_t* msgs, uint32_t msg_len, g2* out, uint8_t* ok) {
    size_t i = HB_TID; if (i >= n) return;
    uint32_t k[8]; load_words(k, sk32 + 32 * i, 8);
    g2 h, r; bool good = map_to_g2(h, msgs + (size_t)msg_len * i, msg_len);
    if (good) pt_mul_ct(r, h, k); else pt_set_inf(r);
    out[i] = r; ok[i] = good ? 1 : 0;
}
// sigma = sk * H for an already-mapped H(m) (the library's H(m) cache, hbls.cu): one item per LANE PAIR, the 256-bit ladder on the
// split carrier.  hm_stride = 0: every item signs the same point.  Output Jacobian (the layout of blsSignature).
__global__ void k_sign_hm_pair(size_t n, const uint8_t* sk32, const g2a* hm, const uint8_t* ok_hm, size_t hm_stride, g2* out, uint8_t* ok) {
    const size_t i = HB_TID >> 1; if (i >= n) return;
    uint32_t k[8]; load_words(k, sk32 + 32 * i, 8);
    const g2a h = hm[i * hm_stride];
    const bool good = ok_hm[i * hm_stride] != 0 && !aff_is_inf(h);
    jac<fp2h> H, R; fp2h_pack(H.x, h.x); fp2h_pack(H.y, h.y); fp2_one(H.z);
    pt_mul_ct(R, H, k);
    g2 r; fp2h_unpack(r.x, R.x); fp2h_unpack(r.y, R.y); fp2h_unpack(r.z, R.z);
    if (!good) pt_set_inf(r);
    if ((threadIdx.x & 1) == 0) { out[i] = r; ok[i] = good ? 1 : 0; }
}
// The same signature through the psi endomorphism (latency path of blsSignHash): the host writes sk = d0 + d1 Z + d2 Z^2 + d3 Z^3 in
// base Z = |z| (four 64-bit digits: sk < r < Z^4); on G2 psi acts as [z] = [-Z], so  sk H = d0 H - d1 psi(H) + d2 psi^2(H) - d3 psi^3(H)
// is ONE 65-column ladder over an 8-entry table (g2_mul_gls_ct: 65 doublings + 66 additions instead of 252 + 64).
__global__ void k_sign_hm_gls_pair(size_t n, const uint64_t* digits, const g2a* hm, const uint8_t* ok_hm, size_t hm_stride, g2* out, uint8_t* ok) {
    const size_t i = HB_TID >> 1; if (i >= n) return;
    const g2a h = hm[i * hm_stride];
    const bool good = ok_hm[i * hm_stride] != 0 && !aff_is_inf(h);
    aff<fp2h> H; fp2h_pack(H.x, h.x); fp2h_pack(H.y, h.y);
    jac<fp2h> R;
    g2_mul_gls_ct(R, H, digits + 4 * i);
    g2 r; fp2h_unpack(r.x, R.x); fp2h_unpack(r.y, R.y); fp2h_unpack(r.z, R.z);
    if (!good) pt_set_inf(r);
    if ((threadIdx.x & 1) == 0) { out[i] = r; ok[i] = good ? 1 : 0; }
}

// ---- single-element ops behind the herumi-shaped C ABI (one thread per op; latency is launch-bound)
enum { OP_G1_ADD = 1, OP_G1_SUB, OP_G2_ADD, OP_G1_EQ, OP_G2_EQ, OP_G1_SER, OP_G2_SER, OP_G1_DES, OP_G2_DES, OP_MAP_SER, OP_G2_DES_ADD };
// one op: device operands a, b (nullable), result out, message length len (OP_MAP_SER)
struct single_desc { const void* a; const void* b; void* out; int op; uint32_t len; };
HB_DEV void run_single(const single_desc& s, int* rc) {
    const void* a = s.a; const void* b = s.b; void* out = s.out;
    switch (s.op) {
    case OP_G1_ADD: case OP_G1_SUB: {
        g1 x = *(const g1*)a, y = *(const g1*)b; if (s.op == OP_G1_SUB) pt_neg(y, y);
        pt_add(x, x, y); *(g1*)out = x; *rc = 0; break; }
    case OP_G2_ADD: { g2 x = *(const g2*)a, y = *(const g2*)b; pt_add(x, x, y); *(g2*)out = x; *rc = 0; break; }
    case OP_G1_EQ: { g1 x = *(const g1*)a, y = *(const g1*)b; *rc = pt_eq(x, y) ? 1 : 0; break; }
    case OP_G2_EQ: { g2 x = *(const g2*)a, y = *(const g2*)b; *rc = pt_eq(x, y) ? 1 : 0; break; }
    case OP_G1_SER: { g1 x = *(const g1*)a; g1_serialize((uint8_t*)out, x); *rc = 48; break; }
    case OP_G2_SER: { g2 x = *(const g2*)a; g2_serialize((uint8_t*)out, x); *rc = 96; break; }
    case OP_G1_DES: { g1 x; bool g = g1_deserialize(x, (const uint8_t*)a, true); if (g) *(g1*)out = x; *rc = g ? 48 : 0; break; }
    case OP_G2_DES: { g2 x; bool g = g2_deserialize(x, (const uint8_t*)a, true); if (g) *(g2*)out = x; *rc = g ? 96 : 0; break; }
    case OP_MAP_SER: { g2 h; bool g = map_to_g2(h, (const uint8_t*)a, s.len); if (g) g2_serialize((uint8_t*)out, h); *rc = g ? 0 : -1; break; }
    case OP_G2_DES_ADD: {   // ballot box: out (Jacobian running sum) += decode(a); rc = 96 ok / 0 undecodable (sum untouched)
        g2 x; bool g = g2_deserialize(x, (const uint8_t*)a, true);
        if (g) { g2 acc = *(const g2*)out; pt_add(acc, acc, x); *(g2*)out = acc; }
        *rc = g ? 96 : 0; break; }
    default: *rc = -1;
    }
}
// thread i runs op i: ops[i] (device array), or `one` when ops is null (n = 1, nothing to stage); rc[i] its return code
__global__ void k_single(size_t n, const single_desc* ops, single_desc one, int* rc) {
    const size_t i = HB_TID; if (i >= n) return;
    run_single(ops ? ops[i] : one, rc + i);
}

// ---- integer-pipe roofline probe: K independent accumulator sets per thread, each fed by lane_mad -- the exact
// mad.lo.cc / madc.hi.cc chains of the field multiplier (SASS: IMAD.WIDE.U32(.X), 6 per lane_mad).  Round 1 probed two loop
// invariants with a plain mad.wide; ptxas hoisted the product and the loop became IADD3 pairs, so the "18 TMAC32/s" it
// reported was half the ALU add rate.  A 32-bit IMAD issues at 16 lanes per clock per scheduler (64 per SM: the throughput table of
// the CUDA C++ Programming Guide for compute capability 9.0), an IMAD.WIDE takes two of those: 8 wide MACs per clock per scheduler.
// bench.py reports what this probe reaches against that figure (tools/probe_int.cu isolates the instruction mix).
template <int K> __global__ void k_probe_carry(int iters, uint32_t seed, uint32_t* sink, unsigned long long* cycles) {
    uint32_t acc[K][14], a[12];
    uint32_t t = seed ^ (uint32_t)HB_TID;
#pragma unroll
    for (int j = 0; j < 12; j++) { t = t * 1664525u + 1013904223u; a[j] = t; }
#pragma unroll
    for (int k = 0; k < K; k++)
#pragma unroll
        for (int j = 0; j < 14; j++) { t = t * 1664525u + 1013904223u; acc[k][j] = t; }
    const uint32_t b = t | 1u;
    const long long c0 = clock64();
    for (int i = 0; i < iters; i++) {
#pragma unroll
        for (int k = 0; k < K; k++) lane_mad(acc[k], a, b);
    }
    const long long c1 = clock64();
    uint32_t s = 0;
#pragma unroll
    for (int k = 0; k < K; k++)
#pragma unroll
        for (int j = 0; j < 14; j++) s ^= acc[k][j];
    if (s == 0x12345u) sink[0] = s;                // never true in practice: keeps the chains alive
    if (HB_TID == 0) cycles[0] = (unsigned long long)(c1 - c0);
}

}  // namespace hb
