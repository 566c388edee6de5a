// harmony_b200/csrc/hbls.cu -- libhbls.so: C ABI (include/hbls.h) over the sm_90a kernels.
// Host side = plumbing only (buffers, streams, launches); every group/field operation runs on the GPU.
// No CPU fallback exists: without a usable CUDA device blsInit fails and every entry point returns HBLS_ERR_CUDA.
#include <cuda_runtime.h>
#include <algorithm>
#include <atomic>
#include <cstdio>
#include <cstdlib>
#include <array>
#include <cstring>
#include <map>
#include <memory>
#include <mutex>
#include <set>
#include <string>
#include <vector>
#include "../../include/hbls.h"
#include "coalesce.hpp"
#include "kernels.cuh"
#include "device_forms.cuh"

using namespace hb;

struct hbls_committee {
    size_t n = 0;
    g1a* table = nullptr;       // device, affine, Montgomery
    g1* total = nullptr;        // device, sum of all rows (lets dense bitmaps be aggregated from their complement)
    ~hbls_committee() { if (table) cudaFree(table); if (total) cudaFree(total); }
};
struct hbls_mask {
    const hbls_committee* c = nullptr;
    std::vector<uint8_t> bitmap;        // Mask.Bitmap (host)
    g1* d_acc = nullptr;                // Mask.AggregatePublic (device, Jacobian)
    ~hbls_mask() { if (d_acc) cudaFree(d_acc); }
};

namespace {

// per-stream scratch: a bump arena + the timing events and the pinned counters of the last batch issued on that stream.
// Calls on one stream are stream-ordered, so re-using its arena from offset 0 is safe; different streams never share one.
struct Scratch {
    uint8_t* base = nullptr; size_t cap = 0;
    cudaEvent_t ev[8] = {}; bool ev_ok = false, ev7_set = false;
    unsigned* h_counts = nullptr;            // pinned: [0] rounds re-verified exactly, [1] groups failed
    cudaEvent_t done = nullptr;
    cudaEvent_t fork = nullptr, join[2] = {}; bool forked = false;      // small batches: decode / hash on two auxiliary streams
    cudaEvent_t mid = nullptr, join2 = nullptr;                          // H(m) cached: "signature decoded" / "subgroup test done"
    // device items form: the mask_item descriptors built on the host, pinned; `items_copied` is recorded after their upload, and the
    // next call on this stream waits for it before it rewrites the buffer
    mask_item* h_items = nullptr; size_t h_items_cap = 0; cudaEvent_t items_copied = nullptr; bool items_pending = false;
};
struct Ctx {
    bool ready = false;
    int device = 0;
    int sm_count = 132;
    cudaStream_t stream = nullptr;
    cudaStream_t aux[2] = {nullptr, nullptr};               // latency path: signature decode and hash-to-G2 run beside the mask aggregation
    std::mutex mu;
    std::map<cudaStream_t, Scratch> scratch;
    std::atomic<uint64_t> launches{0};
    bool stage_timing = false; Scratch* stage_sc = nullptr;
    int batch_mode = 1;                                     // 1: random-linear-combination groups + exact pass over failed groups, 0: exact per round
    // tuning (hbls_set_param)
    long long rlc_min = 12288, rlc_g = 0, tpsm = 384, tpsm_split = 512, tpsm_light = 1024, coop_max = 4096, overlap = 1, coop_wpsm = 14, hash_coop_max = 528, mask_sort = 1, hash_split = 2, tpsm_sw = 512, hash_fallback = 0, rlc_two_phase = 2, tpsm_lines = 512, tpsm_accum = 512, tpsm_cof = 512, tpsm_dec = 512, tpsm_sub = 512, tpsm_scale = 384, tpsm_scale_g2 = 512, tpsm_scale_g1 = 384, scale_split = 1, decode_split = 1, exact_two_phase = 1;
    int* rlc_form = nullptr;                                // device: 1 = the last call that could use blocks had many failed groups (k_rlc_form)
    long long rlc_block = 0;                                // blocks of HB_RLC_M groups (rlc_blocks): 0 automatic, 1 forced on, 2 forced off
    long long scale_joint = 1;                              // signature scaling: 0 a ladder per round + group sums, 1 one joint ladder per group
                                                            // once the groups fill the chip, 2 always the joint ladder
    // coefficient stream: ChaCha20 keyed from /dev/urandom, block counter = call number
    uint32_t chacha_key[8] = {}; uint64_t rlc_calls = 0;
    // last batch
    hbls_batch_info info = {}; Scratch* info_sc = nullptr; bool info_valid = false;
    // last error of a call that cannot return one
    int last_err = 0; char last_err_msg[160] = {};
    // H(m) cache (device-resident, LRU): the messages a node hashes again and again -- the block hash / commit payload it SIGNS
    // itself (consensus/validator.go: prepare / commit votes) and then VERIFIES in PREPARED / COMMITTED (validator.go:219-236,
    // engine.go:630-640), the one message of a leader's vote collection (leader.go:127-290).  Keyed by the 48 zero-padded bytes
    // hash_to_fp reads (A.3: longer inputs are truncated).  Mirrors the reference's own caches on this path (BLSPubKeyCache LRU,
    // crypto/bls/mask.go:35-55; epochCtx committee cache, engine.go:727-761).
    struct HmEntry { uint8_t key[48] = {}; uint64_t stamp = 0; bool used = false, has_reader = false; cudaEvent_t filled = nullptr, read_done = nullptr; };
    static constexpr int HM_N = 64;
    g2a* hm_slots = nullptr; uint8_t* hm_ok = nullptr; HmEntry hm[HM_N];
    uint64_t hm_clock = 0, hm_hits = 0, hm_misses = 0;
    long long hm_cache = 1;                                 // hbls_set_param("hm_cache", 0) turns it off (cold-path measurements)
    hbls_coalesce::Combiner part1;                          // concurrent herumi-API calls (include/hbls.h part 1) -> shared turns
    // built-in self-test (selftest.cuh): kernels launched by the last run, a failed run at init disables the library
    bool st_rec = false, st_failed = false; std::set<std::string> st_kernels;
    long long selftest_flip = 0;                            // test hook: leg + 1 whose expected answer the next run flips
};
Ctx g;

void note_error(cudaError_t e, const char* what, const char* file, int line) {
    fprintf(stderr, "[hbls] CUDA error %s at %s:%d: %s\n", what, file, line, cudaGetErrorString(e));
    g.last_err = (int)e;
    snprintf(g.last_err_msg, sizeof g.last_err_msg, "%s: %s", what, cudaGetErrorString(e));
}
#define CK(call) do { cudaError_t e_ = (call); if (e_ != cudaSuccess) { note_error(e_, #call, __FILE__, __LINE__); return HBLS_ERR_CUDA; } } while (0)

int ensure_init() {
    if (g.st_failed) { fprintf(stderr, "[hbls] the self-test failed at initialisation: the library refuses all work\n"); return HBLS_ERR_SELF_TEST; }
    if (g.ready) return 0;
    fprintf(stderr, "[hbls] not initialised: call blsInit / hbls_init_device first (no CPU fallback)\n");
    return HBLS_ERR_CUDA;
}

struct Arena {
    uint8_t* base; size_t off = 0, cap;
    template <class T> T* take(size_t n) {
        off = (off + 255) & ~(size_t)255;
        T* p = reinterpret_cast<T*>(base + off); off += n * sizeof(T);
        return p;
    }
};
// scratch of stream s, grown to `bytes` (growing frees the old block: cudaFree waits for the device, so no kernel still reads it)
int reserve(cudaStream_t s, size_t bytes, Scratch** out) {
    Scratch& sc = g.scratch[s];
    bytes += 4096;
    if (bytes > sc.cap) {
        if (sc.base) CK(cudaFree(sc.base));
        sc.base = nullptr; sc.cap = 0;
        size_t cap = bytes + bytes / 4;
        CK(cudaMalloc(&sc.base, cap));
        sc.cap = cap;
    }
    if (!sc.h_counts) {
        CK(cudaMallocHost(&sc.h_counts, 64)); sc.h_counts[0] = sc.h_counts[1] = 0;
        CK(cudaEventCreateWithFlags(&sc.done, cudaEventDisableTiming)); CK(cudaEventCreateWithFlags(&sc.fork, cudaEventDisableTiming));
        CK(cudaEventCreateWithFlags(&sc.join[0], cudaEventDisableTiming)); CK(cudaEventCreateWithFlags(&sc.join[1], cudaEventDisableTiming));
        CK(cudaEventCreateWithFlags(&sc.mid, cudaEventDisableTiming)); CK(cudaEventCreateWithFlags(&sc.join2, cudaEventDisableTiming));
    }
    sc.forked = false; sc.ev7_set = false;
    *out = &sc;
    return 0;
}
inline unsigned blocks_for(size_t n, unsigned tpb) { return (unsigned)((n + tpb - 1) / tpb); }

// ------------------------------------------------------------------ H(m) cache.  Caller holds g.mu.  Entries are filled and read on
// whatever stream the call runs on; `filled` orders readers after the fill, `read_done` orders a later overwrite after the readers.
void hm_key(uint8_t key[48], const void* msg, size_t len) { memset(key, 0, 48); if (len) memcpy(key, msg, len > 48 ? 48 : len); }
bool hm_enabled() { return g.hm_cache != 0 && g.hm_slots != nullptr; }
// the cache slot holding key, or -1
int hm_find(const uint8_t key[48]) {
    for (int i = 0; i < Ctx::HM_N; i++) if (g.hm[i].used && memcmp(g.hm[i].key, key, 48) == 0) return i;
    return -1;
}
// hit: stream st copies the cached point into dst / dst_ok and true is returned
bool hm_fetch(const uint8_t key[48], g2a* dst, uint8_t* dst_ok, cudaStream_t st) {
    const int i = hm_find(key);
    if (i < 0) { g.hm_misses++; return false; }
    Ctx::HmEntry& e = g.hm[i];
    cudaStreamWaitEvent(st, e.filled, 0);
    cudaMemcpyAsync(dst, g.hm_slots + i, sizeof(g2a), cudaMemcpyDeviceToDevice, st);
    cudaMemcpyAsync(dst_ok, g.hm_ok + i, 1, cudaMemcpyDeviceToDevice, st);
    cudaEventRecord(e.read_done, st); e.has_reader = true;
    e.stamp = ++g.hm_clock; g.hm_hits++;
    return true;
}
// after stream st has produced H(key) in src / src_ok: keep a copy in the least recently used slot
void hm_store(const uint8_t key[48], const g2a* src, const uint8_t* src_ok, cudaStream_t st) {
    int victim = 0;
    for (int i = 0; i < Ctx::HM_N; i++) {
        if (!g.hm[i].used) { victim = i; break; }
        if (g.hm[i].stamp < g.hm[victim].stamp) victim = i;
    }
    Ctx::HmEntry& e = g.hm[victim];
    if (e.used) { cudaStreamWaitEvent(st, e.filled, 0); if (e.has_reader) cudaStreamWaitEvent(st, e.read_done, 0); }
    cudaMemcpyAsync(g.hm_slots + victim, src, sizeof(g2a), cudaMemcpyDeviceToDevice, st);
    cudaMemcpyAsync(g.hm_ok + victim, src_ok, 1, cudaMemcpyDeviceToDevice, st);
    cudaEventRecord(e.filled, st);
    memcpy(e.key, key, 48); e.used = true; e.has_reader = false; e.stamp = ++g.hm_clock;
}
// while the self-test runs, every launch records its kernel's name (hbls_self_test_kernels)
#define ST_NOTE(kern) do { if (g.st_rec) g.st_kernels.insert(#kern); } while (0)
#define LAUNCH(kern, grid, block, strm, ...) do { kern<<<(grid), (block), 0, (strm)>>>(__VA_ARGS__); g.launches++; ST_NOTE(kern); } while (0)
#define LAUNCH_SMEM(kern, grid, block, smem, strm, ...) do { kern<<<(grid), (block), (smem), (strm)>>>(__VA_ARGS__); g.launches++; ST_NOTE(kern); } while (0)

constexpr unsigned TPB = 64;      // heavy kernels: 64-thread CTAs
// persistent launch geometry for the grid-stride kernels: at most `tpsm` resident threads per SM (default 384) so the per-thread
// stack (Fp12 temporaries) stays in L1/L2
unsigned capped_blocks(size_t n, long long tpsm, unsigned tpb) {
    size_t cap = (size_t)g.sm_count * (size_t)((tpsm < (long long)tpb ? tpb : tpsm) / tpb);
    size_t need = (n + tpb - 1) / tpb;
    return (unsigned)(need < cap ? need : cap);
}
unsigned heavy_blocks(size_t n) { return capped_blocks(n, g.tpsm, TPB); }
unsigned light_blocks(size_t n) { return capped_blocks(n, g.tpsm_light, TPB); }       // small-state kernels: the register count decides
unsigned split_blocks(size_t nthreads) { return capped_blocks(nthreads, g.tpsm_split, HB_TPB_SPLIT); }
// lock-stepped lane-pair kernels: one CTA per SM, its size = the resident threads wanted for that kernel (multiple of 64, <= 512)
unsigned lockstep_cta(long long t) { t = t < 64 ? 64 : (t > HB_TPB_SPLIT ? HB_TPB_SPLIT : t); return (unsigned)(t & ~63ll); }

// hash-to-G2 of a small batch (latency path): one WARP per message while that still leaves every warp its own scheduler's worth of
// an SM (the cofactor clearing runs as VM step programs), else one message per lane pair
void launch_hash_small(cudaStream_t st, size_t n, const uint8_t* d_msgs, uint32_t msg_len, g2a* hm, uint8_t* ok_hm) {
    if ((long long)n <= g.hash_coop_max) LAUNCH(k_hash_to_g2_coop, (unsigned)n, 32, st, n, d_msgs, msg_len, hm, ok_hm, (int)g.hash_fallback);
    else LAUNCH(k_hash_to_g2_pair, blocks_for(2 * n, 32), 32, st, n, d_msgs, msg_len, hm, ok_hm);
}

// hash-to-G2 of a large batch, one message per thread: one kernel, or map + cofactor clearing (hash_split 1), or map + cofactor
// clearing into the Jacobian buffer S (B points) + affine conversion (hash_split 2)
void launch_hash_batch(cudaStream_t s, size_t B, const uint8_t* d_msgs, uint32_t msg_len, g2a* hm, uint8_t* ok_hm, g2* S) {
    if (g.hash_split && HB_BATCH_INV) {
        LAUNCH(k_hash_sw, capped_blocks(B, g.tpsm_sw, TPB), TPB, s, B, d_msgs, msg_len, hm, ok_hm);
        if (g.hash_split >= 2) {        // three kernels: map | cofactor clearing (Jacobian, into the S buffer the scaling stage fills later) | affine
            const unsigned t = lockstep_cta(g.tpsm_cof);
            LAUNCH(k_hash_cofactor_pair, capped_blocks(2 * B, t, t), t, s, B, (const g2a*)hm, (const uint8_t*)ok_hm, S);
            LAUNCH(k_g2_normalize_batch, heavy_blocks(B), TPB, s, B, (const g2*)S, hm);
        } else
            LAUNCH(k_hash_cofactor, heavy_blocks(B), TPB, s, B, hm, (const uint8_t*)ok_hm);
    } else
        LAUNCH(k_hash_to_g2, heavy_blocks(B), TPB, s, B, d_msgs, msg_len, hm, ok_hm);
}

// ------------------------------------------------------------------ coefficient stream (host): ChaCha20 block function, RFC 8439
void chacha20_block(const uint32_t key[8], uint64_t counter, uint32_t out[16], uint32_t block = 0) {
    uint32_t st[16] = {0x61707865u, 0x3320646eu, 0x79622d32u, 0x6b206574u, key[0], key[1], key[2], key[3], key[4], key[5], key[6], key[7],
                       (uint32_t)counter, (uint32_t)(counter >> 32), 0x68626c73u /* "hbls" */, block};
    uint32_t x[16]; memcpy(x, st, sizeof x);
    auto rotl = [](uint32_t v, int c) { return (v << c) | (v >> (32 - c)); };
    auto qr = [&](int a, int b, int c, int d) {
        x[a] += x[b]; x[d] ^= x[a]; x[d] = rotl(x[d], 16); x[c] += x[d]; x[b] ^= x[c]; x[b] = rotl(x[b], 12);
        x[a] += x[b]; x[d] ^= x[a]; x[d] = rotl(x[d], 8);  x[c] += x[d]; x[b] ^= x[c]; x[b] = rotl(x[b], 7);
    };
    for (int r = 0; r < 10; r++) { qr(0, 4, 8, 12); qr(1, 5, 9, 13); qr(2, 6, 10, 14); qr(3, 7, 11, 15); qr(0, 5, 10, 15); qr(1, 6, 11, 12); qr(2, 7, 8, 13); qr(3, 4, 9, 14); }
    for (int i = 0; i < 16; i++) out[i] = x[i] + st[i];
}
// one fresh draw per position inside a group, per call (kernels.cuh: rlc_coeffs); the low bit of each half-scalar pair is forced
// odd on the device (rlc_scale_pair), leaving 63 random bits per coefficient
rlc_coeffs rlc_draw() {
    uint32_t blk[16]; chacha20_block(g.chacha_key, ++g.rlc_calls, blk);
    rlc_coeffs co;
    for (int k = 0; k < HB_RLC_GMAX; k++) co.c[k] = ((uint64_t)blk[2 * k + 1] << 32) | blk[2 * k];
    return co;
}

// blocks: one draw per (position inside a group, member of a block), 16 ChaCha20 blocks of the call's counter
rlc_block_coeffs rlc_draw_block() {
    rlc_block_coeffs cb; const uint64_t call = ++g.rlc_calls; uint32_t blk[16];
    for (int i = 0; i < HB_RLC_GMAX * HB_RLC_M; i++) {
        if ((i & 7) == 0) chacha20_block(g.chacha_key, call, blk, (uint32_t)(i >> 3) + 1);
        cb.c[i / HB_RLC_M][i % HB_RLC_M] = ((uint64_t)blk[2 * (i & 7) + 1] << 32) | blk[2 * (i & 7)];
    }
    return cb;
}
// one independent draw per item (the single combined check of hbls_rlc_partial / hbls_rlc_fold)
std::vector<uint64_t> rlc_draw_items(size_t k) {
    std::vector<uint64_t> c(k); const uint64_t call = ++g.rlc_calls; uint32_t blk[16];
    for (size_t j = 0; j < k; j++) {
        if ((j & 7) == 0) chacha20_block(g.chacha_key, call, blk, (uint32_t)(j >> 3) + 1);
        c[j] = ((uint64_t)blk[2 * (j & 7) + 1] << 32) | blk[2 * (j & 7)];
    }
    return c;
}

// ------------------------------------------------------------------ one verification pass over device-resident inputs.
// batched form: groups of 8 once that still gives every SM a full CTA of lane pairs (fewer Miller-loop pairs and final exponentiations
// per round), else 4
size_t rlc_group_size(size_t B) {
    return (g.rlc_g == 4 || g.rlc_g == 8) ? (size_t)g.rlc_g : (2 * (B / 8) >= (size_t)g.sm_count * HB_TPB_SPLIT ? 8 : 4);
}
// two-phase form: groups per pass = one lane pair per group on every SM (256 lane pairs per SM), i.e. one wave of the line kernel
size_t rlc_chunk_groups() { return (size_t)g.sm_count * (HB_TPB_SPLIT / 2); }
static bool rlc_applies(size_t B);
static bool exact_two_phase(size_t B);
size_t rlc_lines_bytes(size_t B) {
    if (!g.rlc_two_phase) return 0;
    if (!rlc_applies(B)) {      // exact form through the same kernels: "groups" of one round, two pairs each
        if (!exact_two_phase(B)) return 0;
        const size_t ngc = B < rlc_chunk_groups() ? B : rlc_chunk_groups();
        return (size_t)HB_ML_STEPS * 3 * 2 * ngc * 2 * sizeof(fp) + 256;
    }
    const size_t G = rlc_group_size(B), ng = B / G, ngc = ng < rlc_chunk_groups() ? ng : rlc_chunk_groups();
    const size_t rlc_bytes = (size_t)HB_ML_STEPS * 3 * (G + 1) * ngc * 2 * sizeof(fp);
    // the exact pass over the rounds of failed groups runs through the same buffer ("groups" of one round, <= all rounds of the batch)
    const size_t nlc = B < rlc_chunk_groups() ? B : rlc_chunk_groups();
    const size_t list_bytes = g.exact_two_phase ? (size_t)HB_ML_STEPS * 3 * 2 * nlc * 2 * sizeof(fp) + B * sizeof(g2a) + 256 : 0;
    return (rlc_bytes > list_bytes ? rlc_bytes : list_bytes) + 256;
}
// blocks per call at most: S <= ceil(ng / HB_RLC_M) + 31
size_t rlc_nblocks_max(size_t B) { return B / HB_RLC_G / HB_RLC_M + 32; }
size_t verify_scratch_bytes(size_t B) {
    return B * (sizeof(g2a) * 2 + sizeof(g1a) * 2 + sizeof(g1) + sizeof(g2) + 16 + 4 + 7) + HB_MASK_BINS * 4 + (B / HB_RLC_G + 1) * (sizeof(g2a) + 8) + rlc_nblocks_max(B) * (sizeof(g2a) + 1) + 46 * 256
           + (B <= 8192 ? B * (12 * sizeof(fp2) + 3) + 1024 : 0)                // latency path: Miller values of (B, sigma) and (-apk, H(m))
           + rlc_lines_bytes(B);                                                 // two-kernel pairing: the line functions of one chunk
}
struct VerifyBufs { g2a* sig; g2a* hm; g1a* pkneg; g1* apk; uint8_t* ok_sig; uint8_t* ok_hm; uint8_t* ok_pk;
                    g1a* pk_scaled; g2* S; uint8_t* bad; g2a* Sg; uint8_t* group_ok; uint32_t* fail_list; unsigned* counts; g2a* Sb; uint8_t* block_ok;
                    fp2* f1; uint8_t* irr1; fp2* f2; uint8_t* irr2; uint8_t* ok_sub;
                    uint16_t* mask_cost; unsigned* mask_hist; uint32_t* mask_order; fp* lines; uint8_t* verdict; };
VerifyBufs carve_verify(Arena& ar, size_t B) {
    VerifyBufs v;
    v.sig = ar.take<g2a>(B); v.hm = ar.take<g2a>(B); v.pkneg = ar.take<g1a>(B); v.apk = ar.take<g1>(B);
    v.ok_sig = ar.take<uint8_t>(B); v.ok_hm = ar.take<uint8_t>(B); v.ok_pk = ar.take<uint8_t>(B);
    v.pk_scaled = ar.take<g1a>(B); v.S = ar.take<g2>(B); v.bad = ar.take<uint8_t>(B);
    v.Sg = ar.take<g2a>(B / HB_RLC_G + 1); v.group_ok = ar.take<uint8_t>(B / HB_RLC_G + 1);
    v.fail_list = ar.take<uint32_t>(B); v.counts = ar.take<unsigned>(5);      // [0] [1] k_rlc_finish, [2] [3] form gates, [4] per-group check list
    v.Sb = ar.take<g2a>(rlc_nblocks_max(B)); v.block_ok = ar.take<uint8_t>(rlc_nblocks_max(B));
    v.mask_cost = ar.take<uint16_t>(B); v.mask_hist = ar.take<unsigned>(HB_MASK_BINS); v.mask_order = ar.take<uint32_t>(B);
    v.verdict = ar.take<uint8_t>(B);
    v.lines = nullptr;
    if (rlc_lines_bytes(B)) v.lines = reinterpret_cast<fp*>(ar.take<uint8_t>(rlc_lines_bytes(B)));
    v.f1 = v.f2 = nullptr; v.irr1 = v.irr2 = v.ok_sub = nullptr;
    if (B <= 8192) { v.f1 = ar.take<fp2>(6 * B); v.irr1 = ar.take<uint8_t>(B); v.f2 = ar.take<fp2>(6 * B); v.irr2 = ar.take<uint8_t>(B); v.ok_sub = ar.take<uint8_t>(B); }
    return v;
}
// Small batches (latency path): the inputs are on the device from here on -- signature decode and hash-to-G2 may start on the
// auxiliary streams while the caller's stream still aggregates the public keys (launch_verify_tail joins them before the pairing).
static bool latency_path(size_t B);
void fork_point(size_t B, Scratch* sc, cudaStream_t s) {
    if (!latency_path(B) || !g.overlap || g.stage_timing) return;
    if (cudaEventRecord(sc->fork, s) == cudaSuccess) sc->forked = true;
}
// batched (random-linear-combination) form applies: default mode and a batch large enough
static bool rlc_applies(size_t B) { return g.batch_mode == 1 && (long long)B >= g.rlc_min && B >= 2 * HB_RLC_GMAX; }
static bool latency_path(size_t B) { return !rlc_applies(B) && (long long)B <= g.coop_max; }
// blocks of HB_RLC_M groups share one final exponentiation and one generator pair (kernels.cuh: rlc_block_coeffs).  They need the
// two-kernel pairing with every group in ONE chunk of the line buffer (a block must not span chunks); automatically from one whole
// block on, rlc_block = 1 / 2 forces them on / off (wherever they can run at all)
static bool rlc_blocks(size_t ng, bool two_phase) {
    if (!two_phase || g.rlc_block == 2 || ng > rlc_chunk_groups()) return false;
    return g.rlc_block == 1 || ng >= HB_RLC_M;
}
// the groups' Miller values of the block form: 6 Fp2 per group, behind the G round pairs' lines (the buffer holds G + 1 pairs)
static fp2* rlc_fm(const VerifyBufs& v, size_t G, size_t ng) { return reinterpret_cast<fp2*>(v.lines + (size_t)HB_ML_STEPS * 3 * G * ng * 2); }
// exact checks of batches beyond the warp-per-round range run as line kernel + accumulator kernel too (twice the lane pairs in the
// first one; the second no longer carries the running points)
static bool exact_two_phase(size_t B) { return g.rlc_two_phase >= 2 && g.exact_two_phase && !rlc_applies(B) && (long long)B > g.coop_max; }
// exact check of n rounds (contiguous arrays) as "groups" of one round through k_rlc_lines_split<1> / k_rlc_accum_split<1>
void launch_exact_two_phase(size_t n, const g2a* sig, const g1a* pkneg, const g2a* hm, const uint8_t* ok_a, const uint8_t* ok_b, const uint8_t* ok_c,
                            uint8_t* bad, uint8_t* verdict, fp* lines, uint8_t* d_results, cudaStream_t s);
// Message grouping of the device forms (device_forms.cuh): a hash table of >= 2k slots, the distinct messages' keys and points
struct MsgGroups { uint32_t mask; uint32_t* slot_item; uint32_t* slot_rep; uint32_t* item_slot; uint32_t* pos; uint32_t* grp; uint8_t* keys;
                   unsigned* count; g2a* hm_d; uint8_t* ok_d; };
size_t group_slots(size_t k) { size_t T = 64; while (T < 2 * k) T <<= 1; return T; }
size_t group_bytes(size_t k) { return group_slots(k) * 8 + k * (12 + 48 + sizeof(g2a) + 1) + 10 * 256; }
MsgGroups carve_groups(Arena& ar, size_t k) {
    MsgGroups m; const size_t T = group_slots(k);
    m.mask = (uint32_t)(T - 1); m.slot_item = ar.take<uint32_t>(T); m.slot_rep = ar.take<uint32_t>(T);
    m.item_slot = ar.take<uint32_t>(k); m.pos = ar.take<uint32_t>(k); m.grp = ar.take<uint32_t>(k); m.keys = ar.take<uint8_t>(48 * k);
    m.count = ar.take<unsigned>(1); m.hm_d = ar.take<g2a>(k); m.ok_d = ar.take<uint8_t>(k);
    return m;
}
// H(m) of the k items through their d distinct messages: group, hash the d keys with the form d calls for (launch_hash_small /
// launch_hash_batch with d in place of k: warp per message up to hash_coop_max, lane pair up to coop_max -- or k on the latency
// path --, thread per message beyond), gather to hm / ok_hm.  `pairs`: the call is on the latency path (no thread-per-item form).
void launch_hash_grouped(cudaStream_t s, size_t k, const MsgGroups& m, const uint8_t* d_msgs, uint32_t msg_len, bool pairs, g2a* hm,
                         uint8_t* ok_hm, g2* S) {
    cudaMemsetAsync(m.slot_item, 0xff, (size_t)(m.mask + 1) * 4, s);
    cudaMemsetAsync(m.slot_rep, 0xff, (size_t)(m.mask + 1) * 4, s);
    uint32_t blk[16]; chacha20_block(g.chacha_key, ++g.rlc_calls, blk);          // the table's hash key: fresh per call, never seen outside
    const uint64_t k0 = ((uint64_t)blk[1] << 32) | blk[0], k1 = ((uint64_t)blk[3] << 32) | blk[2];
    LAUNCH(k_group_insert, blocks_for(k, 256), 256, s, k, d_msgs, msg_len, m.mask, k0, k1, m.slot_item, m.slot_rep, m.item_slot);
    LAUNCH(k_group_compact, 1, HB_GRP_SCAN, s, k, d_msgs, msg_len, (const uint32_t*)m.slot_rep, (const uint32_t*)m.item_slot, m.pos, m.grp, m.keys, m.count);
    const unsigned long long coop_hi = (unsigned long long)g.hash_coop_max;
    const unsigned long long pair_hi = pairs ? (unsigned long long)k : (unsigned long long)(g.coop_max > g.hash_coop_max ? g.coop_max : g.hash_coop_max);
    if (!pairs) {          // map, then cofactor clearing and affine conversion over all k slots (the identity beyond what the map wrote)
        LAUNCH(k_hash_keys_sw, capped_blocks(k, g.tpsm_sw, TPB), TPB, s, k, (const unsigned*)m.count, pair_hi, (const uint8_t*)m.keys, m.hm_d, m.ok_d);
        const unsigned t = lockstep_cta(g.tpsm_cof);
        LAUNCH(k_hash_cofactor_pair, capped_blocks(2 * k, t, t), t, s, k, (const g2a*)m.hm_d, (const uint8_t*)m.ok_d, S);
        LAUNCH(k_g2_normalize_batch, heavy_blocks(k), TPB, s, k, (const g2*)S, m.hm_d);
    }
    const size_t cg = (long long)k < g.hash_coop_max ? k : (size_t)(g.hash_coop_max > 0 ? g.hash_coop_max : 1);
    LAUNCH(k_hash_keys_coop, (unsigned)cg, 32, s, (const unsigned*)m.count, coop_hi, (const uint8_t*)m.keys, m.hm_d, m.ok_d, (int)g.hash_fallback);
    LAUNCH(k_hash_keys_pair, blocks_for(2 * k, 32), 32, s, (const unsigned*)m.count, coop_hi, pair_hi, (const uint8_t*)m.keys, m.hm_d, m.ok_d);
    LAUNCH(k_broadcast_hm, blocks_for(k, 256), 256, s, k, (const uint32_t*)m.grp, (const g2a*)m.hm_d, (const uint8_t*)m.ok_d, hm, ok_hm);
}
#define STAGE_EV(i, sc, strm) do { if (g.stage_timing && (sc)->ev_ok) cudaEventRecord((sc)->ev[i], (strm)); } while (0)
// v.apk holds the Jacobian (aggregate) public key of every round; ok_pk (nullable) = per-round "key decoded" flags of the triple form
// h_msg (nullable): host copy of THE message when the call has a single one (one round, or a same-message batch) -- the key of the
// H(m) cache.  mg (nullable, device forms): H(m) once per distinct message, grouped on the device (same_msg / h_msg unused)
void launch_verify_tail(size_t B, const VerifyBufs& v, Scratch* sc, const uint8_t* d_sig96, const uint8_t* d_msgs, uint32_t msg_len,
                        const uint8_t* ok_pk, uint8_t* d_results, cudaStream_t s, bool same_msg, const uint8_t* h_msg = nullptr,
                        const MsgGroups* mg = nullptr) {
    STAGE_EV(1, sc, s);
    const bool rlc = rlc_applies(B);
    // the batched check consumes the Jacobian sums directly; -apk in affine form is then only needed for the rounds of failed groups
    // small batches (latency path): one item per lane pair, binary-GCD inversions; large ones: one item per thread, persistent
    const bool pairs = latency_path(B);
    if (!rlc) {
        if (pairs) LAUNCH(k_g1_normalize_lat, blocks_for(B, 32), 32, s, B, v.apk, v.pkneg, 1);
        else LAUNCH(k_g1_normalize, blocks_for(B, TPB), TPB, s, B, v.apk, v.pkneg, 1, (const int*)nullptr);
    }
    STAGE_EV(2, sc, s);
    const bool forked = pairs && sc->forked;              // decode on aux[0], hash on aux[1], concurrently with the work above
    cudaStream_t sd = forked ? g.aux[0] : s, sh = forked ? g.aux[1] : s;
    if (forked) { cudaStreamWaitEvent(sd, sc->fork, 0); cudaStreamWaitEvent(sh, sc->fork, 0); }
    const size_t coop_cap = (size_t)g.sm_count * (size_t)(g.coop_wpsm > 0 ? g.coop_wpsm : 1);      // resident warps (one round each)
    const unsigned coop_grid = (unsigned)(B < coop_cap ? B : coop_cap);
    const bool split_ml = forked && v.f1 != nullptr;       // Miller value of (B, sigma) on the decode stream, beside hash-to-G2
    // one message (one round, or a same-message batch): H(m) once -- from the cache when this node has hashed it before (it signed
    // it, verified it, or prefetched it)
    const bool one_msg = (same_msg && B > 1) || (B == 1 && h_msg);
    const bool use_cache = one_msg && h_msg != nullptr && hm_enabled();
    uint8_t key[48]; bool hit = false;
    if (use_cache) { hm_key(key, h_msg, msg_len); hit = hm_fetch(key, v.hm, v.ok_hm, sh); }
    // H(m) known up front: the two Miller values do not depend on each other -- (-apk, H(m)) starts right after the key aggregation
    // on the caller's stream, (B, sigma) after the decode on the decode stream with the signature's subgroup test beside it
    const bool warm = hit && split_ml;
    if (pairs) LAUNCH(k_g2_decode_pair, blocks_for(2 * B, 32), 32, sd, B, d_sig96, v.sig, v.ok_sig, warm ? 0 : 1);
    else if (g.decode_split) {
        LAUNCH(k_g2_decode, capped_blocks(B, g.tpsm_dec, TPB), TPB, s, B, d_sig96, v.sig, v.ok_sig, 0);
        const unsigned t = lockstep_cta(g.tpsm_sub);
        LAUNCH(k_g2_subgroup_pair, capped_blocks(2 * B, t, t), t, s, B, v.sig, (const uint8_t*)v.ok_sig, v.ok_sig, 1);
    } else LAUNCH(k_g2_decode, capped_blocks(B, g.tpsm_dec, TPB), TPB, s, B, d_sig96, v.sig, v.ok_sig, 1);
    if (warm) {
        cudaEventRecord(sc->mid, sd);
        LAUNCH(k_miller_pq_coop, coop_grid, 32, sd, B, (const g1a*)nullptr, v.sig, v.ok_sig, v.f1, v.irr1);
    } else if (split_ml) LAUNCH(k_miller1_coop, coop_grid, 32, sd, B, v.sig, v.ok_sig, v.f1, v.irr1);
    STAGE_EV(3, sc, s);
    if (mg)
        launch_hash_grouped(sh, B, *mg, d_msgs, msg_len, pairs, v.hm, v.ok_hm, v.S);
    else if (one_msg) {
        if (!hit) {
            if (pairs) launch_hash_small(sh, 1, d_msgs, msg_len, v.hm, v.ok_hm);
            else LAUNCH(k_hash_to_g2, 1, TPB, sh, (size_t)1, d_msgs, msg_len, v.hm, v.ok_hm);
            if (use_cache) hm_store(key, v.hm, v.ok_hm, sh);
        }
        if (B > 1) LAUNCH(k_broadcast_hm, blocks_for(B, 256), 256, sh, B, (const uint32_t*)nullptr, (const g2a*)v.hm, (const uint8_t*)v.ok_hm, v.hm, v.ok_hm);
    } else if (pairs)
        launch_hash_small(sh, B, d_msgs, msg_len, v.hm, v.ok_hm);
    else
        launch_hash_batch(s, B, d_msgs, msg_len, v.hm, v.ok_hm, v.S);
    if (warm) {
        cudaEventRecord(sc->join[1], sh); cudaStreamWaitEvent(s, sc->join[1], 0);
        LAUNCH(k_miller_pq_coop, coop_grid, 32, s, B, (const g1a*)v.pkneg, v.hm, (const uint8_t*)v.ok_hm, v.f2, v.irr2);
        cudaStreamWaitEvent(sh, sc->mid, 0);
        LAUNCH(k_g2_subgroup_pair, blocks_for(2 * B, 32), 32, sh, B, v.sig, v.ok_sig, v.ok_sub);
        cudaEventRecord(sc->join2, sh); cudaEventRecord(sc->join[0], sd);
        cudaStreamWaitEvent(s, sc->join[0], 0); cudaStreamWaitEvent(s, sc->join2, 0);
        cudaMemcpyAsync(v.ok_sig, v.ok_sub, B, cudaMemcpyDeviceToDevice, s);          // decode flag := decoded AND in the subgroup
    } else if (forked) {
        cudaEventRecord(sc->join[0], sd); cudaEventRecord(sc->join[1], sh);
        cudaStreamWaitEvent(s, sc->join[0], 0); cudaStreamWaitEvent(s, sc->join[1], 0);
    }
    STAGE_EV(4, sc, s);
    hbls_batch_info& bi = g.info;
    bi = hbls_batch_info{}; bi.rounds = B; bi.mode = rlc ? 1 : 0;
    cudaMemsetAsync(v.counts, 0, 5 * sizeof(unsigned), s);
    if (rlc) {
        // batched form (north-star "batched Miller loop + shared final exponentiation"): strided groups of G rounds; G = 8 once
        // that still gives every SM a full CTA of lane pairs (fewer Miller-loop pairs and final exponentiations per round), else 4
        const size_t G = rlc_group_size(B);
        const size_t ng = B / G, nr = ng * G, tail = B - nr;
        const rlc_coeffs co = rlc_draw();
        const bool full = 2 * ng >= (size_t)g.sm_count * HB_TPB_SPLIT;
        const unsigned pb = full ? split_blocks(2 * ng) : blocks_for(2 * ng, 64), pt = full ? HB_TPB_SPLIT : 64;
        const bool two_phase = g.rlc_two_phase && v.lines != nullptr && (full || g.rlc_two_phase >= 2);
        // blocks of HB_RLC_M groups: group g is member g / S of block g mod S; coefficients per (position, member)
        const bool blocks = rlc_blocks(ng, two_phase);
        const size_t S = blocks ? (((ng + HB_RLC_M - 1) / HB_RLC_M + 31) & ~(size_t)31) : 0;
        const rlc_block_coeffs cb = blocks ? rlc_draw_block() : rlc_block_coeffs{};
        // blocks possible: the device picks the form from how the last such call ended (k_rlc_form); counts[2] / counts[3] gate the
        // group form's / block form's kernels, the scaling kernels take the matching coefficients
        const unsigned* blk_gate = blocks ? v.counts + 3 : nullptr;
        if (blocks) LAUNCH(k_rlc_form, 1, 32, s, ng, g.rlc_block == 1 ? 1 : 0, (const int*)g.rlc_form, v.counts + 2);
        bool joint = false;
        if (g.scale_split && HB_BATCH_INV) {
            LAUNCH(k_rlc_scale_g1, capped_blocks(nr, g.tpsm_scale_g1, TPB), TPB, s, nr, ng, v.apk, co, v.pk_scaled, S, cb, blk_gate);
            const unsigned t = lockstep_cta(g.tpsm_scale_g2);
            // the joint ladder runs a lane pair per GROUP: G times fewer items than the per-round ladder, so it needs a full chip of groups
            joint = g.scale_joint >= 2 || (g.scale_joint == 1 && full);
            if (joint) {          // one ladder per group into the Jacobian Sg (the first ng entries of S), then the shared-inversion affine form
                if (G == 8) LAUNCH(k_rlc_group_scale_g2_pair<8>, capped_blocks(2 * ng, t, t), t, s, ng, v.apk, v.sig, v.hm, v.ok_sig, v.ok_hm, ok_pk, co, v.S, v.bad, S, cb, blk_gate);
                else LAUNCH(k_rlc_group_scale_g2_pair<4>, capped_blocks(2 * ng, t, t), t, s, ng, v.apk, v.sig, v.hm, v.ok_sig, v.ok_hm, ok_pk, co, v.S, v.bad, S, cb, blk_gate);
                LAUNCH(k_g2_normalize_batch, heavy_blocks(ng), TPB, s, ng, (const g2*)v.S, v.Sg);
            } else
                LAUNCH(k_rlc_scale_g2_pair, capped_blocks(2 * nr, t, t), t, s, nr, ng, v.apk, v.sig, v.hm, v.ok_sig, v.ok_hm, ok_pk, co, v.S, v.bad, S, cb, blk_gate);
        } else
        LAUNCH(k_rlc_scale, capped_blocks(nr, g.tpsm_scale, TPB), TPB, s, nr, ng, v.apk, v.sig, v.hm, v.ok_sig, v.ok_hm, ok_pk, co, (const uint64_t*)nullptr, v.pk_scaled, v.S, v.bad, S, cb, blk_gate);
        if (!joint && G == 8) LAUNCH(k_rlc_group_sum<8>, heavy_blocks(ng), TPB, s, ng, v.S, v.Sg);
        else if (!joint) LAUNCH(k_rlc_group_sum<4>, heavy_blocks(ng), TPB, s, ng, v.S, v.Sg);
        STAGE_EV(5, sc, s);
        if (two_phase) {
            // running points in their own kernel (lines to HBM, read once), accumulator + final exponentiation in the second
            for (size_t g0 = 0; g0 < ng; g0 += rlc_chunk_groups()) {
                const size_t ngc = ng - g0 < rlc_chunk_groups() ? ng - g0 : rlc_chunk_groups();
                // a batch that does not fill the chip: 64-thread CTAs spread over the SMs (the line kernel has G + 1 times the lane pairs)
                const unsigned lt = full ? lockstep_cta(g.tpsm_lines) : 64, at = full ? lockstep_cta(g.tpsm_accum) : 64;
                const unsigned lb = full ? capped_blocks(2 * (G + 1) * ngc, lt, lt) : blocks_for(2 * (G + 1) * ngc, 64);
                const unsigned ab = full ? capped_blocks(2 * ngc, at, at) : blocks_for(2 * ngc, 64);
                // blocks possible (one chunk): both forms are launched and the device gates (k_rlc_form) let exactly one of them run
                const unsigned* gate_groups = blocks ? v.counts + 2 : nullptr;
                const unsigned* gate_blocks = v.counts + 3;
                if (G == 8) LAUNCH(k_rlc_lines_split<8>, lb, lt, s, ng, g0, ngc, v.pk_scaled, v.hm, v.Sg, v.lines, gate_groups);
                else LAUNCH(k_rlc_lines_split<4>, lb, lt, s, ng, g0, ngc, v.pk_scaled, v.hm, v.Sg, v.lines, gate_groups);
                if (blocks && G == 8) LAUNCH(k_rlc_lines_blk<8>, lb, lt, s, ng, g0, ngc, v.pk_scaled, v.hm, v.lines, gate_blocks);
                else if (blocks) LAUNCH(k_rlc_lines_blk<4>, lb, lt, s, ng, g0, ngc, v.pk_scaled, v.hm, v.lines, gate_blocks);
                if (g0 == 0) { STAGE_EV(7, sc, s); sc->ev7_set = g.stage_timing && sc->ev_ok; }       // line kernel | accumulator kernel (first chunk)
                if (G == 8) LAUNCH(k_rlc_accum_split<8>, ab, at, s, ng, g0, ngc, (const fp*)v.lines, v.bad, v.group_ok, gate_groups);
                else LAUNCH(k_rlc_accum_split<4>, ab, at, s, ng, g0, ngc, (const fp*)v.lines, v.bad, v.group_ok, gate_groups);
                if (blocks && G == 8) LAUNCH(k_rlc_accum_blk<8>, ab, at, s, ng, g0, ngc, (const fp*)v.lines, v.bad, v.group_ok, rlc_fm(v, G, ng), gate_blocks);
                else if (blocks) LAUNCH(k_rlc_accum_blk<4>, ab, at, s, ng, g0, ngc, (const fp*)v.lines, v.bad, v.group_ok, rlc_fm(v, G, ng), gate_blocks);
            }
            if (blocks) {
                // one final exponentiation and one generator pair per block (warp per block), then the groups of the failed blocks
                // alone: FE( their Miller value * Miller(B, Sg) ) == 1, a lane pair each, the list spread evenly over the lock-stepped
                // CTAs.  group_ok then holds every group's own verdict, as without blocks.
                fp2* fm = rlc_fm(v, G, ng);
                const unsigned cb_grid = full ? split_blocks(2 * ng) : blocks_for(2 * ng, 64), cb_tpb = full ? HB_TPB_SPLIT : 64;
                const unsigned* gate = v.counts + 3;
                LAUNCH(k_rlc_block_sum, heavy_blocks(S), TPB, s, S, ng, (const g2a*)v.Sg, v.Sb, gate);
                const size_t coop_cap = (size_t)g.sm_count * (size_t)(g.coop_wpsm > 0 ? g.coop_wpsm : 1);
                LAUNCH(k_rlc_block_coop, (unsigned)(S < coop_cap ? S : coop_cap), 32, s, S, ng, (const fp2*)fm, (const g2a*)v.Sb, (const uint8_t*)v.group_ok, v.block_ok, gate);
                LAUNCH(k_rlc_block_list, blocks_for(ng, 256), 256, s, ng, S, (const uint8_t*)v.block_ok, v.group_ok, v.fail_list, v.counts + 4, gate);
                LAUNCH(k_rlc_group_check_list, cb_grid, cb_tpb, s, (const unsigned*)v.counts + 4, (const uint32_t*)v.fail_list, (const fp2*)fm,
                       (const g2a*)v.Sg, v.group_ok);
            }
        } else if (G == 8)
            LAUNCH_SMEM(k_rlc_pairing_split<8>, pb, pt, HB_SMEM_F ? pt * HB_SMEM_F_WORDS * 4 : 0, s, ng, v.pk_scaled, v.hm, v.Sg, v.bad, v.group_ok);
        else
            LAUNCH_SMEM(k_rlc_pairing_split<4>, pb, pt, HB_SMEM_F ? pt * HB_SMEM_F_WORDS * 4 : 0, s, ng, v.pk_scaled, v.hm, v.Sg, v.bad, v.group_ok);
        // exact pass over the rounds of failed groups only (compacted on the device; the launches are sized for the worst case and
        // return at once when the list is short or empty)
        LAUNCH(k_rlc_finish, blocks_for(nr, 256), 256, s, nr, ng, v.group_ok, d_results, v.fail_list, v.counts);
        if (blocks) LAUNCH(k_rlc_form_update, 1, 32, s, ng, (const unsigned*)v.counts, g.rlc_form);     // the next call's form
        LAUNCH(k_g1_normalize_list, heavy_blocks(nr), TPB, s, v.counts, v.fail_list, v.apk, v.pkneg, 1);
        if (two_phase && g.exact_two_phase) {
            // the listed rounds, gathered into contiguous arrays, through the line / accumulator kernels as "groups" of one round; the
            // launches are sized for the worst case and return at once beyond the device-side count
            const size_t nlc = nr < rlc_chunk_groups() ? nr : rlc_chunk_groups();
            g2a* hm_c = reinterpret_cast<g2a*>(v.lines + (size_t)HB_ML_STEPS * 3 * 2 * nlc * 2);      // behind the chunk's lines
            g2a* sig_c = reinterpret_cast<g2a*>(v.S); g1a* pk_c = v.pk_scaled;                        // both free after the group pass
            const unsigned* cnt = v.counts;
            LAUNCH(k_exact_prepare, blocks_for(nr, 256), 256, s, nr, (const uint32_t*)v.fail_list, (const g2a*)v.sig, (const g1a*)v.pkneg, (const g2a*)v.hm,
                   (const uint8_t*)v.ok_sig, (const uint8_t*)v.ok_hm, ok_pk, pk_c, hm_c, sig_c, v.bad, d_results, cnt);
            const bool lfull = 2 * nr >= (size_t)g.sm_count * HB_TPB_SPLIT;
            const unsigned bt = lfull ? HB_TPB_SPLIT : 64;
            for (size_t g0 = 0; g0 < nr; g0 += rlc_chunk_groups()) {
                const size_t nc = nr - g0 < rlc_chunk_groups() ? nr - g0 : rlc_chunk_groups();
                const unsigned lb = lfull ? split_blocks(4 * nc) : blocks_for(4 * nc, 64), ab = lfull ? split_blocks(2 * nc) : blocks_for(2 * nc, 64);
                LAUNCH(k_rlc_lines_split<1>, lb, bt, s, nr, g0, nc, (const g1a*)pk_c, (const g2a*)hm_c, (const g2a*)sig_c, v.lines, cnt);
                LAUNCH(k_rlc_accum_split<1>, ab, bt, s, nr, g0, nc, (const fp*)v.lines, (const uint8_t*)v.bad, v.verdict, cnt);
            }
            LAUNCH(k_exact_publish, blocks_for(nr, 256), 256, s, nr, (const uint32_t*)v.fail_list, (const uint8_t*)v.verdict, d_results, cnt);
        } else if (2 * nr >= (size_t)g.sm_count * HB_TPB_SPLIT)
            LAUNCH(k_pairing_verify_split_list, split_blocks(2 * nr), HB_TPB_SPLIT, s, v.counts, v.fail_list, v.sig, v.pkneg, v.hm, v.ok_sig, v.ok_hm, ok_pk, d_results);
        else
            LAUNCH(k_pairing_verify_split_list, blocks_for(2 * nr, 64), 64, s, v.counts, v.fail_list, v.sig, v.pkneg, v.hm, v.ok_sig, v.ok_hm, ok_pk, d_results);
        LAUNCH(k_pairing_fixup_list, heavy_blocks(nr), TPB, s, v.counts, v.fail_list, v.sig, v.pkneg, v.hm, v.ok_sig, v.ok_hm, ok_pk, d_results);
        if (tail) {       // the < G rounds that do not fill a group are always verified exactly
            LAUNCH(k_g1_normalize, 1, TPB, s, tail, v.apk + nr, v.pkneg + nr, 1, (const int*)nullptr);
            LAUNCH(k_pairing_verify_split, blocks_for(2 * tail, 64), 64, s, tail, v.sig + nr, v.pkneg + nr, v.hm + nr, v.ok_sig + nr, v.ok_hm + nr,
                   ok_pk ? ok_pk + nr : (const uint8_t*)nullptr, d_results + nr, (const int*)nullptr);
            LAUNCH(k_pairing_fixup, 1, TPB, s, tail, v.sig + nr, v.pkneg + nr, v.hm + nr, v.ok_sig + nr, v.ok_hm + nr,
                   ok_pk ? ok_pk + nr : (const uint8_t*)nullptr, d_results + nr, (const int*)nullptr);
        }
        bi.group_size = (int32_t)G; bi.groups = ng; bi.tail_rounds = (uint32_t)tail; bi.cta_threads = pt;
    } else {
        // exact form at every batch size: a lane pair per round.  Large batches use 512-thread lock-stepped CTAs (one per SM),
        // small ones 64-thread CTAs spread over the SMs.
        STAGE_EV(5, sc, s);
        const bool full = 2 * B >= (size_t)g.sm_count * HB_TPB_SPLIT;
        const bool coop = (long long)B <= g.coop_max;        // latency form: one warp per round (vm.cuh), up to 14 resident rounds per SM (15 KB of slots each)
        if (coop && warm)
            LAUNCH(k_fe2_coop, coop_grid, 32, s, B, v.f1, v.irr1, v.f2, v.irr2, v.ok_sig, v.ok_hm, ok_pk, (const uint8_t*)nullptr, d_results);
        else if (coop && split_ml)
            LAUNCH(k_pairing_coop2, coop_grid, 32, s, B, v.f1, v.irr1, v.pkneg, v.hm, v.ok_sig, v.ok_hm, ok_pk, d_results);
        else if (coop)
            LAUNCH(k_pairing_coop, coop_grid, 32, s, B, v.sig, v.pkneg, v.hm, v.ok_sig, v.ok_hm, ok_pk, d_results);
        else if (exact_two_phase(B) && v.lines)
            launch_exact_two_phase(B, v.sig, v.pkneg, v.hm, v.ok_sig, v.ok_hm, ok_pk, v.bad, v.verdict, v.lines, d_results, s);
        else if (full)
            LAUNCH(k_pairing_verify_split, split_blocks(2 * B), HB_TPB_SPLIT, s, B, v.sig, v.pkneg, v.hm, v.ok_sig, v.ok_hm, ok_pk, d_results, (const int*)nullptr);
        else
            LAUNCH(k_pairing_verify_split, blocks_for(2 * B, 64), 64, s, B, v.sig, v.pkneg, v.hm, v.ok_sig, v.ok_hm, ok_pk, d_results, (const int*)nullptr);
        LAUNCH(k_pairing_fixup, heavy_blocks(B), TPB, s, B, v.sig, v.pkneg, v.hm, v.ok_sig, v.ok_hm, ok_pk, d_results, (const int*)nullptr);
        bi.cta_threads = coop ? 32 : (full ? HB_TPB_SPLIT : 64);
    }
    STAGE_EV(6, sc, s);
    cudaMemcpyAsync(sc->h_counts, v.counts, 2 * sizeof(unsigned), cudaMemcpyDeviceToHost, s);
    cudaEventRecord(sc->done, s);
    g.info_sc = sc; g.info_valid = true;
    if (g.stage_timing && sc->ev_ok) g.stage_sc = sc;
}

void launch_exact_two_phase(size_t n, const g2a* sig, const g1a* pkneg, const g2a* hm, const uint8_t* ok_a, const uint8_t* ok_b, const uint8_t* ok_c,
                            uint8_t* bad, uint8_t* verdict, fp* lines, uint8_t* d_results, cudaStream_t s) {
    LAUNCH(k_exact_prepare, blocks_for(n, 256), 256, s, n, (const uint32_t*)nullptr, sig, pkneg, hm, ok_a, ok_b, ok_c,
           (g1a*)nullptr, (g2a*)nullptr, (g2a*)nullptr, bad, d_results);
    const bool full = 2 * n >= (size_t)g.sm_count * HB_TPB_SPLIT;
    for (size_t g0 = 0; g0 < n; g0 += rlc_chunk_groups()) {
        const size_t nc = n - g0 < rlc_chunk_groups() ? n - g0 : rlc_chunk_groups();
        const unsigned bt = full ? HB_TPB_SPLIT : 64;
        const unsigned lb = full ? split_blocks(4 * nc) : blocks_for(4 * nc, 64), ab = full ? split_blocks(2 * nc) : blocks_for(2 * nc, 64);
        LAUNCH(k_rlc_lines_split<1>, lb, bt, s, n, g0, nc, pkneg, hm, sig, lines);
        LAUNCH(k_rlc_accum_split<1>, ab, bt, s, n, g0, nc, (const fp*)lines, (const uint8_t*)bad, verdict);
    }
    LAUNCH(k_exact_publish, blocks_for(n, 256), 256, s, n, (const uint32_t*)nullptr, (const uint8_t*)verdict, d_results);
}

// sk (little-endian u64 x 4, < r < Z^4) -> its four base-Z digits, Z = |z| = 0xd201000000010000 (plain long division on the host)
bool sk_digits_base_z(const uint64_t sk[4], uint64_t dig[4]) {
    const uint64_t Z = 0xd201000000010000ull;
    uint64_t v[4] = {sk[0], sk[1], sk[2], sk[3]};
    for (int k = 0; k < 3; k++) {
        unsigned __int128 rem = 0;
        for (int i = 3; i >= 0; i--) { const unsigned __int128 cur = (rem << 64) | v[i]; v[i] = (uint64_t)(cur / Z); rem = cur % Z; }
        dig[k] = (uint64_t)rem;
    }
    dig[3] = v[0];
    return (v[1] | v[2] | v[3]) == 0;                 // always for sk < r < Z^4; a hand-filled struct >= Z^4 takes the plain ladder
}

// r (BLS12-381 group order), little-endian u64
const uint64_t R_ORDER[4] = {0xffffffff00000001ull, 0x53bda402fffe5bfeull, 0x3339d80809a1d805ull, 0x73eda753299d7d48ull};
bool scalar_lt_r(const uint64_t k[4]) {
    for (int i = 3; i >= 0; i--) { if (k[i] < R_ORDER[i]) return true; if (k[i] > R_ORDER[i]) return false; }
    return false;
}

// ------------------------------------------------------------------ herumi-API calls (part 1 of include/hbls.h), n requests at a
// time.  Concurrent calls from different threads are combined into turns (coalesce.hpp); a turn stages the inputs of all its requests
// with one copy, runs each kernel once over the requests that need it and copies the results back once.  A lone call is a turn of
// one and launches the kernels a call has always launched.
// The single checks against a committee (hbls_aggregate_verify: AGG) and a resident mask (hbls_mask_verify: MASK) join the same
// turns: with VERIFY they are the turn's verify requests and share its warp-per-round cap.
enum { RQ_VERIFY, RQ_SIGN, RQ_PUBKEY, RQ_SINGLE, RQ_AGG, RQ_MASK };
constexpr size_t PART1_CAP = 1024;       // sign / GetPublicKey / single-element requests per turn (verify: coop_max, the warp-per-round limit)
struct Part1Req : hbls_coalesce::Request {
    const void* a = nullptr; const void* b = nullptr;   // VERIFY: signature, public key; AGG / MASK: the serialized signature (96 bytes);
                                                        // SIGN / PUBKEY: secret key; SINGLE: operands
    size_t an = 0, bn = 0;                              // SINGLE: operand bytes
    const void* msg = nullptr; size_t len = 0;          // VERIFY / AGG / MASK / SIGN: the hash (first 48 bytes); SINGLE: the message length
    void* out = nullptr; size_t on = 0;                 // SIGN / PUBKEY: the result struct; SINGLE: the result bytes
    const hbls_committee* com = nullptr;                // AGG: the committee, and the bitmap of blen = (n + 7) / 8 bytes
    const uint8_t* bitmap = nullptr; size_t blen = 0;
    const hbls_mask* mask = nullptr;                    // MASK: the mask whose resident aggregate key is checked
    int op = 0;                                         // SINGLE: OP_*
    int err = 0;                                        // HBLS_ERR_CUDA when the turn's device work failed (nothing written)
    int rc = 0;                                         // VERIFY / AGG / MASK: 1 / 0; SIGN: 0 / -1; SINGLE: the op's return code
};
static bool is_verify(int kind) { return kind == RQ_VERIFY || kind == RQ_AGG || kind == RQ_MASK; }
static_assert(sizeof(g1) == sizeof(blsPublicKey) && sizeof(g2) == sizeof(blsSignature), "herumi struct layout");
// byte layout of one staging copy: 256-byte aligned sections
struct Layout {
    size_t size = 0;
    size_t put(size_t bytes) { const size_t off = (size + 255) & ~(size_t)255; size = off + (bytes ? bytes : 1); return off; }
};

// One turn: the requests rq[0..n) under g.mu.  d_apk / sig96 (a lone hbls_mask_verify: one verify request): the key is already on
// the device and the signature is serialized (decoded and subgroup-checked here).  Otherwise the verify requests run in the order
// AGG, MASK, VERIFY through one pipeline: their keys land in one array of Jacobian keys inside the staging buffer (AGG: summed from
// the committee tables by k_mask_aggregate_items, MASK: the resident aggregate copied device to device, VERIFY: staged), the AGG /
// MASK signatures are decoded with the subgroup test and the VERIFY structs made affine, then one pairing launch checks them all.
// Fills in each request's results and returns 0, or HBLS_ERR_CUDA with no result written.
int part1_locked(Part1Req* const* rq, size_t n, const g1* d_apk = nullptr, const uint8_t* sig96 = nullptr) {
    cudaStream_t s = g.stream;
    std::vector<Part1Req*> ver, sgn, pub, one;
    for (size_t i = 0; i < n; i++) (is_verify(rq[i]->kind) ? ver : rq[i]->kind == RQ_SIGN ? sgn : rq[i]->kind == RQ_PUBKEY ? pub : one).push_back(rq[i]);
    auto vrank = [](int kind) { return kind == RQ_AGG ? 0 : kind == RQ_MASK ? 1 : 2; };
    std::stable_sort(ver.begin(), ver.end(), [&](const Part1Req* x, const Part1Req* y) { return vrank(x->kind) < vrank(y->kind); });
    size_t na = 0, nser = 0;                            // AGG requests; AGG + MASK requests (serialized signatures)
    for (const Part1Req* r : ver) { na += r->kind == RQ_AGG; nser += r->kind != RQ_VERIFY; }
    if (d_apk) na = nser = 0;
    size_t bm_bytes = 0;
    for (size_t i = 0; i < na; i++) bm_bytes += ver[i]->blen;
    // signing keys in base |z| first (ladder over psi), hand-filled keys >= Z^4 after them (plain ladder)
    std::vector<uint64_t> dig; size_t ngls = 0;
    {
        std::vector<Part1Req*> rest;
        for (Part1Req* r : sgn) {
            uint64_t d[4];
            if (sk_digits_base_z(static_cast<const blsSecretKey*>(r->a)->d, d)) { sgn[ngls++] = r; dig.insert(dig.end(), d, d + 4); }
            else rest.push_back(r);
        }
        std::copy(rest.begin(), rest.end(), sgn.begin() + ngls);
    }
    const size_t nv = ver.size(), ns = sgn.size(), np = pub.size(), n1 = one.size(), nh = nv + ns;
    // H(m): one table entry per distinct message of the verify and sign requests (the key hm_key builds); entries the cache holds at
    // the back, the misses at the front (contiguous: one hash launch), idx[i] = entry of request i (verify requests, then sign)
    std::vector<std::array<uint8_t, 48>> keys; std::vector<uint32_t> idx(nh);
    {
        std::map<std::array<uint8_t, 48>, uint32_t> seen;
        for (size_t i = 0; i < nh; i++) {
            const Part1Req* r = i < nv ? ver[i] : sgn[i - nv];
            std::array<uint8_t, 48> k; hm_key(k.data(), r->msg, r->len);
            auto it = seen.emplace(k, (uint32_t)keys.size());
            if (it.second) keys.push_back(k);
            idx[i] = it.first->second;
        }
    }
    const size_t nk = keys.size();
    std::vector<uint32_t> pos(nk); std::vector<bool> cached(nk, false); size_t nmiss = 0;
    for (size_t d = 0; d < nk; d++) cached[d] = hm_enabled() && hm_find(keys[d].data()) >= 0;
    for (size_t d = 0, hit = 0; d < nk; d++) pos[d] = cached[d] ? (uint32_t)(nk - 1 - hit++) : (uint32_t)nmiss++;
    bool gather = nk != nh;
    for (size_t i = 0; i < nh; i++) { idx[i] = pos[idx[i]]; gather |= idx[i] != i; }
    // staging (host -> device, one copy) and results (device -> host, one copy)
    Layout in, out;
    const size_t i_apk = d_apk ? 0 : in.put(nv * sizeof(g1)), i_sig = in.put(sig96 ? 96 : (nv - nser) * sizeof(g2)), i_keys = in.put(nmiss * 48);
    // AGG / MASK: the serialized signatures, the decode flags of every verify request, the mask_item descriptors and their bitmaps
    const size_t i_ser = nser ? in.put(nser * 96) : 0, i_sok = nser ? in.put(nv) : 0;
    const size_t i_items = na ? in.put(na * sizeof(mask_item)) : 0, i_bm = na ? in.put(bm_bytes) : 0;
    const size_t i_idx = gather ? in.put(nh * 4) : 0, i_dig = in.put(dig.size() * 8), i_sk = in.put((ns - ngls) * 32), i_pub = in.put(np * 32);
    std::vector<size_t> i_a(n1), i_b(n1), o_out(n1);
    for (size_t j = 0; j < n1; j++) { i_a[j] = in.put(one[j]->an); i_b[j] = in.put(one[j]->bn); o_out[j] = out.put(one[j]->on); }
    const size_t i_desc = n1 > 1 ? in.put(n1 * sizeof(single_desc)) : 0;
    const size_t o_res = out.put(nv), o_sig = out.put(ns * sizeof(g2)), o_sok = out.put(ns), o_pub = out.put(np * sizeof(g1)), o_rc = out.put(n1 * sizeof(int));
    Scratch* sc;
    if (int e = reserve(s, in.size + out.size + nv * (sizeof(g1a) + sizeof(g2a) + 1) + (nk + nh) * (sizeof(g2a) + 1) + 16 * 256, &sc)) return e;
    Arena ar{sc->base, 0, sc->cap};
    uint8_t* din = ar.take<uint8_t>(in.size); uint8_t* dout = ar.take<uint8_t>(out.size);
    g1a* pkneg = ar.take<g1a>(nv); g2a* vsig = ar.take<g2a>(nv); uint8_t* ok_sig = ar.take<uint8_t>(nv);
    g2a* hm = ar.take<g2a>(nh); uint8_t* ok_hm = ar.take<uint8_t>(nh);
    g2a* th = gather ? ar.take<g2a>(nk) : hm; uint8_t* tok = gather ? ar.take<uint8_t>(nk) : ok_hm;      // the H(m) table
    std::vector<uint8_t> hin(in.size), hout(out.size);
    for (size_t i = nser; i < nv && !d_apk; i++) memcpy(&hin[i_apk + i * sizeof(g1)], ver[i]->b, sizeof(g1));
    if (sig96) memcpy(&hin[i_sig], sig96, 96);
    else for (size_t i = nser; i < nv; i++) memcpy(&hin[i_sig + (i - nser) * sizeof(g2)], ver[i]->a, sizeof(g2));
    if (nser) {
        for (size_t i = 0; i < nser; i++) memcpy(&hin[i_ser + 96 * i], ver[i]->a, 96);
        memset(&hin[i_sok], 1, nv);                      // VERIFY structs count as decoded; the decode writes the first nser flags
        for (size_t i = 0, off = 0; i < na; i++) {
            const Part1Req& r = *ver[i];
            const mask_item it{r.com->table, din + i_bm + off, (uint64_t)r.com->n};
            memcpy(&hin[i_items + i * sizeof(mask_item)], &it, sizeof it);
            if (r.blen) memcpy(&hin[i_bm + off], r.bitmap, r.blen);
            off += r.blen;
        }
    }
    for (size_t d = 0; d < nk; d++) if (!cached[d]) memcpy(&hin[i_keys + 48 * pos[d]], keys[d].data(), 48);
    if (gather) memcpy(&hin[i_idx], idx.data(), nh * 4);
    if (!dig.empty()) memcpy(&hin[i_dig], dig.data(), dig.size() * 8);
    for (size_t i = ngls; i < ns; i++) memcpy(&hin[i_sk + 32 * (i - ngls)], static_cast<const blsSecretKey*>(sgn[i]->a)->d, 32);
    for (size_t i = 0; i < np; i++) memcpy(&hin[i_pub + 32 * i], static_cast<const blsSecretKey*>(pub[i]->a)->d, 32);
    std::vector<single_desc> desc(n1);
    for (size_t j = 0; j < n1; j++) {
        if (one[j]->an) memcpy(&hin[i_a[j]], one[j]->a, one[j]->an);
        if (one[j]->bn) memcpy(&hin[i_b[j]], one[j]->b, one[j]->bn);
        desc[j] = single_desc{din + i_a[j], din + i_b[j], dout + o_out[j], one[j]->op, (uint32_t)one[j]->len};
    }
    if (n1 > 1) memcpy(&hin[i_desc], desc.data(), n1 * sizeof(single_desc));
    CK(cudaMemcpyAsync(din, hin.data(), in.size, cudaMemcpyHostToDevice, s));
    int* drc = reinterpret_cast<int*>(dout + o_rc);
    if (n1) LAUNCH(k_single, blocks_for(n1, 32), 32, s, n1, n1 > 1 ? (const single_desc*)(din + i_desc) : (const single_desc*)nullptr, desc[0], drc);
    if (np) LAUNCH(k_g1_mul_gen, blocks_for(np, 32), 32, s, np, (const uint8_t*)(din + i_pub), reinterpret_cast<g1*>(dout + o_pub));
    const uint8_t* vok_sig = nullptr;
    if (nv) {
        g1* apk = reinterpret_cast<g1*>(din + i_apk);
        if (na) LAUNCH(k_mask_aggregate_items, blocks_for(na * 32, 128), 128, s, na, (const mask_item*)(din + i_items), apk);
        for (size_t i = na; i < nser; i++) CK(cudaMemcpyAsync(apk + i, ver[i]->mask->d_acc, sizeof(g1), cudaMemcpyDeviceToDevice, s));
        LAUNCH(k_g1_normalize_lat, blocks_for(nv, 32), 32, s, nv, d_apk ? d_apk : (const g1*)apk, pkneg, 1);
        if (sig96) { LAUNCH(k_g2_decode_pair, 1, 32, s, (size_t)1, (const uint8_t*)(din + i_sig), vsig, ok_sig, 1); vok_sig = ok_sig; }
        else {
            if (nser) { LAUNCH(k_g2_decode_pair, blocks_for(2 * nser, 32), 32, s, nser, (const uint8_t*)(din + i_ser), vsig, din + i_sok, 1); vok_sig = din + i_sok; }
            if (nv > nser) LAUNCH(k_g2_normalize, blocks_for(nv - nser, 32), 32, s, nv - nser, reinterpret_cast<const g2*>(din + i_sig), vsig + nser);
        }
    }
    // H(m): cached entries (this node signed, verified or prefetched the message before), then one launch over the misses
    for (size_t d = 0; d < nk; d++) if (cached[d]) hm_fetch(keys[d].data(), th + pos[d], tok + pos[d], s);
    if (hm_enabled()) g.hm_misses += nmiss;
    if (nmiss) {
        launch_hash_small(s, nmiss, din + i_keys, 48, th, tok);
        if (hm_enabled()) for (size_t d = 0; d < nk; d++) if (!cached[d]) hm_store(keys[d].data(), th + pos[d], tok + pos[d], s);
    }
    if (gather) LAUNCH(k_broadcast_hm, blocks_for(nh, 256), 256, s, nh, (const uint32_t*)(din + i_idx), (const g2a*)th, (const uint8_t*)tok, hm, ok_hm);
    if (nv) {
        uint8_t* dres = dout + o_res;
        const size_t coop_cap = (size_t)g.sm_count * (size_t)(g.coop_wpsm > 0 ? g.coop_wpsm : 1);
        if (g.coop_max >= 1) LAUNCH(k_pairing_coop, (unsigned)(nv < coop_cap ? nv : coop_cap), 32, s, nv, vsig, pkneg, hm, (const uint8_t*)ok_hm, vok_sig, (const uint8_t*)nullptr, dres);
        else LAUNCH(k_pairing_verify_split, blocks_for(2 * nv, 64), 64, s, nv, vsig, pkneg, hm, (const uint8_t*)ok_hm, vok_sig, (const uint8_t*)nullptr, dres, (const int*)nullptr);
        LAUNCH(k_pairing_fixup, blocks_for(nv, 32), 32, s, nv, vsig, pkneg, hm, (const uint8_t*)ok_hm, vok_sig, (const uint8_t*)nullptr, dres, (const int*)nullptr);
    }
    g2* dsig_out = reinterpret_cast<g2*>(dout + o_sig); uint8_t* dsok = dout + o_sok;
    if (ngls) LAUNCH(k_sign_hm_gls_pair, blocks_for(2 * ngls, 32), 32, s, ngls, (const uint64_t*)(din + i_dig), hm + nv, (const uint8_t*)ok_hm + nv, (size_t)1, dsig_out, dsok);
    if (ns > ngls) LAUNCH(k_sign_hm_pair, blocks_for(2 * (ns - ngls), 32), 32, s, ns - ngls, (const uint8_t*)(din + i_sk), hm + nv + ngls, (const uint8_t*)ok_hm + nv + ngls,
                          (size_t)1, dsig_out + ngls, dsok + ngls);
    CK(cudaGetLastError());
    CK(cudaMemcpyAsync(hout.data(), dout, out.size, cudaMemcpyDeviceToHost, s));
    CK(cudaStreamSynchronize(s));
    if (na) {            // committee checks in the turn: an exact-mode batch of na rounds, a warp per round (hbls_last_batch_info)
        g.info = hbls_batch_info{}; g.info.mode = 0; g.info.rounds = na; g.info.cta_threads = 32;
        sc->h_counts[0] = sc->h_counts[1] = 0;
        CK(cudaEventRecord(sc->done, s));
        g.info_sc = sc; g.info_valid = true;
    }
    for (size_t i = 0; i < nv; i++) ver[i]->rc = hout[o_res + i] ? 1 : 0;
    for (size_t i = 0; i < ns; i++) { memcpy(sgn[i]->out, &hout[o_sig + i * sizeof(g2)], sizeof(g2)); sgn[i]->rc = hout[o_sok + i] ? 0 : -1; }
    for (size_t i = 0; i < np; i++) memcpy(pub[i]->out, &hout[o_pub + i * sizeof(g1)], sizeof(g1));
    for (size_t j = 0; j < n1; j++) {
        Part1Req& r = *one[j]; int rc; memcpy(&rc, &hout[o_rc + j * sizeof(int)], sizeof(int));
        if (r.on && rc >= 0 && !((r.op == OP_G1_DES || r.op == OP_G2_DES) && rc == 0) && !(r.op == OP_MAP_SER && rc != 0)) memcpy(r.out, &hout[o_out[j]], r.on);
        r.rc = rc;
    }
    return 0;
}

int agg_verify_one_locked(Part1Req& r);       // a lone AGG request: the path of hbls_aggregate_verify_batch with one round

// runs r in a turn of the combiner (from any thread; the caller must not hold g.mu).  A turn of one AGG or MASK request runs the
// launches its call made before it could be combined: the three-stream latency path of one round, or part1_locked on the mask's key.
void part1_submit(Part1Req& r) {
    g.part1.submit(r, g.mu,
        [](int kind) { return kind == RQ_VERIFY ? (size_t)(g.coop_max > 0 ? g.coop_max : 1) : PART1_CAP; },
        [](hbls_coalesce::Request** rq, size_t n) {
            std::vector<Part1Req*> turn(n);
            for (size_t i = 0; i < n; i++) turn[i] = static_cast<Part1Req*>(rq[i]);
            Part1Req& r0 = *turn[0];
            int e;
            if (n == 1 && r0.kind == RQ_AGG) e = agg_verify_one_locked(r0);
            else if (n == 1 && r0.kind == RQ_MASK) e = part1_locked(turn.data(), 1, r0.mask->d_acc, static_cast<const uint8_t*>(r0.a));
            else e = part1_locked(turn.data(), n);
            for (Part1Req* r : turn) r->err = e;
        },
        [](int kind) { return is_verify(kind) ? (int)RQ_VERIFY : kind; });
}
int single_op(int op, const void* a, size_t an, const void* b, size_t bn, void* out, size_t on, int* rc_out, uint32_t len = 0) {
    if (int e = ensure_init()) return e;
    Part1Req r; r.kind = RQ_SINGLE; r.op = op; r.a = a; r.an = an; r.b = b; r.bn = bn; r.out = out; r.on = on; r.len = len;
    part1_submit(r);
    if (r.err) return r.err;
    *rc_out = r.rc;
    return 0;
}

// SHA-256 (host; GetAddress = first 20 bytes of SHA-256 of the serialized key)
struct Sha256 {
    static uint32_t rotr(uint32_t x, int n) { return (x >> n) | (x << (32 - n)); }
    static void digest(const uint8_t* msg, size_t len, uint8_t out[32]) {
        static const uint32_t K[64] = {
            0x428a2f98,0x71374491,0xb5c0fbcf,0xe9b5dba5,0x3956c25b,0x59f111f1,0x923f82a4,0xab1c5ed5,0xd807aa98,0x12835b01,0x243185be,0x550c7dc3,0x72be5d74,0x80deb1fe,0x9bdc06a7,0xc19bf174,
            0xe49b69c1,0xefbe4786,0x0fc19dc6,0x240ca1cc,0x2de92c6f,0x4a7484aa,0x5cb0a9dc,0x76f988da,0x983e5152,0xa831c66d,0xb00327c8,0xbf597fc7,0xc6e00bf3,0xd5a79147,0x06ca6351,0x14292967,
            0x27b70a85,0x2e1b2138,0x4d2c6dfc,0x53380d13,0x650a7354,0x766a0abb,0x81c2c92e,0x92722c85,0xa2bfe8a1,0xa81a664b,0xc24b8b70,0xc76c51a3,0xd192e819,0xd6990624,0xf40e3585,0x106aa070,
            0x19a4c116,0x1e376c08,0x2748774c,0x34b0bcb5,0x391c0cb3,0x4ed8aa4a,0x5b9cca4f,0x682e6ff3,0x748f82ee,0x78a5636f,0x84c87814,0x8cc70208,0x90befffa,0xa4506ceb,0xbef9a3f7,0xc67178f2};
        uint32_t h[8] = {0x6a09e667,0xbb67ae85,0x3c6ef372,0xa54ff53a,0x510e527f,0x9b05688c,0x1f83d9ab,0x5be0cd19};
        std::vector<uint8_t> m(msg, msg + len);
        m.push_back(0x80);
        while (m.size() % 64 != 56) m.push_back(0);
        uint64_t bits = (uint64_t)len * 8;
        for (int i = 7; i >= 0; i--) m.push_back((uint8_t)(bits >> (8 * i)));
        for (size_t off = 0; off < m.size(); off += 64) {
            uint32_t w[64];
            for (int i = 0; i < 16; i++) w[i] = ((uint32_t)m[off + 4 * i] << 24) | ((uint32_t)m[off + 4 * i + 1] << 16) | ((uint32_t)m[off + 4 * i + 2] << 8) | m[off + 4 * i + 3];
            for (int i = 16; i < 64; i++) {
                uint32_t s0 = rotr(w[i - 15], 7) ^ rotr(w[i - 15], 18) ^ (w[i - 15] >> 3), s1 = rotr(w[i - 2], 17) ^ rotr(w[i - 2], 19) ^ (w[i - 2] >> 10);
                w[i] = w[i - 16] + s0 + w[i - 7] + s1;
            }
            uint32_t a = h[0], b = h[1], c = h[2], d = h[3], e = h[4], f = h[5], gg = h[6], hh = h[7];
            for (int i = 0; i < 64; i++) {
                uint32_t S1 = rotr(e, 6) ^ rotr(e, 11) ^ rotr(e, 25), ch = (e & f) ^ (~e & gg), t1 = hh + S1 + ch + K[i] + w[i];
                uint32_t S0 = rotr(a, 2) ^ rotr(a, 13) ^ rotr(a, 22), mj = (a & b) ^ (a & c) ^ (b & c), t2 = S0 + mj;
                hh = gg; gg = f; f = e; e = d + t1; d = c; c = b; b = a; a = t1 + t2;
            }
            h[0] += a; h[1] += b; h[2] += c; h[3] += d; h[4] += e; h[5] += f; h[6] += gg; h[7] += hh;
        }
        for (int i = 0; i < 8; i++) for (int j = 0; j < 4; j++) out[4 * i + j] = (uint8_t)(h[i] >> (24 - 8 * j));
    }
};

// SHA-512 (host; only for the test-only blsSign/blsVerify string API: mcl Fp::setHashOf, SURVEY A.7)
struct Sha512 {
    static uint64_t rotr(uint64_t x, int n) { return (x >> n) | (x << (64 - n)); }
    static void digest(const uint8_t* msg, size_t len, uint8_t out[64]) {
        static const uint64_t K[80] = {
            0x428a2f98d728ae22ull,0x7137449123ef65cdull,0xb5c0fbcfec4d3b2full,0xe9b5dba58189dbbcull,0x3956c25bf348b538ull,0x59f111f1b605d019ull,0x923f82a4af194f9bull,0xab1c5ed5da6d8118ull,
            0xd807aa98a3030242ull,0x12835b0145706fbeull,0x243185be4ee4b28cull,0x550c7dc3d5ffb4e2ull,0x72be5d74f27b896full,0x80deb1fe3b1696b1ull,0x9bdc06a725c71235ull,0xc19bf174cf692694ull,
            0xe49b69c19ef14ad2ull,0xefbe4786384f25e3ull,0x0fc19dc68b8cd5b5ull,0x240ca1cc77ac9c65ull,0x2de92c6f592b0275ull,0x4a7484aa6ea6e483ull,0x5cb0a9dcbd41fbd4ull,0x76f988da831153b5ull,
            0x983e5152ee66dfabull,0xa831c66d2db43210ull,0xb00327c898fb213full,0xbf597fc7beef0ee4ull,0xc6e00bf33da88fc2ull,0xd5a79147930aa725ull,0x06ca6351e003826full,0x142929670a0e6e70ull,
            0x27b70a8546d22ffcull,0x2e1b21385c26c926ull,0x4d2c6dfc5ac42aedull,0x53380d139d95b3dfull,0x650a73548baf63deull,0x766a0abb3c77b2a8ull,0x81c2c92e47edaee6ull,0x92722c851482353bull,
            0xa2bfe8a14cf10364ull,0xa81a664bbc423001ull,0xc24b8b70d0f89791ull,0xc76c51a30654be30ull,0xd192e819d6ef5218ull,0xd69906245565a910ull,0xf40e35855771202aull,0x106aa07032bbd1b8ull,
            0x19a4c116b8d2d0c8ull,0x1e376c085141ab53ull,0x2748774cdf8eeb99ull,0x34b0bcb5e19b48a8ull,0x391c0cb3c5c95a63ull,0x4ed8aa4ae3418acbull,0x5b9cca4f7763e373ull,0x682e6ff3d6b2b8a3ull,
            0x748f82ee5defb2fcull,0x78a5636f43172f60ull,0x84c87814a1f0ab72ull,0x8cc702081a6439ecull,0x90befffa23631e28ull,0xa4506cebde82bde9ull,0xbef9a3f7b2c67915ull,0xc67178f2e372532bull,
            0xca273eceea26619cull,0xd186b8c721c0c207ull,0xeada7dd6cde0eb1eull,0xf57d4f7fee6ed178ull,0x06f067aa72176fbaull,0x0a637dc5a2c898a6ull,0x113f9804bef90daeull,0x1b710b35131c471bull,
            0x28db77f523047d84ull,0x32caab7b40c72493ull,0x3c9ebe0a15c9bebcull,0x431d67c49c100d4cull,0x4cc5d4becb3e42b6ull,0x597f299cfc657e2aull,0x5fcb6fab3ad6faecull,0x6c44198c4a475817ull};
        uint64_t h[8] = {0x6a09e667f3bcc908ull,0xbb67ae8584caa73bull,0x3c6ef372fe94f82bull,0xa54ff53a5f1d36f1ull,0x510e527fade682d1ull,0x9b05688c2b3e6c1full,0x1f83d9abfb41bd6bull,0x5be0cd19137e2179ull};
        std::vector<uint8_t> m(msg, msg + len);
        m.push_back(0x80);
        while (m.size() % 128 != 112) m.push_back(0);
        for (int i = 0; i < 8; i++) m.push_back(0);
        uint64_t bits = (uint64_t)len * 8;
        for (int i = 7; i >= 0; i--) m.push_back((uint8_t)(bits >> (8 * i)));
        for (size_t off = 0; off < m.size(); off += 128) {
            uint64_t w[80];
            for (int i = 0; i < 16; i++) { w[i] = 0; for (int j = 0; j < 8; j++) w[i] = (w[i] << 8) | m[off + 8 * i + j]; }
            for (int i = 16; i < 80; i++) {
                uint64_t s0 = rotr(w[i - 15], 1) ^ rotr(w[i - 15], 8) ^ (w[i - 15] >> 7);
                uint64_t s1 = rotr(w[i - 2], 19) ^ rotr(w[i - 2], 61) ^ (w[i - 2] >> 6);
                w[i] = w[i - 16] + s0 + w[i - 7] + s1;
            }
            uint64_t a = h[0], b = h[1], c = h[2], d = h[3], e = h[4], f = h[5], gg = h[6], hh = h[7];
            for (int i = 0; i < 80; i++) {
                uint64_t S1 = rotr(e, 14) ^ rotr(e, 18) ^ rotr(e, 41), ch = (e & f) ^ (~e & gg);
                uint64_t t1 = hh + S1 + ch + K[i] + w[i];
                uint64_t S0 = rotr(a, 28) ^ rotr(a, 34) ^ rotr(a, 39), mj = (a & b) ^ (a & c) ^ (b & c);
                uint64_t t2 = S0 + mj;
                hh = gg; gg = f; f = e; e = d + t1; d = c; c = b; b = a; a = t1 + t2;
            }
            h[0] += a; h[1] += b; h[2] += c; h[3] += d; h[4] += e; h[5] += f; h[6] += gg; h[7] += hh;
        }
        for (int i = 0; i < 8; i++) for (int j = 0; j < 8; j++) out[8 * i + j] = (uint8_t)(h[i] >> (56 - 8 * j));
    }
};

}  // namespace

struct hbls_ballot_box {
    const hbls_committee* c = nullptr;
    std::vector<uint8_t> collected;     // signers already counted
    g2* d_sum = nullptr;                // running aggregate signature (device, Jacobian)
    ~hbls_ballot_box() { if (d_sum) cudaFree(d_sum); }
};

namespace {
int popcount_slots(const uint8_t* bm, size_t n) {          // set bits among slots i < n only (padding bits of the last byte never count)
    int c = 0;
    for (size_t i = 0; i < (n >> 3); i++) c += __builtin_popcount(bm[i]);
    if (n & 7) c += __builtin_popcount(bm[n >> 3] & ((1u << (n & 7)) - 1u));
    return c;
}
bool all_messages_equal(const uint8_t* msgs, size_t n, size_t msg_len) {
    for (size_t i = 1; i < n; i++) if (memcmp(msgs, msgs + i * msg_len, msg_len) != 0) return false;
    return n > 1;
}
// serial mask aggregation of large batches: rounds sorted by the number of point additions they need (device counting sort, when
// mask_sort is on), so that the lanes of a warp finish together; v.apk receives the Jacobian sums
void launch_mask_serial(const hbls_committee* c, size_t B, const uint8_t* d_bitmaps, size_t blen, const VerifyBufs& v, cudaStream_t s) {
    const uint32_t* order = nullptr;
    if (g.mask_sort && B <= 0xffffffffull) {
        cudaMemsetAsync(v.mask_hist, 0, HB_MASK_BINS * sizeof(unsigned), s);
        LAUNCH(k_mask_count, blocks_for(B, 256), 256, s, B, c->n, d_bitmaps, blen, v.mask_cost, v.mask_hist);
        LAUNCH(k_mask_scan, 1, 32, s, v.mask_hist);
        LAUNCH(k_mask_scatter, blocks_for(B, 256), 256, s, B, v.mask_cost, v.mask_hist, v.mask_order);
        order = v.mask_order;
    }
    LAUNCH(k_mask_aggregate_serial, light_blocks(B), TPB, s, B, c->n, c->table, c->total, d_bitmaps, blen, v.apk, order);
}
// rounds against one committee, everything device-resident
int agg_verify_device_locked(const hbls_committee* c, size_t B, const uint8_t* d_bitmaps, size_t blen, const uint8_t* d_sigs,
                             const uint8_t* d_msgs, size_t msg_len, uint8_t* d_results, cudaStream_t s, Scratch* sc, Arena& ar, bool same_msg,
                             VerifyBufs* v_out = nullptr, const uint8_t* h_msg = nullptr, const MsgGroups* mg = nullptr) {
    VerifyBufs v = carve_verify(ar, B);
    fork_point(B, sc, s);
    STAGE_EV(0, sc, s);
    if (B >= (size_t)g.sm_count * 256)
        launch_mask_serial(c, B, d_bitmaps, blen, v, s);
    else
        LAUNCH(k_mask_aggregate, blocks_for(B * 32, 128), 128, s, B, c->n, c->table, d_bitmaps, blen, v.apk);
    launch_verify_tail(B, v, sc, d_sigs, d_msgs, (uint32_t)msg_len, nullptr, d_results, s, same_msg, h_msg, mg);
    if (v_out) *v_out = v;
    return 0;
}
// Mask.SetMask with g.mu held (bitmap: m->bitmap.size() bytes)
int set_mask_locked(hbls_mask* m, const uint8_t* bitmap) {
    const size_t blen = m->bitmap.size(), n = m->c->n;
    std::vector<uint8_t> delta(2 * blen + 2, 0);                       // row 0: bits to Add (0 -> 1), row 1: bits to Sub (1 -> 0)
    bool any = false;
    for (size_t i = 0; i < n; i++) {                                   // only slots i < n exist (mask.go:121: for i := range m.Publics)
        const uint8_t msk = (uint8_t)(1u << (i & 7)); const bool was = m->bitmap[i >> 3] & msk, now = bitmap[i >> 3] & msk;
        if (!was && now) { delta[i >> 3] |= msk; any = true; }
        if (was && !now) { delta[blen + (i >> 3)] |= msk; any = true; }
    }
    if (!any) return 0;
    Scratch* sc; if (int e = reserve(g.stream, 2 * blen + 4096, &sc)) return e;
    Arena ar{sc->base, 0, sc->cap};
    uint8_t* dbm = ar.take<uint8_t>(2 * blen + 2); g1* dtmp = ar.take<g1>(2); int* drc = ar.take<int>(1);
    CK(cudaMemcpyAsync(dbm, delta.data(), 2 * blen, cudaMemcpyHostToDevice, g.stream));
    LAUNCH(k_mask_aggregate, 1, 64, g.stream, (size_t)2, n, m->c->table, dbm, blen, dtmp);
    LAUNCH(k_single, 1, 32, g.stream, (size_t)1, (const single_desc*)nullptr, single_desc{m->d_acc, dtmp + 0, m->d_acc, OP_G1_ADD, 0u}, drc);
    LAUNCH(k_single, 1, 32, g.stream, (size_t)1, (const single_desc*)nullptr, single_desc{m->d_acc, dtmp + 1, m->d_acc, OP_G1_SUB, 0u}, drc);
    CK(cudaStreamSynchronize(g.stream));
    for (size_t i = 0; i < n; i++) {
        const uint8_t msk = (uint8_t)(1u << (i & 7));
        m->bitmap[i >> 3] = (uint8_t)((m->bitmap[i >> 3] & ~msk) | (bitmap[i >> 3] & msk));
    }
    return 0;
}
void ensure_stage_events(Scratch* sc) {
    if (g.stage_timing && !sc->ev_ok) { for (int i = 0; i < 8; i++) cudaEventCreate(&sc->ev[i]); sc->ev_ok = true; }
}
}  // namespace

int self_test_at_init();      // selftest.cuh: HBLS_SELF_TEST=1 runs hbls_self_test here

extern "C" {

int hbls_init_device(int device) {
    std::lock_guard<std::mutex> lk(g.mu);
    if (g.st_failed) return HBLS_ERR_SELF_TEST;
    if (g.ready) return 0;
    int count = 0;
    cudaError_t e = cudaGetDeviceCount(&count);
    if (e != cudaSuccess || count == 0) {
        fprintf(stderr, "[hbls] no CUDA device (%s): this backend has no CPU fallback\n", e == cudaSuccess ? "count = 0" : cudaGetErrorString(e));
        return HBLS_ERR_CUDA;
    }
    if (device < 0 || device >= count) device = 0;
    CK(cudaSetDevice(device));
    cudaDeviceProp prop; CK(cudaGetDeviceProperties(&prop, device));
    g.device = device; g.sm_count = prop.multiProcessorCount;
    CK(cudaStreamCreateWithFlags(&g.stream, cudaStreamNonBlocking));
    CK(cudaStreamCreateWithFlags(&g.aux[0], cudaStreamNonBlocking)); CK(cudaStreamCreateWithFlags(&g.aux[1], cudaStreamNonBlocking));
    { FILE* f = fopen("/dev/urandom", "rb"); if (!f || fread(g.chacha_key, 1, 32, f) != 32) { if (f) fclose(f); fprintf(stderr, "[hbls] cannot read /dev/urandom\n"); return HBLS_ERR_CUDA; } fclose(f); }
    auto envll = [](const char* name, long long dflt) { const char* e = getenv(name); return e ? atoll(e) : dflt; };
    g.rlc_min = envll("HBLS_RLC_MIN", 12288); g.rlc_g = envll("HBLS_RLC_G", 0); g.coop_max = envll("HBLS_COOP_MAX", 4096);
    g.tpsm = envll("HBLS_TPSM", 384); g.tpsm_split = envll("HBLS_TPSM_SPLIT", 512); g.tpsm_light = envll("HBLS_TPSM_LIGHT", 1024);
    // the heavy kernels keep their Fp12 temporaries in per-thread local memory: give L1 the whole 228 KB
#if HB_SMEM_F
    CK(cudaFuncSetAttribute(k_rlc_pairing_split<4>, cudaFuncAttributeMaxDynamicSharedMemorySize, HB_TPB_SPLIT * HB_SMEM_F_WORDS * 4));
    CK(cudaFuncSetAttribute(k_rlc_pairing_split<8>, cudaFuncAttributeMaxDynamicSharedMemorySize, HB_TPB_SPLIT * HB_SMEM_F_WORDS * 4));
#else
    CK(cudaFuncSetAttribute(k_rlc_pairing_split<4>, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxL1));
    CK(cudaFuncSetAttribute(k_rlc_pairing_split<8>, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxL1));
#endif
    CK(cudaFuncSetAttribute(k_rlc_lines_split<1>, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxL1));
    CK(cudaFuncSetAttribute(k_rlc_accum_split<1>, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxL1));
    CK(cudaFuncSetAttribute(k_rlc_lines_split<4>, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxL1));
    CK(cudaFuncSetAttribute(k_rlc_lines_split<8>, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxL1));
    CK(cudaFuncSetAttribute(k_rlc_accum_split<4>, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxL1));
    CK(cudaFuncSetAttribute(k_rlc_accum_split<8>, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxL1));
    CK(cudaFuncSetAttribute(k_pairing_verify_split, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxL1));
    CK(cudaFuncSetAttribute(k_pairing_verify_split_list, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxL1));
    CK(cudaFuncSetAttribute(k_hash_to_g2, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxL1));
    CK(cudaFuncSetAttribute(k_g2_decode, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxL1));
    CK(cudaFuncSetAttribute(k_rlc_scale, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxL1));
    CK(cudaFuncSetAttribute(k_mask_aggregate_serial, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxL1));
    CK(cudaFuncSetAttribute(k_mask_aggregate, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxL1));
    CK(cudaMalloc(&g.hm_slots, Ctx::HM_N * sizeof(g2a))); CK(cudaMalloc(&g.hm_ok, Ctx::HM_N));
    CK(cudaMalloc(&g.rlc_form, sizeof(int))); CK(cudaMemset(g.rlc_form, 0, sizeof(int)));
    for (int i = 0; i < Ctx::HM_N; i++) {
        CK(cudaEventCreateWithFlags(&g.hm[i].filled, cudaEventDisableTiming)); CK(cudaEventCreateWithFlags(&g.hm[i].read_done, cudaEventDisableTiming));
    }
    g.hm_cache = envll("HBLS_HM_CACHE", 1); g.mask_sort = envll("HBLS_MASK_SORT", 1); g.hash_coop_max = envll("HBLS_HASH_COOP_MAX", 4ll * g.sm_count);     // one warp per message while every scheduler gets one
    g.rlc_two_phase = envll("HBLS_RLC_2P", 2); g.tpsm_lines = envll("HBLS_TPSM_LINES", 512); g.tpsm_accum = envll("HBLS_TPSM_ACCUM", 512); g.tpsm_cof = envll("HBLS_TPSM_COF", 512); g.tpsm_dec = envll("HBLS_TPSM_DEC", 512); g.tpsm_sub = envll("HBLS_TPSM_SUB", 512); g.tpsm_scale = envll("HBLS_TPSM_SCALE", 384); g.tpsm_scale_g1 = envll("HBLS_TPSM_SCALE_G1", 384); g.tpsm_scale_g2 = envll("HBLS_TPSM_SCALE_G2", 512); g.scale_split = envll("HBLS_SCALE_SPLIT", 1); g.scale_joint = envll("HBLS_SCALE_JOINT", 1); g.decode_split = envll("HBLS_DECODE_SPLIT", 1); g.exact_two_phase = envll("HBLS_EXACT_2P", 1);
    g.rlc_block = envll("HBLS_RLC_BLOCK", 0);
    g.hash_split = envll("HBLS_HASH_SPLIT", 2); g.tpsm_sw = envll("HBLS_TPSM_SW", 512);
    CK(cudaFuncSetAttribute(k_hash_sw, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxL1));
    CK(cudaFuncSetAttribute(k_hash_cofactor, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxL1));
    CK(cudaFuncSetAttribute(k_hash_cofactor_pair, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxL1));
    CK(cudaFuncSetAttribute(k_g2_normalize_batch, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxL1));
    g.ready = true;
    return self_test_at_init();
}
int blsInit(int curve, int compiledTimeVar) {
    if (curve != HBLS_BLS12_381 || compiledTimeVar != HBLS_COMPILED_TIME_VAR) return -1;
    const char* d = getenv("HBLS_DEVICE");
    if (!d) d = getenv("LOCAL_RANK");
    return hbls_init_device(d ? atoi(d) : 0);
}
uint64_t hbls_kernel_launch_count(void) { return g.launches.load(); }
int hbls_build_info(void) { return (HB_BATCH_INV ? 1 : 0) | (HB_BATCH_K << 8); }
int hbls_get_device(void) { if (int e = ensure_init()) return e; std::lock_guard<std::mutex> lk(g.mu); return g.device; }
void hbls_set_batch_mode(int mode) { std::lock_guard<std::mutex> lk(g.mu); g.batch_mode = mode ? 1 : 0; }
int hbls_get_batch_mode(void) { std::lock_guard<std::mutex> lk(g.mu); return g.batch_mode; }
// tuning knobs by name (hbls_set_param); the self-test saves and restores all of them
struct ParamDef { const char* name; long long Ctx::* slot; };
const ParamDef PARAMS[] = {
    {"rlc_min", &Ctx::rlc_min}, {"rlc_g", &Ctx::rlc_g}, {"tpsm", &Ctx::tpsm}, {"tpsm_split", &Ctx::tpsm_split}, {"tpsm_light", &Ctx::tpsm_light}, {"coop_max", &Ctx::coop_max},
    {"overlap", &Ctx::overlap}, {"coop_wpsm", &Ctx::coop_wpsm}, {"hm_cache", &Ctx::hm_cache}, {"hash_coop_max", &Ctx::hash_coop_max}, {"mask_sort", &Ctx::mask_sort}, {"hash_split", &Ctx::hash_split},
    {"hash_fallback", &Ctx::hash_fallback}, {"rlc_two_phase", &Ctx::rlc_two_phase}, {"tpsm_cof", &Ctx::tpsm_cof}, {"tpsm_dec", &Ctx::tpsm_dec}, {"tpsm_sub", &Ctx::tpsm_sub}, {"tpsm_scale", &Ctx::tpsm_scale}, {"tpsm_scale_g1", &Ctx::tpsm_scale_g1}, {"tpsm_scale_g2", &Ctx::tpsm_scale_g2},
    {"scale_split", &Ctx::scale_split}, {"decode_split", &Ctx::decode_split}, {"exact_two_phase", &Ctx::exact_two_phase}, {"tpsm_lines", &Ctx::tpsm_lines}, {"tpsm_accum", &Ctx::tpsm_accum}, {"tpsm_sw", &Ctx::tpsm_sw},
    {"rlc_block", &Ctx::rlc_block}, {"scale_joint", &Ctx::scale_joint}, {"selftest_flip", &Ctx::selftest_flip}};
static long long* param_slot(const char* name) {
    if (!name) return nullptr;
    for (const ParamDef& p : PARAMS) if (!strcmp(name, p.name)) return &(g.*p.slot);
    return nullptr;
}
int hbls_set_param(const char* name, long long value) {
    std::lock_guard<std::mutex> lk(g.mu);
    long long* p = param_slot(name);
    if (!p || value < 0) return HBLS_ERR_ARG;
    if (p == &g.rlc_g && value != 0 && value != 4 && value != 8) return HBLS_ERR_ARG;
    if ((p == &g.rlc_block || p == &g.scale_joint) && value > 2) return HBLS_ERR_ARG;
    *p = value; return 0;
}
long long hbls_get_param(const char* name) { std::lock_guard<std::mutex> lk(g.mu); long long* p = param_slot(name); return p ? *p : -1; }
int hbls_last_error(char* msg, size_t msg_cap) {
    std::lock_guard<std::mutex> lk(g.mu);
    int e = g.last_err;
    if (msg && msg_cap) { strncpy(msg, g.last_err_msg, msg_cap - 1); msg[msg_cap - 1] = 0; }
    g.last_err = 0; g.last_err_msg[0] = 0;
    return e;
}
int hbls_last_batch_info(hbls_batch_info* out) {
    std::lock_guard<std::mutex> lk(g.mu);
    if (!out || !g.info_valid || !g.info_sc) return HBLS_ERR_ARG;
    CK(cudaEventSynchronize(g.info_sc->done));
    *out = g.info;
    out->rounds_rechecked = g.info_sc->h_counts[0]; out->groups_failed = g.info_sc->h_counts[1];
    return 0;
}

// ------------------------------------------------------------------ secret keys (host bytes; no group arithmetic)
int blsSecretKeySetByCSPRNG(blsSecretKey* sec) {
    if (g.st_failed) return -1;
    FILE* f = fopen("/dev/urandom", "rb");
    if (!f) return -1;
    size_t got = fread(sec->d, 1, 32, f); fclose(f);
    if (got != 32) return -1;
    sec->d[3] &= 0x3fffffffffffffffull;          // < 2^254 < r
    return 0;
}
size_t blsSecretKeySerialize(void* buf, size_t maxBufSize, const blsSecretKey* sec) { if (maxBufSize < 32 || g.st_failed) return 0; memcpy(buf, sec->d, 32); return 32; }
size_t blsSecretKeyDeserialize(blsSecretKey* sec, const void* buf, size_t bufSize) {
    if (bufSize < 32 || g.st_failed) return 0;
    uint64_t k[4]; memcpy(k, buf, 32);
    if (!scalar_lt_r(k)) return 0;
    memcpy(sec->d, k, 32); return 32;
}
int blsSecretKeyIsEqual(const blsSecretKey* l, const blsSecretKey* r) { return !g.st_failed && memcmp(l, r, 32) == 0; }

// ------------------------------------------------------------------ single-element group ops.  The herumi signatures of Add / Sub /
// GetPublicKey are void: on a CUDA failure the destination becomes the identity and the error is kept for hbls_last_error().
void blsPublicKeyAdd(blsPublicKey* pub, const blsPublicKey* rhs) { int rc; if (single_op(OP_G1_ADD, pub, 144, rhs, 144, pub, 144, &rc)) memset(pub, 0, sizeof *pub); }
void blsPublicKeySub(blsPublicKey* pub, const blsPublicKey* rhs) { int rc; if (single_op(OP_G1_SUB, pub, 144, rhs, 144, pub, 144, &rc)) memset(pub, 0, sizeof *pub); }
void blsSignatureAdd(blsSignature* sig, const blsSignature* rhs) { int rc; if (single_op(OP_G2_ADD, sig, 288, rhs, 288, sig, 288, &rc)) memset(sig, 0, sizeof *sig); }
int blsPublicKeyIsEqual(const blsPublicKey* l, const blsPublicKey* r) { int rc = 0; if (single_op(OP_G1_EQ, l, 144, r, 144, nullptr, 0, &rc)) return 0; return rc; }
int blsSignatureIsEqual(const blsSignature* l, const blsSignature* r) { int rc = 0; if (single_op(OP_G2_EQ, l, 288, r, 288, nullptr, 0, &rc)) return 0; return rc; }
size_t blsPublicKeySerialize(void* buf, size_t maxBufSize, const blsPublicKey* pub) {
    if (maxBufSize < 48) return 0; int rc = 0; if (single_op(OP_G1_SER, pub, 144, nullptr, 0, buf, 48, &rc)) return 0; return rc == 48 ? 48 : 0; }
size_t blsSignatureSerialize(void* buf, size_t maxBufSize, const blsSignature* sig) {
    if (maxBufSize < 96) return 0; int rc = 0; if (single_op(OP_G2_SER, sig, 288, nullptr, 0, buf, 96, &rc)) return 0; return rc == 96 ? 96 : 0; }
size_t blsPublicKeyDeserialize(blsPublicKey* pub, const void* buf, size_t bufSize) {
    if (bufSize < 48) return 0; int rc = 0; if (single_op(OP_G1_DES, buf, 48, nullptr, 0, pub, 144, &rc)) return 0; return rc == 48 ? 48 : 0; }
size_t blsSignatureDeserialize(blsSignature* sig, const void* buf, size_t bufSize) {
    if (bufSize < 96) return 0; int rc = 0; if (single_op(OP_G2_DES, buf, 96, nullptr, 0, sig, 288, &rc)) return 0; return rc == 96 ? 96 : 0; }
int hbls_map_to_g2(const void* msg, size_t msg_len, uint8_t out96[96]) {
    if (msg_len > 48) msg_len = 48;      // only the first 48 bytes matter (SURVEY A.3)
    int rc = -1; if (int e = single_op(OP_MAP_SER, msg, msg_len, nullptr, 0, out96, 96, &rc, (uint32_t)msg_len)) return e; return rc; }
// asynchronous: enqueues H(msg) on the hash stream and returns; a later SignHash / VerifyHash / aggregate-verify of that message
// finds the point in the cache (stream-ordered after the fill).  0 ok (also when already cached or the cache is off).
int hbls_hash_prefetch(const void* msg, size_t msg_len) {
    if (int e = ensure_init()) return e;
    std::lock_guard<std::mutex> lk(g.mu);
    if (!hm_enabled()) return 0;
    if (msg_len > 48) msg_len = 48;
    uint8_t key[48]; hm_key(key, msg, msg_len);
    if (const int i = hm_find(key); i >= 0) { g.hm[i].stamp = ++g.hm_clock; return 0; }
    cudaStream_t st = g.aux[1];
    Scratch* sc; if (int e = reserve(st, 4096, &sc)) return e;
    Arena ar{sc->base, 0, sc->cap};
    uint8_t* dmsg = ar.take<uint8_t>(64); g2a* dhm = ar.take<g2a>(1); uint8_t* dok = ar.take<uint8_t>(1);
    // the 48 key bytes ARE the bytes hash_to_fp reads (pageable source: the runtime stages it before cudaMemcpyAsync returns)
    CK(cudaMemcpyAsync(dmsg, key, 48, cudaMemcpyHostToDevice, st));
    launch_hash_small(st, 1, dmsg, 48, dhm, dok);
    hm_store(key, dhm, dok, st);
    CK(cudaGetLastError());
    return 0;
}
int hbls_coalesce_stats(uint64_t* turns, uint64_t* requests, uint64_t* max_turn) {
    const hbls_coalesce::Stats st = g.part1.stats();
    if (turns) *turns = st.turns;
    if (requests) *requests = st.requests;
    if (max_turn) *max_turn = st.max_turn;
    return 0;
}
int hbls_hash_cache_stats(uint64_t* hits, uint64_t* misses) {
    std::lock_guard<std::mutex> lk(g.mu);
    if (hits) *hits = g.hm_hits;
    if (misses) *misses = g.hm_misses;
    return 0;
}
int hbls_get_address(const blsPublicKey* pub, uint8_t out20[20]) {
    uint8_t ser[48], dg[32];
    if (blsPublicKeySerialize(ser, 48, pub) != 48) return HBLS_ERR_CUDA;
    Sha256::digest(ser, 48, dg); memcpy(out20, dg, 20); return 0;
}

void blsGetPublicKey(blsPublicKey* pub, const blsSecretKey* sec) {
    memset(pub, 0, sizeof *pub);
    if (ensure_init()) return;
    Part1Req r; r.kind = RQ_PUBKEY; r.a = sec; r.out = pub;
    part1_submit(r);
}
int blsSignHash(blsSignature* sig, const blsSecretKey* sec, const void* h, size_t size) {
    if (int e = ensure_init()) return e;
    // H(m) on a lane pair (kept in the H(m) cache: the validator verifies the aggregate over the very message it signs here), then
    // the ladder sk * H: over psi with sk in base |z| (kernels.cuh k_sign_hm_gls_pair), else the 255-bit ladder on the split carrier
    Part1Req r; r.kind = RQ_SIGN; r.a = sec; r.msg = h; r.len = size; r.out = sig;
    part1_submit(r);
    return r.err ? r.err : r.rc;
}
int blsVerifyHash(const blsSignature* sig, const blsPublicKey* pub, const void* h, size_t size) {
    if (ensure_init()) return 0;
    Part1Req r; r.kind = RQ_VERIFY; r.a = sig; r.b = pub; r.msg = h; r.len = size;
    part1_submit(r);
    return !r.err && r.rc == 1 ? 1 : 0;
}
void blsSign(blsSignature* sig, const blsSecretKey* sec, const void* m, size_t size) {
    uint8_t dg[64]; Sha512::digest((const uint8_t*)m, size, dg);
    if (blsSignHash(sig, sec, dg, 64) != 0) memset(sig, 0, sizeof *sig);
}
int blsVerify(const blsSignature* sig, const blsPublicKey* pub, const void* m, size_t size) {
    uint8_t dg[64]; Sha512::digest((const uint8_t*)m, size, dg);
    return blsVerifyHash(sig, pub, dg, 64);
}

// ------------------------------------------------------------------ committee table
static int committee_create_locked(hbls_committee** out, const uint8_t* pk48, size_t n, size_t* bad_index) {
    std::unique_ptr<hbls_committee> c(new hbls_committee); c->n = n;       // freed (with its device tables) on every early return
    size_t nn = n ? n : 1;
    CK(cudaMalloc(&c->table, nn * sizeof(g1a)));
    Scratch* sc; if (int e = reserve(g.stream, nn * 49 + 4096, &sc)) return e;
    Arena ar{sc->base, 0, sc->cap};
    uint8_t* din = ar.take<uint8_t>(nn * 48); uint8_t* dok = ar.take<uint8_t>(nn);
    std::vector<uint8_t> ok(nn, 1);
    if (n) {
        CK(cudaMemcpyAsync(din, pk48, n * 48, cudaMemcpyHostToDevice, g.stream));
        LAUNCH(k_g1_decode, blocks_for(n, TPB), TPB, g.stream, n, din, c->table, dok, 1, 0);
        CK(cudaMalloc(&c->total, sizeof(g1)));
        LAUNCH(k_g1_sum, 1, 128, g.stream, n, c->table, c->total);
        CK(cudaMemcpyAsync(ok.data(), dok, n, cudaMemcpyDeviceToHost, g.stream));
        CK(cudaStreamSynchronize(g.stream));
    }
    for (size_t i = 0; i < n; i++) if (!ok[i]) { if (bad_index) *bad_index = i; return HBLS_ERR_DECODE; }
    *out = c.release(); return 0;
}
int hbls_committee_create(hbls_committee** out, const uint8_t* pk48, size_t n, size_t* bad_index) {
    if (int e = ensure_init()) return e;
    if (!out) return HBLS_ERR_ARG;
    std::lock_guard<std::mutex> lk(g.mu);
    return committee_create_locked(out, pk48, n, bad_index);
}
void hbls_committee_destroy(hbls_committee* c) { if (!c) return; std::lock_guard<std::mutex> lk(g.mu); cudaDeviceSynchronize(); delete c; }
size_t hbls_committee_size(const hbls_committee* c) { return c ? c->n : 0; }

static int mask_aggregate_locked(const hbls_committee* c, const uint8_t* bitmap, size_t blen, uint8_t out_pk48[48]) {
    Scratch* sc; if (int e = reserve(g.stream, blen + 4096, &sc)) return e;
    Arena ar{sc->base, 0, sc->cap};
    uint8_t* dbm = ar.take<uint8_t>(blen ? blen : 1); g1* dacc = ar.take<g1>(1); uint8_t* dout = ar.take<uint8_t>(48);
    if (blen) CK(cudaMemcpyAsync(dbm, bitmap, blen, cudaMemcpyHostToDevice, g.stream));
    LAUNCH(k_mask_aggregate, 1, 32, g.stream, (size_t)1, c->n, c->table, dbm, blen, dacc);
    LAUNCH(k_g1_serialize, 1, 32, g.stream, (size_t)1, dacc, dout);
    CK(cudaMemcpyAsync(out_pk48, dout, 48, cudaMemcpyDeviceToHost, g.stream));
    CK(cudaStreamSynchronize(g.stream));
    return 0;
}
int hbls_mask_aggregate(const hbls_committee* c, const uint8_t* bitmap, size_t blen, uint8_t out_pk48[48]) {
    if (int e = ensure_init()) return e;
    if (!c || blen != ((c->n + 7) >> 3)) return HBLS_ERR_ARG;
    std::lock_guard<std::mutex> lk(g.mu);
    return mask_aggregate_locked(c, bitmap, blen, out_pk48);
}

static int aggregate_sigs_locked(const uint8_t* sig96, size_t n, uint8_t out96[96]) {
    size_t nn = n ? n : 1;
    Scratch* sc; if (int e = reserve(g.stream, nn * (96 + sizeof(g2a) + 1) + 4096, &sc)) return e;
    Arena ar{sc->base, 0, sc->cap};
    uint8_t* din = ar.take<uint8_t>(nn * 96); g2a* dpts = ar.take<g2a>(nn); uint8_t* dok = ar.take<uint8_t>(nn);
    g2* dsum = ar.take<g2>(1); uint8_t* dout = ar.take<uint8_t>(96);
    std::vector<uint8_t> ok(nn, 1);
    if (n) {
        CK(cudaMemcpyAsync(din, sig96, n * 96, cudaMemcpyHostToDevice, g.stream));
        LAUNCH(k_g2_decode, heavy_blocks(n), TPB, g.stream, n, din, dpts, dok, 1);
    }
    LAUNCH(k_g2_sum, 1, HB_SUM_THREADS, g.stream, n, dpts, dsum);
    LAUNCH(k_g2_serialize, 1, 32, g.stream, (size_t)1, dsum, dout);
    if (n) CK(cudaMemcpyAsync(ok.data(), dok, n, cudaMemcpyDeviceToHost, g.stream));
    CK(cudaMemcpyAsync(out96, dout, 96, cudaMemcpyDeviceToHost, g.stream));
    CK(cudaStreamSynchronize(g.stream));
    for (size_t i = 0; i < n; i++) if (!ok[i]) return HBLS_ERR_DECODE;
    return 0;
}
int hbls_aggregate_sigs(const uint8_t* sig96, size_t n, uint8_t out96[96]) {
    if (int e = ensure_init()) return e;
    std::lock_guard<std::mutex> lk(g.mu);
    return aggregate_sigs_locked(sig96, n, out96);
}

// ------------------------------------------------------------------ aggregate verification
int hbls_aggregate_verify_batch_device(const hbls_committee* c, size_t B, const void* d_bitmaps, size_t blen, const void* d_sigs96,
                                       const void* d_msgs, size_t msg_len, void* d_results, void* stream) {
    if (int e = ensure_init()) return e;
    if (!c || blen != ((c->n + 7) >> 3)) return HBLS_ERR_ARG;
    if (B == 0) return 0;
    std::lock_guard<std::mutex> lk(g.mu);
    cudaStream_t s = stream ? (cudaStream_t)stream : g.stream;
    Scratch* sc; if (int e = reserve(s, verify_scratch_bytes(B), &sc)) return e;
    ensure_stage_events(sc);
    Arena ar{sc->base, 0, sc->cap};
    int rc = agg_verify_device_locked(c, B, (const uint8_t*)d_bitmaps, blen, (const uint8_t*)d_sigs96, (const uint8_t*)d_msgs, msg_len, (uint8_t*)d_results, s, sc, ar, false);
    CK(cudaGetLastError());
    return rc;
}
// ------------------------------------------------------------------ bodies of the batch verifiers, shared by their host and device
// forms: inputs in HBM, work enqueued on stream s in the scratch the caller reserved there, statuses computed on the device
// (device_forms.cuh).  The H(m) hints are those launch_verify_tail takes: same_msg / h_msg from a host form (it sees the messages),
// mg from a device form (messages grouped on the device).
// triples: keys decoded on the device, verdicts into d_results; d_status (nullable) receives the HBLS_VB_* codes
static void verify_triples_body(size_t k, const uint8_t* d_pk, const uint8_t* d_sig, const uint8_t* d_msgs, size_t msg_len, uint8_t* d_results,
                                uint8_t* d_status, cudaStream_t s, Scratch* sc, Arena& ar, bool same_msg, const MsgGroups* mg) {
    VerifyBufs v = carve_verify(ar, k);
    fork_point(k, sc, s);
    STAGE_EV(0, sc, s);
    // keys stay Jacobian (z = 1): the same tail as a mask aggregate, so independent triples also go through the batched groups
    LAUNCH(k_g1_decode_jac, heavy_blocks(k), TPB, s, k, d_pk, v.apk, v.ok_pk, 1);
    launch_verify_tail(k, v, sc, d_sig, d_msgs, (uint32_t)msg_len, v.ok_pk, d_results, s, same_msg, nullptr, mg);
    if (!d_status) return;
    uint8_t* dflags = ar.take<uint8_t>(k);
    LAUNCH(k_pack_flags, blocks_for(k, 256), 256, s, k, v.ok_sig, v.ok_hm, (const uint8_t*)v.ok_pk, dflags);
    LAUNCH(k_status_triples, blocks_for(k, 256), 256, s, k, (const uint8_t*)dflags, (const uint8_t*)d_results, d_status);
}
// header ranges against one committee: HBLS_HDR_* codes into d_status
static void verify_headers_body(const hbls_committee* c, size_t n, const uint8_t* d_sigs, const uint8_t* d_bitmaps, size_t blen,
                                const uint8_t* d_payloads, size_t payload_len, size_t quorum, uint8_t* d_status, cudaStream_t s, Scratch* sc,
                                Arena& ar, bool same_msg, const uint8_t* h_msg, const MsgGroups* mg) {
    uint8_t* dres = ar.take<uint8_t>(n); uint8_t* dflags = ar.take<uint8_t>(n);
    VerifyBufs v;
    agg_verify_device_locked(c, n, d_bitmaps, blen, d_sigs, d_payloads, payload_len, dres, s, sc, ar, same_msg, &v, h_msg, mg);
    LAUNCH(k_pack_flags, blocks_for(n, 256), 256, s, n, v.ok_sig, v.ok_hm, (const uint8_t*)nullptr, dflags);
    LAUNCH(k_status_headers, blocks_for(n, 256), 256, s, n, c->n, d_bitmaps, blen, quorum, (const uint8_t*)dflags, (const uint8_t*)dres, d_status);
}
// items of a multi-committee batch (their bitmaps back to back in d_bitmaps): verdicts into d_results.  The descriptors (table,
// bitmap, slots per item) come from the host array of handles.  They are written into the stream's own pinned buffer and uploaded
// with an asynchronous copy; an event recorded after that copy guards the buffer, so a later call on the same stream waits (on the
// host) only if the earlier upload has not run yet.  A pageable copy would synchronise the stream.
static int verify_items_body(size_t k, const hbls_committee* const* committees, const uint8_t* d_bitmaps, const uint8_t* d_sigs,
                             const uint8_t* d_msgs, size_t msg_len, uint8_t* d_results, cudaStream_t s, Scratch* sc, Arena& ar, bool same_msg,
                             const MsgGroups* mg) {
    if (sc->items_pending) { CK(cudaEventSynchronize(sc->items_copied)); sc->items_pending = false; }
    if (!sc->items_copied) CK(cudaEventCreateWithFlags(&sc->items_copied, cudaEventDisableTiming));
    if (k > sc->h_items_cap) {
        if (sc->h_items) CK(cudaFreeHost(sc->h_items));
        sc->h_items = nullptr; sc->h_items_cap = 0;
        CK(cudaMallocHost(&sc->h_items, k * sizeof(mask_item)));
        sc->h_items_cap = k;
    }
    VerifyBufs v = carve_verify(ar, k);
    mask_item* ditems = ar.take<mask_item>(k);
    size_t off = 0;
    for (size_t j = 0; j < k; j++) {
        sc->h_items[j].table = committees[j]->table; sc->h_items[j].bitmap = d_bitmaps + off; sc->h_items[j].n = committees[j]->n;
        off += (committees[j]->n + 7) >> 3;
    }
    CK(cudaMemcpyAsync(ditems, sc->h_items, k * sizeof(mask_item), cudaMemcpyHostToDevice, s));
    CK(cudaEventRecord(sc->items_copied, s)); sc->items_pending = true;
    fork_point(k, sc, s);
    STAGE_EV(0, sc, s);
    LAUNCH(k_mask_aggregate_items, blocks_for(k * 32, 128), 128, s, k, (const mask_item*)ditems, v.apk);
    launch_verify_tail(k, v, sc, d_sigs, d_msgs, (uint32_t)msg_len, nullptr, d_results, s, same_msg, nullptr, mg);
    return 0;
}

// ------------------------------------------------------------------ host forms: the inputs staged on g.stream, one synchronise
// rounds against one committee: verdicts into out (hbls_aggregate_verify_batch); with `status`, the HBLS_HDR_* codes under quorum
// (hbls_verify_headers).  One message for all rounds: it keys the H(m) cache.
static int agg_verify_host_locked(const hbls_committee* c, size_t B, const uint8_t* bitmaps, size_t blen, const uint8_t* sigs96,
                                  const uint8_t* msgs, size_t msg_len, uint8_t* out, bool status = false, size_t quorum = 0) {
    Scratch* sc; if (int e = reserve(g.stream, verify_scratch_bytes(B) + B * (blen + 96 + msg_len + 3) + 4096, &sc)) return e;
    ensure_stage_events(sc);
    Arena ar{sc->base, 0, sc->cap};
    uint8_t* dbm = ar.take<uint8_t>(B * blen + 1); uint8_t* dsig = ar.take<uint8_t>(B * 96); uint8_t* dmsg = ar.take<uint8_t>(B * msg_len + 1);
    uint8_t* dout = ar.take<uint8_t>(B);
    if (blen) CK(cudaMemcpyAsync(dbm, bitmaps, B * blen, cudaMemcpyHostToDevice, g.stream));
    CK(cudaMemcpyAsync(dsig, sigs96, B * 96, cudaMemcpyHostToDevice, g.stream));
    if (msg_len) CK(cudaMemcpyAsync(dmsg, msgs, B * msg_len, cudaMemcpyHostToDevice, g.stream));
    const bool same = all_messages_equal(msgs, B, msg_len);
    const uint8_t* h_msg = (same || B == 1) ? msgs : nullptr;
    if (status) verify_headers_body(c, B, dsig, dbm, blen, dmsg, msg_len, quorum, dout, g.stream, sc, ar, same, h_msg, nullptr);
    else agg_verify_device_locked(c, B, dbm, blen, dsig, dmsg, msg_len, dout, g.stream, sc, ar, same, nullptr, h_msg);
    CK(cudaMemcpyAsync(out, dout, B, cudaMemcpyDeviceToHost, g.stream));
    CK(cudaStreamSynchronize(g.stream));
    return 0;
}
int hbls_aggregate_verify_batch(const hbls_committee* c, size_t B, const uint8_t* bitmaps, size_t blen, const uint8_t* sigs96,
                                const uint8_t* msgs, size_t msg_len, uint8_t* results) {
    if (int e = ensure_init()) return e;
    if (!c || blen != ((c->n + 7) >> 3)) return HBLS_ERR_ARG;
    if (B == 0) return 0;
    std::lock_guard<std::mutex> lk(g.mu);
    return agg_verify_host_locked(c, B, bitmaps, blen, sigs96, msgs, msg_len, results);
}
// a single check: a request of the Part-1 combiner (concurrent callers share turns; a lone call is agg_verify_one_locked)
int hbls_aggregate_verify(const hbls_committee* c, const uint8_t* bitmap, size_t blen, const uint8_t sig96[96], const void* msg, size_t msg_len) {
    if (int e = ensure_init()) return e;
    if (!c || blen != ((c->n + 7) >> 3) || !sig96) return HBLS_ERR_ARG;
    Part1Req r; r.kind = RQ_AGG; r.com = c; r.bitmap = bitmap; r.blen = blen; r.a = sig96; r.msg = msg; r.len = msg_len;
    part1_submit(r);
    return r.err ? r.err : r.rc;
}
// engine.go:630-640: DecodeSigBitmap (signature deserialise) -> IsQuorumAchievedByMask -> VerifyHash
int hbls_verify_headers(const hbls_committee* c, size_t n, const uint8_t* sigs96, const uint8_t* bitmaps, size_t blen,
                        const uint8_t* payloads, size_t payload_len, size_t quorum, uint8_t* status) {
    if (int e = ensure_init()) return e;
    if (!c || blen != ((c->n + 7) >> 3) || !status) return HBLS_ERR_ARG;        // DecodeSigBitmap: mask.SetMask length error (sig.go:43)
    if (n == 0) return 0;
    std::lock_guard<std::mutex> lk(g.mu);
    return agg_verify_host_locked(c, n, bitmaps, blen, sigs96, payloads, payload_len, status, true, quorum);
}

static int aggregate_verify_items_locked(size_t k, const hbls_committee* const* committees, const uint8_t* bitmaps, const uint8_t* sigs96,
                                const uint8_t* msgs, size_t msg_len, uint8_t* results) {
    size_t bm_bytes = 0;
    for (size_t j = 0; j < k; j++) bm_bytes += (committees[j]->n + 7) >> 3;
    Scratch* sc; if (int e = reserve(g.stream, verify_scratch_bytes(k) + bm_bytes + k * (96 + msg_len + 1 + sizeof(mask_item)) + 4096, &sc)) return e;
    ensure_stage_events(sc);
    Arena ar{sc->base, 0, sc->cap};
    uint8_t* dbm = ar.take<uint8_t>(bm_bytes + 1); uint8_t* dsig = ar.take<uint8_t>(k * 96); uint8_t* dmsg = ar.take<uint8_t>(k * msg_len + 1);
    uint8_t* dres = ar.take<uint8_t>(k);
    if (bm_bytes) CK(cudaMemcpyAsync(dbm, bitmaps, bm_bytes, cudaMemcpyHostToDevice, g.stream));
    CK(cudaMemcpyAsync(dsig, sigs96, k * 96, cudaMemcpyHostToDevice, g.stream));
    if (msg_len) CK(cudaMemcpyAsync(dmsg, msgs, k * msg_len, cudaMemcpyHostToDevice, g.stream));
    if (int e = verify_items_body(k, committees, dbm, dsig, dmsg, msg_len, dres, g.stream, sc, ar, all_messages_equal(msgs, k, msg_len), nullptr)) return e;
    CK(cudaMemcpyAsync(results, dres, k, cudaMemcpyDeviceToHost, g.stream));
    CK(cudaStreamSynchronize(g.stream));
    return 0;
}
int hbls_aggregate_verify_items(size_t k, const hbls_committee* const* committees, const uint8_t* bitmaps, const uint8_t* sigs96,
                                const uint8_t* msgs, size_t msg_len, uint8_t* results) {
    if (int e = ensure_init()) return e;
    if (k == 0) return 0;
    if (!committees || !results) return HBLS_ERR_ARG;
    for (size_t j = 0; j < k; j++) if (!committees[j]) return HBLS_ERR_ARG;
    std::lock_guard<std::mutex> lk(g.mu);
    return aggregate_verify_items_locked(k, committees, bitmaps, sigs96, msgs, msg_len, results);
}

// hbls_verify_batch: verdicts into out; with `status`, hbls_verify_batch_status: the caller learns WHY an item failed, in the order
// the reference meets the errors (k_status_triples)
static int verify_batch_locked(size_t k, const uint8_t* pk48, const uint8_t* sig96, const uint8_t* msgs, size_t msg_len, uint8_t* out, bool status) {
    Scratch* sc; if (int e = reserve(g.stream, verify_scratch_bytes(k) + k * (48 + 96 + msg_len + 3) + 4096, &sc)) return e;
    ensure_stage_events(sc);
    Arena ar{sc->base, 0, sc->cap};
    uint8_t* dpk = ar.take<uint8_t>(k * 48); uint8_t* dsig = ar.take<uint8_t>(k * 96); uint8_t* dmsg = ar.take<uint8_t>(k * msg_len + 1);
    uint8_t* dres = ar.take<uint8_t>(k); uint8_t* dst = status ? ar.take<uint8_t>(k) : nullptr;
    CK(cudaMemcpyAsync(dpk, pk48, k * 48, cudaMemcpyHostToDevice, g.stream));
    CK(cudaMemcpyAsync(dsig, sig96, k * 96, cudaMemcpyHostToDevice, g.stream));
    if (msg_len) CK(cudaMemcpyAsync(dmsg, msgs, k * msg_len, cudaMemcpyHostToDevice, g.stream));
    verify_triples_body(k, dpk, dsig, dmsg, msg_len, dres, dst, g.stream, sc, ar, all_messages_equal(msgs, k, msg_len), nullptr);
    CK(cudaMemcpyAsync(out, status ? dst : dres, k, cudaMemcpyDeviceToHost, g.stream));
    CK(cudaStreamSynchronize(g.stream));
    return 0;
}
int hbls_verify_batch(size_t k, const uint8_t* pk48, const uint8_t* sig96, const uint8_t* msgs, size_t msg_len, uint8_t* results) {
    if (int e = ensure_init()) return e;
    if (k == 0) return 0;
    std::lock_guard<std::mutex> lk(g.mu);
    return verify_batch_locked(k, pk48, sig96, msgs, msg_len, results, false);
}
int hbls_verify_batch_status(size_t k, const uint8_t* pk48, const uint8_t* sig96, const uint8_t* msgs, size_t msg_len, uint8_t* status) {
    if (int e = ensure_init()) return e;
    if (k == 0) return 0;
    if (!status) return HBLS_ERR_ARG;
    std::lock_guard<std::mutex> lk(g.mu);
    return verify_batch_locked(k, pk48, sig96, msgs, msg_len, status, true);
}

// ------------------------------------------------------------------ device forms: inputs and outputs in HBM (any byte alignment),
// everything enqueued on the caller's stream with no host synchronisation, H(m) once per distinct message (grouped on the device;
// the H(m) cache is neither read nor filled: the host never sees the messages)
static int verify_batch_status_device_locked(size_t k, const uint8_t* d_pk, const uint8_t* d_sig, const uint8_t* d_msgs, size_t msg_len,
                                             uint8_t* d_status, cudaStream_t s) {
    Scratch* sc; if (int e = reserve(s, verify_scratch_bytes(k) + group_bytes(k) + 2 * k + 4096, &sc)) return e;
    ensure_stage_events(sc);
    Arena ar{sc->base, 0, sc->cap};
    const MsgGroups mg = carve_groups(ar, k); uint8_t* dres = ar.take<uint8_t>(k);
    verify_triples_body(k, d_pk, d_sig, d_msgs, msg_len, dres, d_status, s, sc, ar, false, &mg);
    CK(cudaGetLastError());
    return 0;
}
int hbls_verify_batch_status_device(size_t k, const void* d_pk48, const void* d_sig96, const void* d_msgs, size_t msg_len, void* d_status, void* stream) {
    if (int e = ensure_init()) return e;
    if (k == 0) return 0;
    if (!d_status) return HBLS_ERR_ARG;
    std::lock_guard<std::mutex> lk(g.mu);
    return verify_batch_status_device_locked(k, (const uint8_t*)d_pk48, (const uint8_t*)d_sig96, (const uint8_t*)d_msgs, msg_len, (uint8_t*)d_status,
                                             stream ? (cudaStream_t)stream : g.stream);
}
static int verify_headers_device_locked(const hbls_committee* c, size_t n, const uint8_t* d_sigs, const uint8_t* d_bitmaps, size_t blen,
                                        const uint8_t* d_payloads, size_t payload_len, size_t quorum, uint8_t* d_status, cudaStream_t s) {
    Scratch* sc; if (int e = reserve(s, verify_scratch_bytes(n) + group_bytes(n) + 2 * n + 4096, &sc)) return e;
    ensure_stage_events(sc);
    Arena ar{sc->base, 0, sc->cap};
    const MsgGroups mg = carve_groups(ar, n);
    verify_headers_body(c, n, d_sigs, d_bitmaps, blen, d_payloads, payload_len, quorum, d_status, s, sc, ar, false, nullptr, &mg);
    CK(cudaGetLastError());
    return 0;
}
int hbls_verify_headers_device(const hbls_committee* c, size_t n, const void* d_sigs96, const void* d_bitmaps, size_t blen,
                               const void* d_payloads, size_t payload_len, size_t quorum, void* d_status, void* stream) {
    if (int e = ensure_init()) return e;
    if (!c || blen != ((c->n + 7) >> 3) || !d_status) return HBLS_ERR_ARG;
    if (n == 0) return 0;
    std::lock_guard<std::mutex> lk(g.mu);
    return verify_headers_device_locked(c, n, (const uint8_t*)d_sigs96, (const uint8_t*)d_bitmaps, blen, (const uint8_t*)d_payloads, payload_len, quorum,
                                        (uint8_t*)d_status, stream ? (cudaStream_t)stream : g.stream);
}
static int aggregate_verify_items_device_locked(size_t k, const hbls_committee* const* committees, const uint8_t* d_bitmaps, const uint8_t* d_sigs,
                                                const uint8_t* d_msgs, size_t msg_len, uint8_t* d_results, cudaStream_t s) {
    Scratch* sc; if (int e = reserve(s, verify_scratch_bytes(k) + group_bytes(k) + k * sizeof(mask_item) + 4096, &sc)) return e;
    ensure_stage_events(sc);
    Arena ar{sc->base, 0, sc->cap};
    const MsgGroups mg = carve_groups(ar, k);
    if (int e = verify_items_body(k, committees, d_bitmaps, d_sigs, d_msgs, msg_len, d_results, s, sc, ar, false, &mg)) return e;
    CK(cudaGetLastError());
    return 0;
}
int hbls_aggregate_verify_items_device(size_t k, const hbls_committee* const* committees, const void* d_bitmaps, const void* d_sigs96,
                                       const void* d_msgs, size_t msg_len, void* d_results, void* stream) {
    if (int e = ensure_init()) return e;
    if (k == 0) return 0;
    if (!committees || !d_results) return HBLS_ERR_ARG;
    for (size_t j = 0; j < k; j++) if (!committees[j]) return HBLS_ERR_ARG;
    std::lock_guard<std::mutex> lk(g.mu);
    return aggregate_verify_items_device_locked(k, committees, (const uint8_t*)d_bitmaps, (const uint8_t*)d_sigs96, (const uint8_t*)d_msgs, msg_len,
                                                (uint8_t*)d_results, stream ? (cudaStream_t)stream : g.stream);
}

// ------------------------------------------------------------------ persistent Mask / running vote aggregate (SURVEY 8f.2)
int hbls_mask_create(hbls_mask** out, const hbls_committee* c) {
    if (int e = ensure_init()) return e;
    if (!out || !c) return HBLS_ERR_ARG;
    std::lock_guard<std::mutex> lk(g.mu);
    std::unique_ptr<hbls_mask> m(new hbls_mask); m->c = c; m->bitmap.assign((c->n + 7) >> 3, 0);
    CK(cudaMalloc(&m->d_acc, sizeof(g1)));
    CK(cudaMemsetAsync(m->d_acc, 0, sizeof(g1), g.stream));          // all-zero struct = identity (mask.go:88)
    CK(cudaStreamSynchronize(g.stream));
    *out = m.release(); return 0;
}
void hbls_mask_destroy(hbls_mask* m) { if (!m) return; std::lock_guard<std::mutex> lk(g.mu); cudaDeviceSynchronize(); delete m; }
int hbls_mask_clear(hbls_mask* m) {
    if (int e = ensure_init()) return e;
    if (!m) return HBLS_ERR_ARG;
    std::lock_guard<std::mutex> lk(g.mu);
    std::fill(m->bitmap.begin(), m->bitmap.end(), 0);
    CK(cudaMemsetAsync(m->d_acc, 0, sizeof(g1), g.stream));
    CK(cudaStreamSynchronize(g.stream));
    return 0;
}
int hbls_mask_set_mask(hbls_mask* m, const uint8_t* bitmap, size_t blen) {
    if (int e = ensure_init()) return e;
    if (!m || blen != m->bitmap.size()) return HBLS_ERR_ARG;          // mask.go:114-120 "mismatching bitmap lengths"
    std::lock_guard<std::mutex> lk(g.mu);
    return set_mask_locked(m, bitmap);
}
// the read-modify-write of the bitmap stays under g.mu: concurrent callers that set different bits keep each other's bits
int hbls_mask_set_bit(hbls_mask* m, size_t index, int enable) {
    if (int e = ensure_init()) return e;
    if (!m || index >= m->c->n) return HBLS_ERR_ARG;                   // mask.go:138-140 "index out of range"
    std::lock_guard<std::mutex> lk(g.mu);
    std::vector<uint8_t> bm = m->bitmap;
    const uint8_t msk = (uint8_t)(1u << (index & 7));
    if (enable) bm[index >> 3] |= msk; else bm[index >> 3] &= (uint8_t)~msk;
    return set_mask_locked(m, bm.data());
}
int hbls_mask_count_enabled(const hbls_mask* m) {
    if (!m) return HBLS_ERR_ARG;
    std::lock_guard<std::mutex> lk(g.mu);
    return popcount_slots(m->bitmap.data(), m->c->n);
}
int hbls_mask_get(const hbls_mask* m, uint8_t* bitmap_out, size_t blen, uint8_t pk48_out[48]) {
    if (int e = ensure_init()) return e;
    if (!m || (bitmap_out && blen != m->bitmap.size())) return HBLS_ERR_ARG;
    std::lock_guard<std::mutex> lk(g.mu);
    if (bitmap_out) memcpy(bitmap_out, m->bitmap.data(), blen);
    if (pk48_out) {
        Scratch* sc; if (int e = reserve(g.stream, 4096, &sc)) return e;
        Arena ar{sc->base, 0, sc->cap};
        uint8_t* dout = ar.take<uint8_t>(48);
        LAUNCH(k_g1_serialize, 1, 32, g.stream, (size_t)1, (const g1*)m->d_acc, dout);
        CK(cudaMemcpyAsync(pk48_out, dout, 48, cudaMemcpyDeviceToHost, g.stream));
        CK(cudaStreamSynchronize(g.stream));
    }
    return 0;
}
int hbls_mask_verify(const hbls_mask* m, const uint8_t sig96[96], const void* msg, size_t msg_len) {
    if (int e = ensure_init()) return e;
    if (!m || !sig96) return HBLS_ERR_ARG;
    Part1Req r; r.kind = RQ_MASK; r.mask = m; r.a = sig96; r.msg = msg; r.len = msg_len;
    part1_submit(r);
    return r.err ? r.err : r.rc;
}
int hbls_ballot_box_create(hbls_ballot_box** out, const hbls_committee* c) {
    if (int e = ensure_init()) return e;
    if (!out || !c) return HBLS_ERR_ARG;
    std::lock_guard<std::mutex> lk(g.mu);
    std::unique_ptr<hbls_ballot_box> b(new hbls_ballot_box); b->c = c; b->collected.assign((c->n + 7) >> 3, 0);
    CK(cudaMalloc(&b->d_sum, sizeof(g2)));
    CK(cudaMemsetAsync(b->d_sum, 0, sizeof(g2), g.stream));
    CK(cudaStreamSynchronize(g.stream));
    *out = b.release(); return 0;
}
void hbls_ballot_box_destroy(hbls_ballot_box* b) { if (!b) return; std::lock_guard<std::mutex> lk(g.mu); cudaDeviceSynchronize(); delete b; }
static int ballot_box_add_vote_locked(hbls_ballot_box* b, const uint8_t* signer_bitmap, size_t blen, const uint8_t sig96[96]) {
    const size_t n = b->c->n;
    for (size_t i = 0; i < n; i++)                                      // quorum.go:168-181: skip a ballot that shares a signer with a collected one
        if ((signer_bitmap[i >> 3] >> (i & 7)) & 1 && (b->collected[i >> 3] >> (i & 7)) & 1) return 1;
    Scratch* sc; if (int e = reserve(g.stream, 4096, &sc)) return e;
    Arena ar{sc->base, 0, sc->cap};
    uint8_t* dsig = ar.take<uint8_t>(96); int* drc = ar.take<int>(1);
    CK(cudaMemcpyAsync(dsig, sig96, 96, cudaMemcpyHostToDevice, g.stream));
    LAUNCH(k_single, 1, 32, g.stream, (size_t)1, (const single_desc*)nullptr, single_desc{dsig, nullptr, b->d_sum, OP_G2_DES_ADD, 0u}, drc);
    int rc = 0;
    CK(cudaMemcpyAsync(&rc, drc, sizeof(int), cudaMemcpyDeviceToHost, g.stream));
    CK(cudaStreamSynchronize(g.stream));
    if (rc != 96) return HBLS_ERR_DECODE;
    for (size_t i = 0; i < n; i++) if ((signer_bitmap[i >> 3] >> (i & 7)) & 1) b->collected[i >> 3] |= (uint8_t)(1u << (i & 7));
    return 0;
}
int hbls_ballot_box_add_vote(hbls_ballot_box* b, const uint8_t* signer_bitmap, size_t blen, const uint8_t sig96[96]) {
    if (int e = ensure_init()) return e;
    if (!b || !signer_bitmap || blen != b->collected.size()) return HBLS_ERR_ARG;
    std::lock_guard<std::mutex> lk(g.mu);
    return ballot_box_add_vote_locked(b, signer_bitmap, blen, sig96);
}
static_assert(HB_BALLOT_ACCEPTED == HBLS_BALLOT_ACCEPTED && HB_BALLOT_COLLECTED == HBLS_BALLOT_COLLECTED &&
              HB_BALLOT_BAD_SIG_ENCODING == HBLS_BALLOT_BAD_SIG_ENCODING && HB_BALLOT_BAD_SIG == HBLS_BALLOT_BAD_SIG, "ballot status codes");
// a leader's vote queue: same-message aggregate verification over the committee table (mask aggregation, signature decode, H(m)
// once), then the ballot rules in arrival order and the fold of the accepted signatures, all on the device.  One H2D copy of the box's
// bitmap and the queue, one D2H copy of the statuses and the new bitmap, one synchronise.
static int ballot_box_submit_votes_locked(hbls_ballot_box* b, size_t k, const uint8_t* signer_bitmaps, size_t blen, const uint8_t* sigs96,
                                          const void* msg, size_t msg_len, uint8_t* status) {
    auto up = [](size_t x) { return (x + 255) & ~(size_t)255; };            // the arena's alignment: offsets of the staged copy
    const size_t o_sig = up(k * blen), o_col = o_sig + up(k * 96), o_msg = o_col + up(blen), in_bytes = o_msg + msg_len + 1;
    Scratch* sc; if (int e = reserve(g.stream, verify_scratch_bytes(k) + in_bytes + up(k + blen) + up(k) + 4096, &sc)) return e;
    ensure_stage_events(sc);
    Arena ar{sc->base, 0, sc->cap};
    uint8_t* din = ar.take<uint8_t>(in_bytes); uint8_t* dres = ar.take<uint8_t>(k); uint8_t* dacc = ar.take<uint8_t>(k);
    uint8_t* dout = ar.take<uint8_t>(k + blen);                             // statuses, then the new collected bitmap
    std::vector<uint8_t> h(in_bytes, 0);
    memcpy(h.data(), signer_bitmaps, k * blen); memcpy(h.data() + o_sig, sigs96, k * 96);
    memcpy(h.data() + o_col, b->collected.data(), blen); if (msg_len) memcpy(h.data() + o_msg, msg, msg_len);
    CK(cudaMemcpyAsync(din, h.data(), in_bytes, cudaMemcpyHostToDevice, g.stream));
    VerifyBufs v;
    agg_verify_device_locked(b->c, k, din, blen, din + o_sig, din + o_msg, msg_len, dres, g.stream, sc, ar, true, &v, (const uint8_t*)msg);
    LAUNCH(k_ballot_admit, 1, HB_BALLOT_THREADS, g.stream, k, b->c->n, blen, (const uint8_t*)din, (const uint8_t*)dres, (const uint8_t*)v.ok_sig,
           (const uint8_t*)(din + o_col), dout + k, dout, dacc);
    LAUNCH(k_ballot_fold, 1, HB_SUM_THREADS, g.stream, k, (const g2a*)v.sig, (const uint8_t*)dacc, b->d_sum);
    std::vector<uint8_t> back(k + blen);
    CK(cudaMemcpyAsync(back.data(), dout, k + blen, cudaMemcpyDeviceToHost, g.stream));
    CK(cudaStreamSynchronize(g.stream));
    memcpy(status, back.data(), k);
    memcpy(b->collected.data(), back.data() + k, blen);
    return 0;
}
int hbls_ballot_box_submit_votes(hbls_ballot_box* b, size_t k, const uint8_t* signer_bitmaps, size_t blen, const uint8_t* sigs96,
                                 const void* msg, size_t msg_len, uint8_t* status) {
    if (int e = ensure_init()) return e;
    if (!b || !status || blen != b->collected.size() || msg_len > 64 || blen > HB_BALLOT_MAX_BYTES) return HBLS_ERR_ARG;
    if (k == 0) return 0;
    if (!signer_bitmaps || !sigs96 || (msg_len && !msg)) return HBLS_ERR_ARG;
    std::lock_guard<std::mutex> lk(g.mu);
    return ballot_box_submit_votes_locked(b, k, signer_bitmaps, blen, sigs96, msg, msg_len, status);
}
static int ballot_box_aggregate_locked(const hbls_ballot_box* b, uint8_t out_sig96[96], uint8_t* bitmap_out, size_t blen) {
    Scratch* sc; if (int e = reserve(g.stream, 4096, &sc)) return e;
    Arena ar{sc->base, 0, sc->cap};
    uint8_t* dout = ar.take<uint8_t>(96);
    LAUNCH(k_g2_serialize, 1, 32, g.stream, (size_t)1, (const g2*)b->d_sum, dout);
    CK(cudaMemcpyAsync(out_sig96, dout, 96, cudaMemcpyDeviceToHost, g.stream));
    CK(cudaStreamSynchronize(g.stream));
    if (bitmap_out) memcpy(bitmap_out, b->collected.data(), blen);
    return 0;
}
int hbls_ballot_box_aggregate(const hbls_ballot_box* b, uint8_t out_sig96[96], uint8_t* bitmap_out, size_t blen) {
    if (int e = ensure_init()) return e;
    if (!b || !out_sig96 || (bitmap_out && blen != b->collected.size())) return HBLS_ERR_ARG;
    std::lock_guard<std::mutex> lk(g.mu);
    return ballot_box_aggregate_locked(b, out_sig96, bitmap_out, blen);
}

// ------------------------------------------------------------------ ONE batch split over several GPUs (SURVEY 8e, BASELINE configs[3])
struct PartialRecord { g2 S; fp2 f[6]; uint32_t n_items; uint32_t n_bad; };
// the wire record is the first HBLS_PARTIAL_BYTES of the struct
static_assert(offsetof(PartialRecord, n_bad) + sizeof(uint32_t) == HBLS_PARTIAL_BYTES && sizeof(PartialRecord) >= HBLS_PARTIAL_BYTES, "partial record layout");
static int rlc_partial_locked(size_t k, const uint8_t* pk48, const uint8_t* sig96, const uint8_t* msgs, size_t msg_len, uint8_t record[HBLS_PARTIAL_BYTES]) {
    PartialRecord rec; memset(&rec, 0, sizeof rec);
    const size_t kk = k ? k : 1;
    const unsigned W = (unsigned)(kk < (size_t)g.sm_count * 2 ? kk : (size_t)g.sm_count * 2);      // warps that multiply Miller values into partial products
    Scratch* sc; if (int e = reserve(g.stream, verify_scratch_bytes(kk) + kk * (48 + 96 + msg_len + 8) + (W + 2) * 6 * sizeof(fp2) + sizeof(g2) + 8192, &sc)) return e;
    Arena ar{sc->base, 0, sc->cap};
    VerifyBufs v = carve_verify(ar, kk);
    uint8_t* dpk = ar.take<uint8_t>(kk * 48); uint8_t* dsig = ar.take<uint8_t>(kk * 96); uint8_t* dmsg = ar.take<uint8_t>(kk * msg_len + 1);
    uint64_t* dco = ar.take<uint64_t>(kk); fp2* dpart = ar.take<fp2>((size_t)W * 6); fp2* dprod = ar.take<fp2>(6); g2* dS = ar.take<g2>(1);
    if (k) {
        const std::vector<uint64_t> co = rlc_draw_items(k);
        CK(cudaMemcpyAsync(dpk, pk48, k * 48, cudaMemcpyHostToDevice, g.stream));
        CK(cudaMemcpyAsync(dsig, sig96, k * 96, cudaMemcpyHostToDevice, g.stream));
        if (msg_len) CK(cudaMemcpyAsync(dmsg, msgs, k * msg_len, cudaMemcpyHostToDevice, g.stream));
        CK(cudaMemcpyAsync(dco, co.data(), k * 8, cudaMemcpyHostToDevice, g.stream));
        CK(cudaStreamSynchronize(g.stream));                    // co is a local: the copy must have read it before it goes out of scope
    }
    CK(cudaMemsetAsync(v.counts, 0, 2 * sizeof(unsigned), g.stream));
    LAUNCH(k_g1_decode_jac, heavy_blocks(kk), TPB, g.stream, k, dpk, v.apk, v.ok_pk, 1);
    const bool pairs = (long long)k <= g.coop_max;
    if (pairs) { LAUNCH(k_g2_decode_pair, blocks_for(2 * kk, 32), 32, g.stream, k, dsig, v.sig, v.ok_sig, 1); launch_hash_small(g.stream, k, dmsg, (uint32_t)msg_len, v.hm, v.ok_hm); }
    else { LAUNCH(k_g2_decode, heavy_blocks(kk), TPB, g.stream, k, dsig, v.sig, v.ok_sig, 1); LAUNCH(k_hash_to_g2, heavy_blocks(kk), TPB, g.stream, k, dmsg, (uint32_t)msg_len, v.hm, v.ok_hm); }
    rlc_coeffs none{};
    LAUNCH(k_rlc_scale, heavy_blocks(kk), TPB, g.stream, k, (size_t)1, v.apk, v.sig, v.hm, v.ok_sig, v.ok_hm, (const uint8_t*)v.ok_pk, none, (const uint64_t*)dco, v.pk_scaled, v.S, v.bad);
    LAUNCH(k_rlc_partial_coop, W, 32, g.stream, k, v.pk_scaled, v.hm, v.bad, dpart, v.counts);
    LAUNCH(k_rlc_reduce_coop, 1, 32, g.stream, (size_t)W, dpart, dprod);
    LAUNCH(k_g2_sum_jac, 1, HB_SUM_THREADS, g.stream, k, v.S, dS);
    unsigned counts[2] = {0, 0};
    CK(cudaMemcpyAsync(&rec.S, dS, sizeof(g2), cudaMemcpyDeviceToHost, g.stream));
    CK(cudaMemcpyAsync(rec.f, dprod, 6 * sizeof(fp2), cudaMemcpyDeviceToHost, g.stream));
    CK(cudaMemcpyAsync(counts, v.counts, sizeof counts, cudaMemcpyDeviceToHost, g.stream));
    CK(cudaStreamSynchronize(g.stream));
    rec.n_items = (uint32_t)k; rec.n_bad = counts[0];
    memcpy(record, &rec, HBLS_PARTIAL_BYTES);
    return 0;
}
int hbls_rlc_partial(size_t k, const uint8_t* pk48, const uint8_t* sig96, const uint8_t* msgs, size_t msg_len, uint8_t record[HBLS_PARTIAL_BYTES]) {
    if (int e = ensure_init()) return e;
    if (!record) return HBLS_ERR_ARG;
    std::lock_guard<std::mutex> lk(g.mu);
    return rlc_partial_locked(k, pk48, sig96, msgs, msg_len, record);
}
// the device part of hbls_rlc_fold (records that hold items and no undecodable one)
static int rlc_fold_locked(size_t n, const uint8_t* records) {
    Scratch* sc; if (int e = reserve(g.stream, n * (sizeof(g2) + 6 * sizeof(fp2)) + sizeof(g2) + sizeof(g2a) + 4096, &sc)) return e;
    Arena ar{sc->base, 0, sc->cap};
    g2* dS = ar.take<g2>(n); fp2* dparts = ar.take<fp2>(n * 6); g2* dsum = ar.take<g2>(1); g2a* dsg = ar.take<g2a>(1); uint8_t* dres = ar.take<uint8_t>(1);
    std::vector<g2> hs(n); std::vector<fp2> hf(n * 6);
    for (size_t p = 0; p < n; p++) { PartialRecord r; memcpy(&r, records + p * HBLS_PARTIAL_BYTES, HBLS_PARTIAL_BYTES); hs[p] = r.S; for (int i = 0; i < 6; i++) hf[6 * p + i] = r.f[i]; }
    CK(cudaMemcpyAsync(dS, hs.data(), n * sizeof(g2), cudaMemcpyHostToDevice, g.stream));
    CK(cudaMemcpyAsync(dparts, hf.data(), n * 6 * sizeof(fp2), cudaMemcpyHostToDevice, g.stream));
    LAUNCH(k_g2_sum_jac, 1, HB_SUM_THREADS, g.stream, n, dS, dsum);
    LAUNCH(k_g2_normalize, 1, 32, g.stream, (size_t)1, dsum, dsg);
    LAUNCH(k_rlc_fold_coop, 1, 32, g.stream, n, dparts, dsg, dres);
    uint8_t res = 0;
    CK(cudaMemcpyAsync(&res, dres, 1, cudaMemcpyDeviceToHost, g.stream));
    CK(cudaStreamSynchronize(g.stream));                              // hs / hf stay alive until the copies are done
    return res ? 1 : 0;
}
int hbls_rlc_fold(size_t n, const uint8_t* records) {
    if (int e = ensure_init()) return e;
    if (!records) return HBLS_ERR_ARG;
    size_t items = 0, bad = 0;
    for (size_t p = 0; p < n; p++) { PartialRecord r; memcpy(&r, records + p * HBLS_PARTIAL_BYTES, HBLS_PARTIAL_BYTES); items += r.n_items; bad += r.n_bad; }
    if (bad || items == 0) return 0;                                  // an undecodable / identity item somewhere, or nothing to prove: callers verify exactly
    std::lock_guard<std::mutex> lk(g.mu);
    return rlc_fold_locked(n, records);
}

static int sign_hash_batch_locked(size_t k, const uint8_t* sk32, const uint8_t* msgs, size_t msg_len, uint8_t* sig96_out, uint8_t* ok) {
    Scratch* sc; if (int e = reserve(g.stream, k * (32 + msg_len + sizeof(g2) + 96 + 1) + 4096, &sc)) return e;
    Arena ar{sc->base, 0, sc->cap};
    uint8_t* dsk = ar.take<uint8_t>(k * 32); uint8_t* dmsg = ar.take<uint8_t>(k * msg_len + 1); g2* dpts = ar.take<g2>(k);
    uint8_t* dout = ar.take<uint8_t>(k * 96); uint8_t* dok = ar.take<uint8_t>(k);
    CK(cudaMemcpyAsync(dsk, sk32, k * 32, cudaMemcpyHostToDevice, g.stream));
    if (msg_len) CK(cudaMemcpyAsync(dmsg, msgs, k * msg_len, cudaMemcpyHostToDevice, g.stream));
    LAUNCH(k_sign_hash, blocks_for(k, TPB), TPB, g.stream, k, dsk, dmsg, (uint32_t)msg_len, dpts, dok);
    LAUNCH(k_g2_serialize, blocks_for(k, TPB), TPB, g.stream, k, dpts, dout);
    CK(cudaMemcpyAsync(sig96_out, dout, k * 96, cudaMemcpyDeviceToHost, g.stream));
    CK(cudaMemcpyAsync(ok, dok, k, cudaMemcpyDeviceToHost, g.stream));
    CK(cudaStreamSynchronize(g.stream));
    return 0;
}
int hbls_sign_hash_batch(size_t k, const uint8_t* sk32, const uint8_t* msgs, size_t msg_len, uint8_t* sig96_out, uint8_t* ok) {
    if (int e = ensure_init()) return e;
    if (k == 0) return 0;
    std::lock_guard<std::mutex> lk(g.mu);
    return sign_hash_batch_locked(k, sk32, msgs, msg_len, sig96_out, ok);
}
static int get_public_key_batch_locked(size_t k, const uint8_t* sk32, uint8_t* pk48_out) {
    Scratch* sc; if (int e = reserve(g.stream, k * (32 + sizeof(g1) + 48) + 4096, &sc)) return e;
    Arena ar{sc->base, 0, sc->cap};
    uint8_t* dsk = ar.take<uint8_t>(k * 32); g1* dpts = ar.take<g1>(k); uint8_t* dout = ar.take<uint8_t>(k * 48);
    CK(cudaMemcpyAsync(dsk, sk32, k * 32, cudaMemcpyHostToDevice, g.stream));
    LAUNCH(k_g1_mul_gen, blocks_for(k, TPB), TPB, g.stream, k, dsk, dpts);
    LAUNCH(k_g1_serialize, blocks_for(k, TPB), TPB, g.stream, k, dpts, dout);
    CK(cudaMemcpyAsync(pk48_out, dout, k * 48, cudaMemcpyDeviceToHost, g.stream));
    CK(cudaStreamSynchronize(g.stream));
    return 0;
}
int hbls_get_public_key_batch(size_t k, const uint8_t* sk32, uint8_t* pk48_out) {
    if (int e = ensure_init()) return e;
    if (k == 0) return 0;
    std::lock_guard<std::mutex> lk(g.mu);
    return get_public_key_batch_locked(k, sk32, pk48_out);
}

static int fp_mul_batch_locked(size_t n, const uint8_t* a48, const uint8_t* b48, uint8_t* out48) {
    Scratch* sc; if (int e = reserve(g.stream, n * 144 + 4096, &sc)) return e;
    Arena ar{sc->base, 0, sc->cap};
    uint8_t* da = ar.take<uint8_t>(n * 48); uint8_t* db = ar.take<uint8_t>(n * 48); uint8_t* dout = ar.take<uint8_t>(n * 48);
    CK(cudaMemcpyAsync(da, a48, n * 48, cudaMemcpyHostToDevice, g.stream));
    CK(cudaMemcpyAsync(db, b48, n * 48, cudaMemcpyHostToDevice, g.stream));
    LAUNCH(k_fp_mul, blocks_for(n, 128), 128, g.stream, n, da, db, dout);
    CK(cudaMemcpyAsync(out48, dout, n * 48, cudaMemcpyDeviceToHost, g.stream));
    CK(cudaStreamSynchronize(g.stream));
    return 0;
}
int hbls_fp_mul_batch(size_t n, const uint8_t* a48, const uint8_t* b48, uint8_t* out48) {
    if (int e = ensure_init()) return e;
    if (n == 0) return 0;
    std::lock_guard<std::mutex> lk(g.mu);
    return fp_mul_batch_locked(n, a48, b48, out48);
}

void hbls_stage_timing_enable(int on) {
    std::lock_guard<std::mutex> lk(g.mu);
    g.stage_timing = on != 0; g.stage_sc = nullptr;
}
int hbls_stage_timing_get(float* ms_out, int max_stages) {
    std::lock_guard<std::mutex> lk(g.mu);
    Scratch* sc = g.stage_sc;
    if (!sc || !sc->ev_ok) return 0;
    if (cudaEventSynchronize(sc->ev[6]) != cudaSuccess) return 0;
    int n = max_stages < 6 ? max_stages : 6;
    for (int i = 0; i < n; i++) { float ms = 0; cudaEventElapsedTime(&ms, sc->ev[i], sc->ev[i + 1]); ms_out[i] = ms; }
    // 7th value: the line kernel's part of stage 5 when the batched pairing ran as two kernels (first chunk), else 0
    if (max_stages >= 7) { float ms = 0; if (sc->ev7_set) cudaEventElapsedTime(&ms, sc->ev[5], sc->ev[7]); ms_out[6] = ms; n = 7; }
    return n;
}
static int selftest_split_locked(uint32_t iters) {
    Scratch* sc; if (int e = reserve(g.stream, 4096, &sc)) return e;
    uint32_t* d = reinterpret_cast<uint32_t*>(sc->base);
    CK(cudaMemsetAsync(d, 0, 4, g.stream));
    LAUNCH(k_selftest_fp2h, 8, 64, g.stream, iters, 20240922u, d);
    uint32_t bad = 0;
    CK(cudaMemcpyAsync(&bad, d, 4, cudaMemcpyDeviceToHost, g.stream));
    CK(cudaStreamSynchronize(g.stream));
    return (int)bad;
}
int hbls_selftest_split(uint32_t iters) {
    if (int e = ensure_init()) return e;
    std::lock_guard<std::mutex> lk(g.mu);
    return selftest_split_locked(iters);
}
double hbls_probe_mac32_per_s(int iters, double* sm_clock_hz) {
    if (ensure_init()) return -1.0;
    std::lock_guard<std::mutex> lk(g.mu);
    Scratch* sc; if (reserve(g.stream, 4096, &sc)) return -1.0;
    uint32_t* sink = reinterpret_cast<uint32_t*>(sc->base);
    unsigned long long* cyc = reinterpret_cast<unsigned long long*>(sc->base + 256);
    constexpr int K = 4;
    const int threads = 256, blocks = g.sm_count * 2;                  // one wave: 2 x 256 threads x 94 registers per SM
    cudaEvent_t e0, e1; cudaEventCreate(&e0); cudaEventCreate(&e1);
    LAUNCH(k_probe_carry<K>, blocks, threads, g.stream, iters / 8 + 1, 12345u, sink, cyc);     // warm-up
    cudaEventRecord(e0, g.stream);
    LAUNCH(k_probe_carry<K>, blocks, threads, g.stream, iters, 12345u, sink, cyc);
    cudaEventRecord(e1, g.stream);
    if (cudaStreamSynchronize(g.stream) != cudaSuccess) return -1.0;
    float ms = 0; cudaEventElapsedTime(&ms, e0, e1);
    cudaEventDestroy(e0); cudaEventDestroy(e1);
    if (sm_clock_hz) { int khz = 0; cudaDeviceGetAttribute(&khz, cudaDevAttrClockRate, g.device); *sm_clock_hz = khz * 1e3; }   // maximum SM clock
    double macs = (double)blocks * threads * (double)iters * K * 6.0;  // lane_mad = 6 IMAD.WIDE
    return macs / (ms * 1e-3);
}

}  // extern "C"

namespace {
// a turn of one AGG request: exactly what hbls_aggregate_verify_batch does for one round (latency kernels on three streams, the H(m)
// cache keyed by the message, the hbls_last_batch_info record)
int agg_verify_one_locked(Part1Req& r) {
    uint8_t res = 0;
    if (int e = agg_verify_host_locked(r.com, 1, r.bitmap, r.blen, static_cast<const uint8_t*>(r.a), static_cast<const uint8_t*>(r.msg), r.len, &res)) return e;
    r.rc = res ? 1 : 0;
    return 0;
}
}  // namespace

#include "selftest.cuh"
