// tests/emu/emu_kernels.cpp -- TEST HARNESS ONLY: runs the __global__ kernels of harmony_b200/csrc/kernels.cuh on the host
// (HB_HOST_EMU: software carry flags; thread-per-item kernels one "thread" after the other, the lane-pair kernels as a
// 2-thread CTA on two host threads with shuffles / barriers by rendezvous) in the launch order of hbls.cu's
// aggregate-verify pipeline, so the device LOGIC -- mask complement sums, strided batch groups, failed-group lists, result
// codes -- is diffed against the oracle on the GPU-less build box.  Never linked into libhbls.so; the product has no CPU path.
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
static inline unsigned __ballot_sync(unsigned, bool p) { return p ? 1u : 0u; }      // k_pairing_coop itself is not run here (see emu_vm_pairing)
#include "../../harmony_b200/csrc/pairing.cuh"
static inline void __syncthreads() { if (blockDim.x == 2) hb::hb_emu_exchange(0); }       // 2-thread CTA: rendezvous; 1-thread: nothing
static inline unsigned atomicAdd(unsigned* p, unsigned v) { unsigned o = *p; *p += v; return o; }
static inline long long clock64() { return 0; }
template <class T> static inline T __shfl_down_sync(unsigned, T v, int) { return v; }       // warp-cooperative kernels are not run here
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

// The aggregate-verify pipeline of hbls.cu (agg_verify_device_locked + launch_verify_tail) with groups of G rounds.
// mode 1: batched groups + exact fallback, mode 0: exact only.  Returns 0, or -3 if a committee key does not decode.
// chunk: groups per pass of the line buffer (hbls.cu rlc_chunk_groups(), one wave of the line kernel on the device).  0: the group
// form in two halves and the exact forms in one pass; > 0: every loop of launch_verify_tail / launch_exact_two_phase over chunks of
// that many groups, the exact pass over the failed groups' list sized for the worst case (every round) as on the device.
template <int G> static int aggregate_verify_batch(int mode, uint32_t n, const uint8_t* pks48, size_t B, const uint8_t* bitmaps, size_t blen,
                                          const uint8_t* sigs96, const uint8_t* msgs, uint32_t msg_len, uint64_t s0, uint64_t s1,
                                          uint8_t* results, int* any_fail_out, uint8_t* group_ok_out, int* groups_failed_out, size_t chunk) {
    std::vector<g1a> table(n), pkneg(B), pk_scaled(B); std::vector<uint8_t> okk(n), ok_sig(B), ok_hm(B), bad(B), group_ok(B / G + 1);
    std::vector<g1> apk(B); std::vector<g2a> sig(B), hm(B), Sg(B / G + 1); std::vector<g2> S(B);
    run_seq(1, n, [&] { k_g1_decode(n, pks48, table.data(), okk.data(), 1, 0); });
    for (uint32_t i = 0; i < n; i++) if (!okk[i]) return -3;
    g1 total; pt_set_inf(total);
    for (uint32_t i = 0; i < n; i++) pt_add_mixed(total, total, table[i]);
    run_seq(2, 3, [&] { k_mask_aggregate_serial(B, n, table.data(), &total, bitmaps, blen, apk.data()); });     // grid-stride: 6 "threads"
    run_seq(2, 2, [&] { k_g2_decode(B, sigs96, sig.data(), ok_sig.data(), 1); });
    run_seq(3, 1, [&] { k_hash_to_g2(B, msgs, msg_len, hm.data(), ok_hm.data()); });
    int any_fail = 0; bool two_phase_mismatch = false, unwritten = false; std::vector<uint8_t> list_check;
    auto exact = [&](size_t off, size_t cnt, const int* run_if) {
        run_seq(1, (unsigned)cnt, [&] { k_g1_normalize(cnt, apk.data() + off, pkneg.data() + off, 1, run_if); });
        run_pair([&] { k_pairing_verify_split(cnt, sig.data() + off, pkneg.data() + off, hm.data() + off, ok_sig.data() + off, ok_hm.data() + off,
                                              (const uint8_t*)nullptr, results + off, run_if); });
        run_seq(1, 2, [&] { k_pairing_fixup(cnt, sig.data() + off, pkneg.data() + off, hm.data() + off, ok_sig.data() + off, ok_hm.data() + off,
                                            (const uint8_t*)nullptr, results + off, run_if); });
        if (run_if == nullptr && cnt) {      // the same verdicts through the line / accumulator kernels with "groups" of one round (hbls.cu launch_exact_two_phase)
            const size_t W = chunk ? chunk : cnt;
            std::vector<uint8_t> bad1(cnt), verdict(cnt, 0xee), res2(cnt, 0xee);
            std::vector<fp> lines((size_t)HB_ML_STEPS * 3 * 2 * (W < cnt ? W : cnt) * 2);          // one chunk's lines, reused
            run_seq(1, (unsigned)cnt, [&] { k_exact_prepare(cnt, (const uint32_t*)nullptr, sig.data() + off, pkneg.data() + off, hm.data() + off, ok_sig.data() + off, ok_hm.data() + off,
                                                            (const uint8_t*)nullptr, (g1a*)nullptr, (g2a*)nullptr, (g2a*)nullptr, bad1.data(), res2.data()); });
            for (size_t g0 = 0; g0 < cnt; g0 += W) {
                const size_t nc = cnt - g0 < W ? cnt - g0 : W;
                run_pair([&] { k_rlc_lines_split<1>(cnt, g0, nc, pkneg.data() + off, hm.data() + off, sig.data() + off, lines.data()); });
                run_pair([&] { k_rlc_accum_split<1>(cnt, g0, nc, lines.data(), bad1.data(), verdict.data()); });
            }
            for (size_t t = 0; t < cnt; t++) unwritten |= verdict[t] == 0xee;
            run_seq(1, (unsigned)cnt, [&] { k_exact_publish(cnt, (const uint32_t*)nullptr, verdict.data(), res2.data()); });
            run_seq(1, 2, [&] { k_pairing_fixup(cnt, sig.data() + off, pkneg.data() + off, hm.data() + off, ok_sig.data() + off, ok_hm.data() + off,
                                                (const uint8_t*)nullptr, res2.data(), (const int*)nullptr); });
            if (std::memcmp(res2.data(), results + off, cnt) != 0) two_phase_mismatch = true;
        }
    };
    if (mode == 1 && B >= (size_t)G) {
        const size_t ng = B / G, nr = ng * G, tail = B - nr;
        rlc_coeffs co;                                          // stands in for the host's ChaCha20 draw (hbls.cu rlc_draw)
        for (int k = 0; k < HB_RLC_GMAX; k++) { uint64_t x = s0 + 0x9e3779b97f4a7c15ull * (uint64_t)(k + 1); x ^= x >> 30; x *= 0xbf58476d1ce4e5b9ull; x ^= x >> 27; x ^= s1; co.c[k] = x; }
        run_seq(2, 2, [&] { k_rlc_scale(nr, ng, apk.data(), sig.data(), hm.data(), ok_sig.data(), ok_hm.data(), (const uint8_t*)nullptr, co, (const uint64_t*)nullptr, pk_scaled.data(), S.data(), bad.data()); });
        {   // the two-kernel form of the stage (one ladder per kernel) must produce the same points and flags
            std::vector<g1a> pk2(B); std::vector<g2> S2(B); std::vector<uint8_t> bad2(B, 0xee);
            run_seq(2, 2, [&] { k_rlc_scale_g1(nr, ng, apk.data(), co, pk2.data()); });
            run_seq(2, 2, [&] { k_rlc_scale_g2(nr, ng, apk.data(), sig.data(), hm.data(), ok_sig.data(), ok_hm.data(), (const uint8_t*)nullptr, co, S2.data(), bad2.data()); });
            if (std::memcmp(pk2.data(), pk_scaled.data(), nr * sizeof(g1a)) != 0 || std::memcmp(bad2.data(), bad.data(), nr) != 0) return -8;
            for (size_t j = 0; j < nr; j++) if (!pt_eq(S2[j], S[j])) return -8;
        }
        run_seq(1, 2, [&] { k_rlc_group_sum<G>(ng, S.data(), Sg.data()); });
        run_pair([&] { k_rlc_pairing_split<G>(ng, pk_scaled.data(), hm.data(), Sg.data(), bad.data(), group_ok.data()); });
        {   // the two-kernel form (lines to memory, then the accumulator) must give the same verdicts -- in chunks, like a large batch
            std::vector<uint8_t> gok2(ng + 1, 0xee);
            const size_t W = chunk ? chunk : (ng / 2 ? ng / 2 : ng);
            std::vector<fp> lines((size_t)HB_ML_STEPS * 3 * (G + 1) * (W < ng ? W : ng) * 2);    // one chunk's lines, reused
            for (size_t g0 = 0; g0 < ng; g0 += W) {
                const size_t ngc = ng - g0 < W ? ng - g0 : W;
                run_pair([&] { k_rlc_lines_split<G>(ng, g0, ngc, pk_scaled.data(), hm.data(), Sg.data(), lines.data()); });
                run_pair([&] { k_rlc_accum_split<G>(ng, g0, ngc, lines.data(), bad.data(), gok2.data()); });
            }
            if (std::memcmp(gok2.data(), group_ok.data(), ng) != 0) return -9;
        }
        std::vector<uint32_t> list(B); unsigned counts[2] = {0, 0};
        run_seq(2, (unsigned)((nr + 1) / 2), [&] { k_rlc_finish(nr, ng, group_ok.data(), results, list.data(), counts); });
        run_seq(1, 3, [&] { k_g1_normalize_list(&counts[0], list.data(), apk.data(), pkneg.data(), 1); });
        run_pair([&] { k_pairing_verify_split_list(&counts[0], list.data(), sig.data(), pkneg.data(), hm.data(), ok_sig.data(), ok_hm.data(), (const uint8_t*)nullptr, results); });
        std::vector<uint8_t> res_before(results, results + B);
        {   // the list through the line / accumulator kernels (gathered "groups" of one round, device-side count): same verdicts.  The
            // host loops over the worst case, nr listed rounds; chunks at or past the count must return at once and write nothing
            std::vector<uint8_t> res2(B); std::vector<uint32_t> list2(B); unsigned counts2[2] = {0, 0};
            run_seq(2, (unsigned)((nr + 1) / 2), [&] { k_rlc_finish(nr, ng, group_ok.data(), res2.data(), list2.data(), counts2); });
            const size_t W = chunk ? chunk : nr;
            std::vector<g1a> pk_c(B); std::vector<g2a> hm_c(B), sig_c(B); std::vector<uint8_t> bad1(B, 0), verdict(B, 0xee);
            std::vector<fp> lines((size_t)HB_ML_STEPS * 3 * 2 * (W < nr ? W : nr) * 2);
            run_seq(1, (unsigned)nr, [&] { k_exact_prepare(nr, list2.data(), sig.data(), pkneg.data(), hm.data(), ok_sig.data(), ok_hm.data(), (const uint8_t*)nullptr,
                                                           pk_c.data(), hm_c.data(), sig_c.data(), bad1.data(), res2.data(), &counts2[0]); });
            for (size_t g0 = 0; g0 < nr; g0 += W) {
                const size_t nc = nr - g0 < W ? nr - g0 : W;
                run_pair([&] { k_rlc_lines_split<1>(nr, g0, nc, pk_c.data(), hm_c.data(), sig_c.data(), lines.data(), &counts2[0]); });
                run_pair([&] { k_rlc_accum_split<1>(nr, g0, nc, lines.data(), bad1.data(), verdict.data(), &counts2[0]); });
            }
            for (size_t t = 0; t < counts2[0]; t++) unwritten |= verdict[t] == 0xee;
            for (size_t t = counts2[0]; t < B; t++) if (verdict[t] != 0xee) return -10;       // written past the device-side count
            run_seq(1, (unsigned)nr, [&] { k_exact_publish(nr, list2.data(), verdict.data(), res2.data(), &counts2[0]); });
            run_seq(1, 2, [&] { k_pairing_fixup_list(&counts2[0], list2.data(), sig.data(), pkneg.data(), hm.data(), ok_sig.data(), ok_hm.data(), (const uint8_t*)nullptr, res2.data()); });
            list_check = std::move(res2);
        }
        run_seq(1, 2, [&] { k_pairing_fixup_list(&counts[0], list.data(), sig.data(), pkneg.data(), hm.data(), ok_sig.data(), ok_hm.data(), (const uint8_t*)nullptr, results); });
        if (std::memcmp(list_check.data(), results, nr) != 0) two_phase_mismatch = true;
        any_fail = counts[0] != 0;
        if (groups_failed_out) *groups_failed_out = (int)counts[1];
        if (tail) exact(nr, tail, nullptr);
        if (group_ok_out) std::memcpy(group_ok_out, group_ok.data(), ng);
    } else {
        exact(0, B, nullptr);
    }
    if (any_fail_out) *any_fail_out = any_fail;
    if (unwritten) return -11;              // a round of the exact two-kernel forms got no verdict (a chunk skipped or cut short)
    if (two_phase_mismatch) return -7;
    return 0;
}
extern "C" int emu_aggregate_verify_batch(int mode, uint32_t n, const uint8_t* pks48, size_t B, const uint8_t* bitmaps, size_t blen,
                                          const uint8_t* sigs96, const uint8_t* msgs, uint32_t msg_len, uint64_t s0, uint64_t s1,
                                          uint8_t* results, int* any_fail_out, uint8_t* group_ok_out, int G, int* groups_failed_out, size_t chunk) {
    return G == 8 ? aggregate_verify_batch<8>(mode, n, pks48, B, bitmaps, blen, sigs96, msgs, msg_len, s0, s1, results, any_fail_out, group_ok_out, groups_failed_out, chunk)
                  : aggregate_verify_batch<4>(mode, n, pks48, B, bitmaps, blen, sigs96, msgs, msg_len, s0, s1, results, any_fail_out, group_ok_out, groups_failed_out, chunk);
}

// Executed Fp multiplications / squarings of the thread-per-item stages (mask aggregation from the complement side, signature
// decode, hash-to-G2, coefficient scaling + group sums), summed over B rounds: out[2 s] = mul, out[2 s + 1] = sqr for stage s in
// that order.  bench.py's roofline uses these per-round figures (x300 / x234 MAC32); tests/test_emu_kernels.py pins them.
extern "C" int emu_stage_counts(uint32_t n, const uint8_t* pks48, size_t B, const uint8_t* bitmaps, size_t blen, const uint8_t* sigs96,
                                const uint8_t* msgs, uint32_t msg_len, int G, uint64_t* out) {
    std::vector<g1a> table(n), pk_scaled(B); std::vector<uint8_t> okk(n), ok_sig(B), ok_hm(B), bad(B);
    std::vector<g1> apk(B); std::vector<g2a> sig(B), hm(B), Sg(B / G + 1); std::vector<g2> S(B);
    run_seq(1, n, [&] { k_g1_decode(n, pks48, table.data(), okk.data(), 1, 0); });
    for (uint32_t i = 0; i < n; i++) if (!okk[i]) return -3;
    g1 total; pt_set_inf(total);
    for (uint32_t i = 0; i < n; i++) pt_add_mixed(total, total, table[i]);
    uint64_t m0 = hb_emu_cnt_mul, s0 = hb_emu_cnt_sqr; int st = 0;
    auto mark = [&] { out[2 * st] = hb_emu_cnt_mul - m0; out[2 * st + 1] = hb_emu_cnt_sqr - s0; m0 = hb_emu_cnt_mul; s0 = hb_emu_cnt_sqr; st++; };
    run_seq(1, 4, [&] { k_mask_aggregate_serial(B, n, table.data(), &total, bitmaps, blen, apk.data()); }); mark();
    run_seq(1, 4, [&] { k_g2_decode(B, sigs96, sig.data(), ok_sig.data(), 1); }); mark();
    run_seq(1, 4, [&] { k_hash_to_g2(B, msgs, msg_len, hm.data(), ok_hm.data()); }); mark();
    const size_t ng = B / G, nr = ng * G;
    rlc_coeffs co; for (int k = 0; k < HB_RLC_GMAX; k++) co.c[k] = 0x9e3779b97f4a7c15ull * (uint64_t)(k + 3) ^ 0x5851f42d4c957f2dull;
    run_seq(1, 4, [&] { k_rlc_scale(nr, ng, apk.data(), sig.data(), hm.data(), ok_sig.data(), ok_hm.data(), (const uint8_t*)nullptr, co, (const uint64_t*)nullptr, pk_scaled.data(), S.data(), bad.data()); });
    if (G == 8) run_seq(1, 2, [&] { k_rlc_group_sum<8>(ng, S.data(), Sg.data()); }); else run_seq(1, 2, [&] { k_rlc_group_sum<4>(ng, S.data(), Sg.data()); });
    mark();
    return 0;
}

// ---- warp-cooperative pairing (vm.cuh): the step programs of vm_programs.cuh executed with the DEVICE instruction decoders
// (vm_mul / vm_sqr / vm_lin) -- the 32 lanes of a step one after the other (lanes of a step do not communicate; steps are
// separated by __syncwarp on the device).  Checks the binary encoding, the slot layout and the lane roles against the oracle.
static void emu_vm_run(int prog, uint32_t* slots) {
    const int first = VM_PROG_FIRST[prog], n = VM_PROG_STEPS[prog];
    for (int st = first; st < first + n; st++) {
        const uint32_t hdr = VM_STEP_HDR[st]; const int cls = hdr & 0xff;
        // every lane reads before any lane's result becomes visible: stage the stores
        std::vector<uint32_t> snap(slots, slots + VM_SMEM_WORDS), next(slots, slots + VM_SMEM_WORDS);
        for (int lane = 0; lane < 32; lane++) {
            const uint4* ip = VM_INS + ((size_t)st * 16 + (lane >> 1)) * (VM_INS_WORDS / 4);
            const uint32_t w0 = ip[0].x; const int dst = w0 & 0xff, im = lane & 1;
            if (dst == 0xff) continue;
            std::vector<uint32_t> work(snap);
            if (cls == VM_OP_LIN) vm_lin(work.data(), dst, ip[1 + im], (int)(hdr >> 8), im);
            else if (cls == VM_OP_SQR) vm_sqr(work.data(), dst, (w0 >> 8) & 0xff, im);
            else vm_mul(work.data(), dst, (w0 >> 8) & 0xff, (w0 >> 16) & 0xff, im);
            for (int j = 0; j < 12; j++) next[dst * VM_SLOT_WORDS + im * 12 + j] = work[dst * VM_SLOT_WORDS + im * 12 + j];
        }
        std::memcpy(slots, next.data(), VM_SMEM_WORDS * 4);
    }
}
static void emu_cycsqr_run(uint32_t* slots, int run) {
    while (run >= 16) { emu_vm_run(VM_P_CYCSQR16, slots); run -= 16; }
    if (run & 8) emu_vm_run(VM_P_CYCSQR8, slots);
    if (run & 4) emu_vm_run(VM_P_CYCSQR4, slots);
    if (run & 2) emu_vm_run(VM_P_CYCSQR2, slots);
    if (run & 1) emu_vm_run(VM_P_CYCSQR, slots);
}
static void emu_vm_expz(uint32_t* slots) {
    int run = 0;
    for (int i = 62; i >= 0; i--) { run++; if ((K_Z_ABS >> i) & 1) { emu_cycsqr_run(slots, run); run = 0; emu_vm_run(VM_P_MULX, slots); } }
    emu_cycsqr_run(slots, run);
}
// 1 / 0 = verdict of e(B, sig) e(-pk, H(msg)) == 1 through the VM; -1 undecodable input
extern "C" int emu_vm_pairing(const uint8_t* pk48, const uint8_t* sig96, const uint8_t* msg, uint32_t len) {
    g1 pk; g2 sg, h;
    if (!g1_deserialize(pk, pk48, true) || !g2_deserialize(sg, sig96, true) || !map_to_g2(h, msg, len)) return -1;
    g1a pa; g2a sa, ha; pt_to_aff(pa, pk); fp_neg(pa.y, pa.y); pt_to_aff(sa, sg); pt_to_aff(ha, h);
    std::vector<uint32_t> sl(VM_SMEM_WORDS, 0); uint32_t* slots = sl.data();
    for (unsigned lane = 0; lane < 32; lane++) { threadIdx = {lane, 0, 0}; vm_load_consts(slots); }
    threadIdx = {0, 0, 0};
    fp2 v; fp2_zero(v);
    fp_set(v.a, K_G1_X); vm_set_fp2(slots, VM_R_P1X, v); fp_set(v.a, K_G1_Y); vm_set_fp2(slots, VM_R_P1Y, v);
    vm_set_fp2(slots, VM_R_Q1X, sa.x); vm_set_fp2(slots, VM_R_Q1Y, sa.y);
    v.a = pa.x; vm_set_fp2(slots, VM_R_P2X, v); v.a = pa.y; vm_set_fp2(slots, VM_R_P2Y, v);
    vm_set_fp2(slots, VM_R_Q2X, ha.x); vm_set_fp2(slots, VM_R_Q2Y, ha.y);
    emu_vm_run(VM_P_ML_INIT, slots);
    for (int i = 62; i >= 0; ) {
        if ((K_Z_ABS >> i) & 1) { emu_vm_run(VM_P_ML_DBL, slots); emu_vm_run(VM_P_ML_ADD, slots); i--; }
        else if (i >= 1 && !((K_Z_ABS >> (i - 1)) & 1)) { emu_vm_run(VM_P_ML_DBL2, slots); i -= 2; }
        else { emu_vm_run(VM_P_ML_DBL, slots); i--; }
    }
    emu_vm_run(VM_P_FE_INV_A, slots);
    { fp n, ni; vm_ld(n.l, slots, VM_R_NORM, 0); fp_inv_gcd(ni, n); vm_set_fp(slots, VM_R_NINV, ni); }
    emu_vm_run(VM_P_FE_INV_B, slots);
    emu_vm_expz(slots); emu_vm_run(VM_P_GLUE1, slots);
    emu_vm_expz(slots); emu_vm_run(VM_P_GLUE2, slots);
    emu_vm_expz(slots); emu_vm_run(VM_P_GLUE3, slots);
    emu_vm_expz(slots); emu_vm_run(VM_P_GLUE4, slots);
    emu_vm_expz(slots); emu_vm_run(VM_P_GLUE5, slots); emu_vm_run(VM_P_GLUE6, slots);
    fp one; fp_one(one); uint32_t diff = 0;
    for (int lane = 0; lane < 12; lane++) {
        fp x; vm_ld(x.l, slots, VM_R_ACC0 + (lane >> 1), lane & 1);
        for (int j = 0; j < 12; j++) diff |= x.l[j] ^ (lane == 0 ? one.l[j] : 0u);
    }
    return diff == 0 ? 1 : 0;
}

// hash-to-G2 with the cofactor clearing on the VM (k_hash_to_g2_coop's arithmetic: G2_INIT .. G2_AFF through the device decoders)
// against the thread-per-item kernel: 1 identical point, 0 different, -1 the map is undefined for this message, -2 degenerate
static void emu_g2_dbl_run(uint32_t* slots, int run) {
    while (run >= 16) { emu_vm_run(VM_P_G2DBL16, slots); run -= 16; }
    if (run & 8) emu_vm_run(VM_P_G2DBL8, slots);
    if (run & 4) emu_vm_run(VM_P_G2DBL4, slots);
    if (run & 2) emu_vm_run(VM_P_G2DBL2, slots);
    if (run & 1) emu_vm_run(VM_P_G2DBL, slots);
}
static void emu_g2_zmul(uint32_t* slots) {
    int run = 0;
    for (int i = 62; i >= 0; i--) { run++; if ((K_Z_ABS >> i) & 1) { emu_g2_dbl_run(slots, run); run = 0; emu_vm_run(VM_P_G2_ADD, slots); } }
    emu_g2_dbl_run(slots, run);
}
extern "C" int emu_vm_hash(const uint8_t* msg, uint32_t len) {
    g2a want; uint8_t okw = 0;
    run_seq(1, 1, [&] { k_hash_to_g2(1, msg, len, &want, &okw); });
    fp2 t; hash_to_fp(t.a, msg, len); fp_zero(t.b);
    g2 a; if (!sw_map_g2<true>(a, t)) return okw ? 0 : -1;
    std::vector<uint32_t> sl(VM_SMEM_WORDS, 0); uint32_t* slots = sl.data();
    for (unsigned lane = 0; lane < 32; lane++) { threadIdx = {lane, 0, 0}; vm_load_consts(slots); }
    threadIdx = {0, 0, 0};
    vm_set_fp2(slots, VM_R_Q2X, a.x); vm_set_fp2(slots, VM_R_Q2Y, a.y);
    emu_vm_run(VM_P_G2_INIT, slots); emu_g2_zmul(slots);
    emu_vm_run(VM_P_HC_MID, slots); emu_g2_zmul(slots);
    emu_vm_run(VM_P_HC_FIN, slots); emu_vm_run(VM_P_G2_NORM, slots);
    fp n, ni; vm_ld(n.l, slots, VM_R_NORM, 0);
    if (fp_is_zero(n)) return -2;
    fp_inv_gcd(ni, n); vm_set_fp(slots, VM_R_NINV, ni);
    emu_vm_run(VM_P_G2_AFF, slots);
    g2a got; vm_ld(got.x.a.l, slots, VM_R_HX, 0); vm_ld(got.x.b.l, slots, VM_R_HX, 1); vm_ld(got.y.a.l, slots, VM_R_HY, 0); vm_ld(got.y.b.l, slots, VM_R_HY, 1);
    return (okw && std::memcmp(&got, &want, sizeof(g2a)) == 0) ? 1 : 0;
}

// blsSignHash's ladder over psi (k_sign_hm_gls_pair, base-|z| digits of the key) on two host threads against the plain 255-bit ladder of
// k_sign_hash: 1 = the same group element, 0 = different, -1 = the message maps to no point
extern "C" int emu_sign_gls(const uint8_t* sk32, const uint8_t* msg, uint32_t len) {
    g2 want; uint8_t okw = 0;
    run_seq(1, 1, [&] { k_sign_hash(1, sk32, msg, len, &want, &okw); });
    if (!okw) return -1;
    g2a hm; uint8_t okh = 0;
    run_seq(1, 1, [&] { k_hash_to_g2(1, msg, len, &hm, &okh); });
    uint64_t v[4], dig[4]; std::memcpy(v, sk32, 32);
    const uint64_t Z = 0xd201000000010000ull;
    for (int k = 0; k < 3; k++) {
        unsigned __int128 rem = 0;
        for (int i = 3; i >= 0; i--) { const unsigned __int128 cur = (rem << 64) | v[i]; v[i] = (uint64_t)(cur / Z); rem = cur % Z; }
        dig[k] = (uint64_t)rem;
    }
    dig[3] = v[0];
    if (v[1] | v[2] | v[3]) return -2;
    g2 got; uint8_t okg = 0;
    run_pair([&] { k_sign_hm_gls_pair(1, dig, &hm, &okh, 0, &got, &okg); });
    return (okg && pt_eq(got, want)) ? 1 : 0;
}

// lane-pair decode / hash kernels (latency path) on two host threads against the thread-per-item kernels: bit 0 = decoded
// signature identical (point and ok flag), bit 1 = H(m) identical; n items one after the other (pair 0 of a 2-thread CTA)
extern "C" int emu_pair_decode_hash(size_t n, const uint8_t* sigs96, const uint8_t* msgs, uint32_t len) {
    std::vector<g2a> s1(n), s2(n), h1(n), h2(n); std::vector<uint8_t> o1(n), o2(n), k1(n), k2(n);
    run_seq(1, (unsigned)n, [&] { k_g2_decode(n, sigs96, s1.data(), o1.data(), 1); });
    run_seq(1, (unsigned)n, [&] { k_hash_to_g2(n, msgs, len, h1.data(), k1.data()); });
    int res = 3;
    for (size_t i = 0; i < n; i++) {
        run_pair([&] { k_g2_decode_pair(1, sigs96 + 96 * i, &s2[i], &o2[i], 1); });
        run_pair([&] { k_hash_to_g2_pair(1, msgs + (size_t)len * i, len, &h2[i], &k2[i]); });
        if (o1[i] != o2[i] || std::memcmp(&s1[i], &s2[i], sizeof(g2a)) != 0) res &= ~1;
        if (k1[i] != k2[i] || std::memcmp(&h1[i], &h2[i], sizeof(g2a)) != 0) res &= ~2;
    }
    return res;
}

// the decode kernels of every entry point on n serialized points (48 bytes for forms 0-2, 96 for forms 3-8): ok[i] = 1 decoded,
// 0 rejected.  form 0 k_g1_decode, 1 k_g1_decode_jac, 2 k_single OP_G1_DES, 3 k_g2_decode, 4 k_g2_decode (no order check) +
// k_g2_subgroup, 5 k_g2_decode_pair, 6 k_g2_decode_pair (no order check) + k_g2_subgroup_pair, 7 k_single OP_G2_DES, 8 k_single
// OP_G2_DES_ADD.  check = 0 drops the subgroup test from forms 0, 1, 3 and 5 (the decode alone).  Returns 0, or -1 for an unknown form.
extern "C" int emu_decode_flags(int form, int check, size_t n, const uint8_t* in, uint8_t* ok) {
    std::vector<g1a> p1(n); std::vector<g1> j1(n); std::vector<g2a> p2(n); std::vector<g2> j2(n);
    auto single = [&](int op, size_t w) {
        std::vector<single_desc> d(n); std::vector<int> rc(n, -5);
        for (size_t i = 0; i < n; i++) { pt_set_inf(j2[i]); d[i] = single_desc{in + w * i, nullptr, op == OP_G1_DES ? (void*)&j1[i] : (void*)&j2[i], op, 0u}; }
        run_seq(1, (unsigned)n, [&] { k_single(n, d.data(), d[0], rc.data()); });
        for (size_t i = 0; i < n; i++) ok[i] = rc[i] == (int)w ? 1 : 0;
    };
    switch (form) {
    case 0: run_seq(1, (unsigned)n, [&] { k_g1_decode(n, in, p1.data(), ok, check, 0); }); break;
    case 1: run_seq(1, (unsigned)n, [&] { k_g1_decode_jac(n, in, j1.data(), ok, check); }); break;
    case 2: single(OP_G1_DES, 48); break;
    case 3: run_seq(1, (unsigned)n, [&] { k_g2_decode(n, in, p2.data(), ok, check); }); break;
    case 4: run_seq(1, (unsigned)n, [&] { k_g2_decode(n, in, p2.data(), ok, 0); });
            run_seq(1, (unsigned)n, [&] { k_g2_subgroup(n, p2.data(), ok); }); break;
    case 5: for (size_t i = 0; i < n; i++) run_pair([&] { k_g2_decode_pair(1, in + 96 * i, &p2[i], &ok[i], check); }); break;
    case 6: { std::vector<uint8_t> dec(n);
            for (size_t i = 0; i < n; i++) run_pair([&] { k_g2_decode_pair(1, in + 96 * i, &p2[i], &dec[i], 0); });
            for (size_t i = 0; i < n; i++) run_pair([&] { k_g2_subgroup_pair(1, &p2[i], &dec[i], &ok[i]); }); break; }
    case 7: single(OP_G2_DES, 96); break;
    case 8: single(OP_G2_DES_ADD, 96); break;
    default: return -1;
    }
    return 0;
}
