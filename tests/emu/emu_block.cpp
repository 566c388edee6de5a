// tests/emu/emu_block.cpp -- TEST HARNESS ONLY: the block form of the batched verify (hbls.cu rlc_blocks: HB_RLC_M groups share one
// final exponentiation and one generator pair) run on the host in hbls.cu's launch order, on top of the emulation of emu_kernels.cpp.
// The warp-per-block check k_rlc_block_coop is replayed with the device's own VM decoders (emu_vm_run), the lane-pair kernels run on
// two host threads.  Never linked into libhbls.so.
#include "emu_kernels.cpp"

// k_rlc_block_coop for block b: the same program sequence, the lanes of a step one after the other
static uint8_t emu_block_check(size_t b, size_t S, size_t ng, const fp2* fm, const g2a& Sb, const uint8_t* group_ok) {
    for (size_t g = b; g < ng; g += S) if (!group_ok[g]) return 0;
    std::vector<uint32_t> sl(VM_SMEM_WORDS, 0); uint32_t* slots = sl.data();
    for (unsigned lane = 0; lane < 32; lane++) { threadIdx = {lane, 0, 0}; vm_load_consts(slots); }
    threadIdx = {0, 0, 0};
    emu_vm_run(VM_P_A_ONE, slots);
    for (size_t g = b; g < ng; g += S) {
        for (int t = 0; t < 6; t++) vm_set_fp2(slots, VM_R_F0 + t, fm[6 * g + t]);
        emu_vm_run(VM_P_AMULF, slots);
    }
    if (aff_is_inf(Sb)) return 0;
    fp2 v; fp2_zero(v);
    fp_set(v.a, K_G1_X); vm_set_fp2(slots, VM_R_P2X, v); fp_set(v.a, K_G1_Y); vm_set_fp2(slots, VM_R_P2Y, v);
    vm_set_fp2(slots, VM_R_Q2X, Sb.x); vm_set_fp2(slots, VM_R_Q2Y, Sb.y);
    emu_vm_run(VM_P_ML1_INIT, slots);
    for (int i = 62; i >= 0; i--) {
        emu_vm_run(VM_P_ML1_DBL, slots);
        if ((K_Z_ABS >> i) & 1) emu_vm_run(VM_P_ML1_ADD, slots);
    }
    emu_vm_run(VM_P_FMULA, slots);
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

// The aggregate-verify pipeline with blocks: groups of G rounds (round j in group j mod ng), group g member g / S of block g mod S.
// S = 0: the library's choice (ceil(ng / 16) rounded up to a multiple of 32); a smaller S puts several groups into one block with tiny
// batches.  equal_members = 1 replaces the per-member draw by the per-position coefficients of the group form (member m's rounds at
// position k all get c[k], position 0 keeps 1): two bad rounds at one position of two groups of a block then cancel.
// Returns 0, -3 (a committee key does not decode) or -10 (the groups' verdicts differ from the group form's without blocks, which runs
// alongside on the same rounds).  blocks_failed_out / fallback_out: failed blocks, groups checked alone.
template <int G> static int block_verify(uint32_t n, const uint8_t* pks48, size_t B, const uint8_t* bitmaps, size_t blen, const uint8_t* sigs96,
                                         const uint8_t* msgs, uint32_t msg_len, size_t S, uint64_t s0, uint64_t s1, int equal_members,
                                         uint8_t* results, uint8_t* group_ok_out, int* blocks_failed_out, int* fallback_out) {
    std::vector<g1a> table(n), pkneg(B), pk_scaled(B); std::vector<uint8_t> okk(n), ok_sig(B), ok_hm(B), bad(B);
    std::vector<g1> apk(B); std::vector<g2a> sig(B), hm(B); std::vector<g2> Sj(B);
    run_seq(1, n, [&] { k_g1_decode(n, pks48, table.data(), okk.data(), 1, 0); });
    for (uint32_t i = 0; i < n; i++) if (!okk[i]) return -3;
    g1 total; pt_set_inf(total);
    for (uint32_t i = 0; i < n; i++) pt_add_mixed(total, total, table[i]);
    run_seq(2, 3, [&] { k_mask_aggregate_serial(B, n, table.data(), &total, bitmaps, blen, apk.data()); });
    run_seq(2, 2, [&] { k_g2_decode(B, sigs96, sig.data(), ok_sig.data(), 1); });
    run_seq(3, 1, [&] { k_hash_to_g2(B, msgs, msg_len, hm.data(), ok_hm.data()); });
    const size_t ng = B / G, nr = ng * G, tail = B - nr;
    if (!S) S = ((ng + HB_RLC_M - 1) / HB_RLC_M + 31) & ~(size_t)31;
    if (S * HB_RLC_M < ng) return -11;                          // a block holds at most HB_RLC_M groups
    auto mix = [&](uint64_t i) { uint64_t x = s0 + 0x9e3779b97f4a7c15ull * (i + 1); x ^= x >> 30; x *= 0xbf58476d1ce4e5b9ull; x ^= x >> 27; return x ^ s1; };
    rlc_coeffs co; rlc_block_coeffs cb;                          // stand in for the host's ChaCha20 draws (hbls.cu rlc_draw / rlc_draw_block)
    for (int k = 0; k < HB_RLC_GMAX; k++) {
        co.c[k] = mix(k);
        for (int m = 0; m < HB_RLC_M; m++) cb.c[k][m] = equal_members ? (k ? co.c[k] : 1ull) : mix(100 + HB_RLC_M * k + m);
    }
    // coefficient scaling: the two-kernel form and the one-kernel form give the same points and flags
    run_seq(2, 2, [&] { k_rlc_scale_g1(nr, ng, apk.data(), co, pk_scaled.data(), S, cb); });
    run_seq(2, 2, [&] { k_rlc_scale_g2(nr, ng, apk.data(), sig.data(), hm.data(), ok_sig.data(), ok_hm.data(), (const uint8_t*)nullptr, co, Sj.data(), bad.data(), S, cb); });
    {
        std::vector<g1a> pk2(B); std::vector<g2> S2(B); std::vector<uint8_t> bad2(B, 0xee);
        run_seq(2, 2, [&] { k_rlc_scale(nr, ng, apk.data(), sig.data(), hm.data(), ok_sig.data(), ok_hm.data(), (const uint8_t*)nullptr, co, (const uint64_t*)nullptr,
                                        pk2.data(), S2.data(), bad2.data(), S, cb); });
        if (std::memcmp(pk2.data(), pk_scaled.data(), nr * sizeof(g1a)) != 0 || std::memcmp(bad2.data(), bad.data(), nr) != 0) return -8;
        for (size_t j = 0; j < nr; j++) if (!pt_eq(S2[j], Sj[j])) return -8;
    }
    std::vector<g2a> Sg(ng + 1), Sb(S); std::vector<uint8_t> group_ok(ng + 1, 0xee), block_ok(S, 0xee);
    run_seq(1, 2, [&] { k_rlc_group_sum<G>(ng, Sj.data(), Sg.data()); });
    std::vector<fp> lines((size_t)HB_ML_STEPS * 3 * (G + 1) * ng * 2);
    fp2* fm = reinterpret_cast<fp2*>(lines.data() + (size_t)HB_ML_STEPS * 3 * G * ng * 2);       // the groups' Miller values (hbls.cu: VerifyBufs::fm)
    const unsigned* nocount = nullptr;
    run_pair([&] { k_rlc_lines_blk<G>(ng, 0, ng, pk_scaled.data(), hm.data(), lines.data(), nocount); });
    run_pair([&] { k_rlc_accum_blk<G>(ng, 0, ng, lines.data(), bad.data(), group_ok.data(), fm, nocount); });
    run_seq(1, 2, [&] { k_rlc_block_sum(S, ng, Sg.data(), Sb.data()); });
    int bf = 0;
    for (size_t b = 0; b < S; b++) { block_ok[b] = emu_block_check(b, S, ng, fm, Sb[b], group_ok.data()); bf += (b < ng && !block_ok[b]) ? 1 : 0; }
    std::vector<uint32_t> glist(ng + 1); unsigned gcount = 0;
    run_seq(1, (unsigned)ng, [&] { k_rlc_block_list(ng, S, block_ok.data(), group_ok.data(), glist.data(), &gcount); });
    run_pair([&] { k_rlc_group_check_list(&gcount, glist.data(), fm, Sg.data(), group_ok.data()); });
    if (blocks_failed_out) *blocks_failed_out = bf;
    if (fallback_out) *fallback_out = (int)gcount;
    // the group form without blocks on the same rounds (per-position coefficients, G + 1 pairs and a final exponentiation per group)
    if (!equal_members) {
        std::vector<g1a> pk1(B); std::vector<g2> S1(B); std::vector<uint8_t> bad1(B); std::vector<g2a> Sg1(ng + 1); std::vector<uint8_t> gok1(ng + 1, 0xee);
        run_seq(2, 2, [&] { k_rlc_scale(nr, ng, apk.data(), sig.data(), hm.data(), ok_sig.data(), ok_hm.data(), (const uint8_t*)nullptr, co, (const uint64_t*)nullptr,
                                        pk1.data(), S1.data(), bad1.data()); });
        run_seq(1, 2, [&] { k_rlc_group_sum<G>(ng, S1.data(), Sg1.data()); });
        std::vector<fp> lines1((size_t)HB_ML_STEPS * 3 * (G + 1) * ng * 2);
        run_pair([&] { k_rlc_lines_split<G>(ng, 0, ng, pk1.data(), hm.data(), Sg1.data(), lines1.data()); });
        run_pair([&] { k_rlc_accum_split<G>(ng, 0, ng, lines1.data(), bad1.data(), gok1.data()); });
        if (std::memcmp(gok1.data(), group_ok.data(), ng) != 0) return -10;
    }
    // from here on the pipeline of the group form: per-round results, exact pass over the rounds of failed groups, tail
    std::vector<uint32_t> list(B); unsigned counts[2] = {0, 0};
    run_seq(2, (unsigned)((nr + 1) / 2), [&] { k_rlc_finish(nr, ng, group_ok.data(), results, list.data(), counts); });
    run_seq(1, 3, [&] { k_g1_normalize_list(&counts[0], list.data(), apk.data(), pkneg.data(), 1); });
    run_pair([&] { k_pairing_verify_split_list(&counts[0], list.data(), sig.data(), pkneg.data(), hm.data(), ok_sig.data(), ok_hm.data(), (const uint8_t*)nullptr, results); });
    run_seq(1, 2, [&] { k_pairing_fixup_list(&counts[0], list.data(), sig.data(), pkneg.data(), hm.data(), ok_sig.data(), ok_hm.data(), (const uint8_t*)nullptr, results); });
    if (tail) {
        run_seq(1, (unsigned)tail, [&] { k_g1_normalize(tail, apk.data() + nr, pkneg.data() + nr, 1, (const int*)nullptr); });
        run_pair([&] { k_pairing_verify_split(tail, sig.data() + nr, pkneg.data() + nr, hm.data() + nr, ok_sig.data() + nr, ok_hm.data() + nr,
                                              (const uint8_t*)nullptr, results + nr, (const int*)nullptr); });
        run_seq(1, 2, [&] { k_pairing_fixup(tail, sig.data() + nr, pkneg.data() + nr, hm.data() + nr, ok_sig.data() + nr, ok_hm.data() + nr,
                                            (const uint8_t*)nullptr, results + nr, (const int*)nullptr); });
    }
    if (group_ok_out) std::memcpy(group_ok_out, group_ok.data(), ng);
    return 0;
}
extern "C" int emu_block_verify(uint32_t n, const uint8_t* pks48, size_t B, const uint8_t* bitmaps, size_t blen, const uint8_t* sigs96,
                                const uint8_t* msgs, uint32_t msg_len, int G, size_t S, uint64_t s0, uint64_t s1, int equal_members,
                                uint8_t* results, uint8_t* group_ok_out, int* blocks_failed_out, int* fallback_out) {
    return G == 8 ? block_verify<8>(n, pks48, B, bitmaps, blen, sigs96, msgs, msg_len, S, s0, s1, equal_members, results, group_ok_out, blocks_failed_out, fallback_out)
                  : block_verify<4>(n, pks48, B, bitmaps, blen, sigs96, msgs, msg_len, S, s0, s1, equal_members, results, group_ok_out, blocks_failed_out, fallback_out);
}
