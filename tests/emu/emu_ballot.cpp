// tests/emu/emu_ballot.cpp -- TEST HARNESS ONLY: hbls_ballot_box_submit_votes run on the host in hbls.cu's launch order, on top of the
// emulation of emu_kernels.cpp: same-message aggregate verification in its exact form (mask sums from the committee table, signature
// decode, H(m) once, lane-pair pairing on two host threads), then the admission scan k_ballot_admit and the fold k_ballot_fold as
// CTAs of two threads on two host threads (barriers by rendezvous, shared memory shared): the per-vote barrier, the alternating
// "already collected" stamp, the chunk restaging and the tree of the fold run as on the device.  The admission also runs as a CTA of
// one thread and must give the same bytes.  Never linked into libhbls.so.
#include "emu_kernels.cpp"

// One queue of k votes on msg into a box given by its collected bitmap (blen bytes, in/out) and its running sum (Jacobian, the
// 288-byte layout of blsSignature, in/out; all-zero = identity).  status[j] = HBLS_BALLOT_* code, sum96 = the serialized sum.
// Returns 0, -3 (a committee key does not decode), -2 (bitmap wider than the kernel's shared-memory box) or -4 (one thread and two
// threads disagree).
extern "C" int emu_ballot_submit(uint32_t n, const uint8_t* pks48, size_t k, const uint8_t* bitmaps, size_t blen, const uint8_t* sigs96,
                                 const uint8_t* msg, uint32_t msg_len, uint8_t* collected, uint8_t* sum_jac, uint8_t* status, uint8_t* sum96) {
    if (blen > HB_BALLOT_MAX_BYTES) return -2;
    std::vector<g1a> table(n), pkneg(k); std::vector<uint8_t> okk(n), ok_sig(k), ok_hm(k), res(k), acc(k), col_out(blen + 1);
    std::vector<g1> apk(k); std::vector<g2a> sig(k), hm(k);
    run_seq(1, n, [&] { k_g1_decode(n, pks48, table.data(), okk.data(), 1, 0); });
    for (uint32_t i = 0; i < n; i++) if (!okk[i]) return -3;
    g1 total; pt_set_inf(total);
    for (uint32_t i = 0; i < n; i++) pt_add_mixed(total, total, table[i]);
    run_seq(2, 3, [&] { k_mask_aggregate_serial(k, n, table.data(), &total, bitmaps, blen, apk.data()); });
    run_seq(2, 2, [&] { k_g2_decode(k, sigs96, sig.data(), ok_sig.data(), 1); });
    run_seq(1, 1, [&] { k_hash_to_g2(1, msg, msg_len, hm.data(), ok_hm.data()); });          // one message: hashed once, broadcast
    for (size_t j = 1; j < k; j++) { hm[j] = hm[0]; ok_hm[j] = ok_hm[0]; }
    run_seq(1, (unsigned)k, [&] { k_g1_normalize(k, apk.data(), pkneg.data(), 1, (const int*)nullptr); });
    run_pair([&] { k_pairing_verify_split(k, sig.data(), pkneg.data(), hm.data(), ok_sig.data(), ok_hm.data(), (const uint8_t*)nullptr, res.data(), (const int*)nullptr); });
    run_seq(1, 2, [&] { k_pairing_fixup(k, sig.data(), pkneg.data(), hm.data(), ok_sig.data(), ok_hm.data(), (const uint8_t*)nullptr, res.data(), (const int*)nullptr); });
    run_pair([&] { k_ballot_admit(k, n, blen, bitmaps, res.data(), ok_sig.data(), collected, col_out.data(), status, acc.data()); });
    std::vector<uint8_t> st1(k + 1), acc1(k + 1), col1(blen + 1);
    run_seq(1, 1, [&] { k_ballot_admit(k, n, blen, bitmaps, res.data(), ok_sig.data(), collected, col1.data(), st1.data(), acc1.data()); });
    if (std::memcmp(st1.data(), status, k) || std::memcmp(acc1.data(), acc.data(), k) || std::memcmp(col1.data(), col_out.data(), blen)) return -4;
    g2 sum; std::memcpy(&sum, sum_jac, sizeof(g2));
    run_pair([&] { k_ballot_fold(k, sig.data(), acc.data(), &sum); });
    run_seq(1, 1, [&] { k_g2_serialize(1, &sum, sum96); });
    std::memcpy(sum_jac, &sum, sizeof(g2));
    std::memcpy(collected, col_out.data(), blen);
    return 0;
}
extern "C" size_t emu_g2_jac_bytes() { return sizeof(g2); }
