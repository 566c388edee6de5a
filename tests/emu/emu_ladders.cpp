// tests/emu/emu_ladders.cpp -- TEST HARNESS ONLY: the large-batch lane-pair ladder kernels (k_g2_subgroup_pair with zeroing,
// k_hash_cofactor_pair, k_rlc_scale_g2_pair) on two host threads against the thread-per-item kernels they replace in hbls.cu
// (k_g2_subgroup, k_hash_cofactor_jac, k_rlc_scale_g2).  Every function returns the number of items whose outputs differ in any
// byte (points in their stored form and flags), so 0 means bit-for-bit equal.  Reuses emu_kernels.cpp's host shims and launchers.
#include "emu_kernels.cpp"

// n serialized signatures decoded without the order test, then the subgroup test of both forms; ok_out = the pair kernel's flags
extern "C" int emu_ladder_subgroup(size_t n, const uint8_t* sigs96, uint8_t* ok_out) {
    std::vector<g2a> p1(n), p2(n); std::vector<uint8_t> o1(n), o2(n);
    run_seq(1, (unsigned)n, [&] { k_g2_decode(n, sigs96, p1.data(), o1.data(), 0); });
    p2 = p1; o2 = o1;
    run_seq(2, 3, [&] { k_g2_subgroup(n, p1.data(), o1.data()); });
    run_pair([&] { k_g2_subgroup_pair(n, p2.data(), o2.data(), o2.data(), 1); });
    int diff = 0;
    for (size_t i = 0; i < n; i++) diff += (o1[i] != o2[i] || std::memcmp(&p1[i], &p2[i], sizeof(g2a)) != 0) ? 1 : 0;
    std::memcpy(ok_out, o2.data(), n);
    return diff;
}

// n messages through the SW map (k_hash_sw); items whose drop[i] is set lose their ok flag (an undecodable item); then the cofactor
// clearing of both forms into Jacobian points
extern "C" int emu_ladder_cofactor(size_t n, const uint8_t* msgs, uint32_t len, const uint8_t* drop) {
    std::vector<g2a> pts(n); std::vector<uint8_t> ok(n); std::vector<g2> h1(n), h2(n);
    run_seq(2, 3, [&] { k_hash_sw(n, msgs, len, pts.data(), ok.data()); });
    for (size_t i = 0; i < n; i++) if (drop[i]) ok[i] = 0;
    run_seq(2, 3, [&] { k_hash_cofactor_jac(n, pts.data(), ok.data(), h1.data()); });
    run_pair([&] { k_hash_cofactor_pair(n, pts.data(), ok.data(), h2.data()); });
    int diff = 0;
    for (size_t i = 0; i < n; i++) diff += std::memcmp(&h1[i], &h2[i], sizeof(g2)) != 0 ? 1 : 0;
    return diff;
}

// coefficient scaling of the signatures: n rounds (keys, signatures, messages), groups of G = n / ng; blocks != 0 uses per-(position,
// member) coefficients with the block stride of hbls.cu.  The coefficients come from the seed; position 0 (member 0) keeps 1.
extern "C" int emu_ladder_scale(size_t n, const uint8_t* pks48, const uint8_t* sigs96, const uint8_t* msgs, uint32_t len, size_t ng,
                                uint64_t seed, int blocks) {
    std::vector<g1> apk(n); std::vector<g2a> sig(n), hm(n); std::vector<uint8_t> okp(n), oks(n), okh(n), b1(n, 0xee), b2(n, 0xee);
    std::vector<g2> s1(n), s2(n);
    run_seq(1, (unsigned)n, [&] { k_g1_decode_jac(n, pks48, apk.data(), okp.data(), 1); });
    run_seq(1, (unsigned)n, [&] { k_g2_decode(n, sigs96, sig.data(), oks.data(), 1); });
    run_seq(1, (unsigned)n, [&] { k_hash_to_g2(n, msgs, len, hm.data(), okh.data()); });
    rlc_coeffs co; rlc_block_coeffs cb;
    uint64_t x = seed;
    auto next = [&] { x += 0x9e3779b97f4a7c15ull; uint64_t z = x; z = (z ^ (z >> 30)) * 0xbf58476d1ce4e5b9ull; z = (z ^ (z >> 27)) * 0x94d049bb133111ebull; return z ^ (z >> 31); };
    for (int k = 0; k < HB_RLC_GMAX; k++) { co.c[k] = next(); for (int m = 0; m < HB_RLC_M; m++) cb.c[k][m] = next(); }
    const size_t S = blocks ? (((ng + HB_RLC_M - 1) / HB_RLC_M + 31) & ~(size_t)31) : 0;
    const size_t nr = ng * (n / ng);
    run_seq(2, 3, [&] { k_rlc_scale_g2(nr, ng, apk.data(), sig.data(), hm.data(), oks.data(), okh.data(), okp.data(), co, s1.data(), b1.data(), S, cb); });
    run_pair([&] { k_rlc_scale_g2_pair(nr, ng, apk.data(), sig.data(), hm.data(), oks.data(), okh.data(), okp.data(), co, s2.data(), b2.data(), S, cb); });
    int diff = 0;
    for (size_t j = 0; j < nr; j++) diff += (b1[j] != b2[j] || std::memcmp(&s1[j], &s2[j], sizeof(g2)) != 0) ? 1 : 0;
    return diff;
}
