// tests/emu/emu_zladders.cpp -- TEST HARNESS ONLY: the |z| ladders hbls.cu runs with an affine base, on two host threads: the subgroup
// test k_g2_subgroup_pair (g2_in_subgroup_aff) against the thread kernel k_g2_subgroup, and the cofactor clearing
// k_hash_cofactor_z1_pair + k_hash_cofactor_z2_pair (g2_clear_cofactor_aff_z1 / _z2) against k_hash_cofactor_pair, both followed by
// k_g2_normalize_batch.  Every function returns the number of items whose outputs differ in any byte.  Reuses emu_kernels.cpp's host
// shims and launchers.
#include "emu_kernels.cpp"

// n serialized points decoded without the order test; items with drop[i] lose their ok flag; then both subgroup tests (zeroing).
// ok_out = the pair kernel's flags
extern "C" int emu_zl_subgroup(size_t n, const uint8_t* pts96, const uint8_t* drop, uint8_t* ok_out) {
    std::vector<g2a> p1(n), p2(n); std::vector<uint8_t> o1(n), o2(n);
    run_seq(1, (unsigned)n, [&] { k_g2_decode(n, pts96, p1.data(), o1.data(), 0); });
    for (size_t i = 0; i < n; i++) if (drop[i]) o1[i] = 0;
    p2 = p1; o2 = o1;
    run_seq(2, 3, [&] { k_g2_subgroup(n, p1.data(), o1.data()); });
    run_pair([&] { k_g2_subgroup_pair(n, p2.data(), o2.data(), o2.data(), 1); });
    int diff = 0;
    for (size_t i = 0; i < n; i++) diff += (o1[i] != o2[i] || std::memcmp(&p1[i], &p2[i], sizeof(g2a)) != 0) ? 1 : 0;
    std::memcpy(ok_out, o2.data(), n);
    return diff;
}

// np serialized points decoded without the order test (items 0 .. np) and nm messages through the SW map (items np .. np + nm); items
// with drop[i] lose their ok flag; then both cofactor clearings and the affine conversion.  ok_out = the flags the clearings saw.
extern "C" int emu_zl_cofactor(size_t np, const uint8_t* pts96, size_t nm, const uint8_t* msgs, uint32_t len, const uint8_t* drop,
                               uint8_t* ok_out) {
    const size_t n = np + nm;
    std::vector<g2a> pts(n), a1(n), a2(n); std::vector<uint8_t> ok(n); std::vector<g2> h1(n), h2(n);
    run_seq(1, (unsigned)np, [&] { k_g2_decode(np, pts96, pts.data(), ok.data(), 0); });
    run_seq(2, 3, [&] { k_hash_sw(nm, msgs, len, pts.data() + np, ok.data() + np); });
    for (size_t i = 0; i < n; i++) if (drop[i]) ok[i] = 0;
    run_pair([&] { k_hash_cofactor_pair(n, pts.data(), ok.data(), h1.data()); });
    run_pair([&] { k_hash_cofactor_z1_pair(n, pts.data(), ok.data(), h2.data()); });
    run_pair([&] { k_hash_cofactor_z2_pair(n, pts.data(), ok.data(), h2.data()); });
    run_seq(1, 3, [&] { k_g2_normalize_batch(n, h1.data(), a1.data()); });
    run_seq(1, 3, [&] { k_g2_normalize_batch(n, h2.data(), a2.data()); });
    int diff = 0;
    for (size_t i = 0; i < n; i++) diff += std::memcmp(&a1[i], &a2[i], sizeof(g2a)) != 0 ? 1 : 0;
    std::memcpy(ok_out, ok.data(), n);
    return diff;
}
