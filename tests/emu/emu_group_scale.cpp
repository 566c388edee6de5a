// tests/emu/emu_group_scale.cpp -- TEST HARNESS ONLY: the joint per-group ladder of the coefficient stage (k_rlc_group_scale_g2_pair
// on two host threads, then k_g2_normalize_batch) against the per-round form it replaces for large batches (k_rlc_scale_g2 +
// k_rlc_group_sum<G>), and the executed Fp products of both.  Reuses emu_kernels.cpp's host shims and launchers.
#include "emu_kernels.cpp"

namespace {
struct Rounds { std::vector<g1> apk; std::vector<g2a> sig, hm; std::vector<uint8_t> okp, oks, okh; };
Rounds decode_rounds(size_t n, const uint8_t* pks48, const uint8_t* sigs96, const uint8_t* msgs, uint32_t len) {
    Rounds r; r.apk.resize(n); r.sig.resize(n); r.hm.resize(n); r.okp.resize(n); r.oks.resize(n); r.okh.resize(n);
    run_seq(1, (unsigned)n, [&] { k_g1_decode_jac(n, pks48, r.apk.data(), r.okp.data(), 1); });
    run_seq(1, (unsigned)n, [&] { k_g2_decode(n, sigs96, r.sig.data(), r.oks.data(), 1); });
    run_seq(1, (unsigned)n, [&] { k_hash_to_g2(n, msgs, len, r.hm.data(), r.okh.data()); });
    return r;
}
// coeffs = 8 per-position draws followed by 8 x 16 per-(position, member) draws
void unpack_coeffs(const uint64_t* coeffs, rlc_coeffs& co, rlc_block_coeffs& cb) {
    std::memcpy(co.c, coeffs, sizeof co.c); std::memcpy(cb.c, coeffs + HB_RLC_GMAX, sizeof cb.c);
}
size_t block_stride(size_t ng) { return ((ng + HB_RLC_M - 1) / HB_RLC_M + 31) & ~(size_t)31; }      // hbls.cu launch_verify_tail

template <int G> int group_scale(size_t n, const uint8_t* pks48, const uint8_t* sigs96, const uint8_t* msgs, uint32_t len, size_t ng,
                                 const uint64_t* coeffs, int blocks, int gate, uint8_t* bad_out, uint8_t* sg_out) {
    const Rounds r = decode_rounds(n, pks48, sigs96, msgs, len);
    rlc_coeffs co; rlc_block_coeffs cb; unpack_coeffs(coeffs, co, cb);
    const size_t S = blocks ? block_stride(ng) : 0, nr = ng * G;
    unsigned gv = gate < 0 ? 0u : (unsigned)gate; const unsigned* gp = gate < 0 ? nullptr : &gv;
    std::vector<g2> s1(nr), j2(ng); std::vector<g2a> sg1(ng), sg2(ng); std::vector<uint8_t> b1(nr, 0xee), b2(nr, 0xee);
    run_seq(2, 3, [&] { k_rlc_scale_g2(nr, ng, r.apk.data(), r.sig.data(), r.hm.data(), r.oks.data(), r.okh.data(), r.okp.data(), co, s1.data(), b1.data(), S, cb, gp); });
    run_seq(1, 2, [&] { k_rlc_group_sum<G>(ng, s1.data(), sg1.data()); });
    run_pair([&] { k_rlc_group_scale_g2_pair<G>(ng, r.apk.data(), r.sig.data(), r.hm.data(), r.oks.data(), r.okh.data(), r.okp.data(), co, j2.data(), b2.data(), S, cb, gp); });
    run_seq(1, 3, [&] { k_g2_normalize_batch(ng, j2.data(), sg2.data()); });
    int diff = 0;
    for (size_t g = 0; g < ng; g++) diff += std::memcmp(&sg1[g], &sg2[g], sizeof(g2a)) != 0 ? 1 : 0;
    for (size_t j = 0; j < nr; j++) diff += b1[j] != b2[j] ? 1 : 0;
    std::memcpy(bad_out, b2.data(), nr);
    for (size_t g = 0; g < ng; g++) {
        const fp* c[4] = {&sg2[g].x.a, &sg2[g].x.b, &sg2[g].y.a, &sg2[g].y.b};
        for (int i = 0; i < 4; i++) { fp v; fp_to_int(v, *c[i]); store_words(sg_out + 192 * g + 48 * i, v.l, 12); }
    }
    return diff;
}

// executed Fp mul / sqr of the stage's G2 side for n rounds in groups of G (per-position coefficients, the unit one at position 0), on
// the fp2 carrier: the lane-pair kernels run the same point formulas, but their split products are not counted.  out[0..1]: a
// ladder per round (rlc_scale_g2) + k_rlc_group_sum<G>; out[2..3]: the joint ladder per group (pt_mul_joint_naf over sigma_k and
// psi^2 sigma_k, as k_rlc_group_scale_g2_pair) + k_g2_normalize_batch, one group per thread as the device launches it.  Returns the
// number of groups whose affine sums differ.
template <int G> int group_scale_counts(size_t n, const uint8_t* sigs96, const uint64_t* coeffs, uint64_t* out) {
    std::vector<g2a> sig(n); std::vector<uint8_t> oks(n);
    run_seq(1, (unsigned)n, [&] { k_g2_decode(n, sigs96, sig.data(), oks.data(), 1); });
    rlc_coeffs co; rlc_block_coeffs cb; unpack_coeffs(coeffs, co, cb);
    const size_t ng = n / G, nr = ng * G;
    std::vector<g2> s1(nr), j2(ng); std::vector<g2a> sg1(ng), sg2(ng);
    uint64_t m0 = hb_emu_cnt_mul, q0 = hb_emu_cnt_sqr;
    for (size_t j = 0; j < nr; j++) {
        const uint64_t c = rlc_coeff(co, j, ng, 0, cb);
        if (c == 1ull) pt_from_aff(s1[j], sig[j]); else rlc_scale_g2(s1[j], sig[j], c);
    }
    run_seq(1, (unsigned)ng, [&] { k_rlc_group_sum<G>(ng, s1.data(), sg1.data()); });
    out[0] = hb_emu_cnt_mul - m0; out[1] = hb_emu_cnt_sqr - q0; m0 = hb_emu_cnt_mul; q0 = hb_emu_cnt_sqr;
    for (size_t g = 0; g < ng; g++) {
        uint32_t k[2 * G];
        for (int t = 0; t < G; t++) { const uint64_t c = rlc_coeff(co, (size_t)t * ng + g, ng, 0, cb); k[2 * t] = (uint32_t)c | 1u; k[2 * t + 1] = (uint32_t)(c >> 32); }
        pt_mul_joint_naf<fp2, 2 * G>(j2[g], k, [&](int t, g2a& q) {
            q = sig[(size_t)(t >> 1) * ng + g];
            if (t & 1) { fp2_mul_fp(q.x, q.x, fp_k(K_PSI2_CX)); fp2_neg(q.y, q.y); }
        });
    }
    run_seq(1, (unsigned)ng, [&] { k_g2_normalize_batch(ng, j2.data(), sg2.data()); });
    out[2] = hb_emu_cnt_mul - m0; out[3] = hb_emu_cnt_sqr - q0;
    int diff = 0;
    for (size_t g = 0; g < ng; g++) diff += std::memcmp(&sg1[g], &sg2[g], sizeof(g2a)) != 0 ? 1 : 0;
    return diff;
}
}  // namespace

// n rounds (keys, signatures, messages) in ng groups of G = 4 or 8 (n = ng G); blocks != 0: per-(position, member) coefficients with
// hbls.cu's member stride; gate < 0: no device gate, else its value (0 selects the per-position coefficients).  Returns the number of
// groups whose affine Sg differ in any byte plus the number of rounds whose bad flags differ; bad_out (n bytes) and sg_out (ng x 192
// bytes: x.a, x.b, y.a, y.b little-endian) receive the joint form's outputs.
extern "C" int emu_group_scale(int G, size_t n, const uint8_t* pks48, const uint8_t* sigs96, const uint8_t* msgs, uint32_t len, size_t ng,
                               const uint64_t* coeffs, int blocks, int gate, uint8_t* bad_out, uint8_t* sg_out) {
    if (n != ng * (size_t)G) return -1;
    return G == 8 ? group_scale<8>(n, pks48, sigs96, msgs, len, ng, coeffs, blocks, gate, bad_out, sg_out)
                  : group_scale<4>(n, pks48, sigs96, msgs, len, ng, coeffs, blocks, gate, bad_out, sg_out);
}
extern "C" int emu_group_scale_counts(int G, size_t n, const uint8_t* sigs96, const uint64_t* coeffs, uint64_t* out) {
    return G == 8 ? group_scale_counts<8>(n, sigs96, coeffs, out) : group_scale_counts<4>(n, sigs96, coeffs, out);
}
