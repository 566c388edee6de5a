// tests/emu/emu_coeff_source.cpp -- TEST HARNESS ONLY: the secrets of calls captured into a CUDA graph, on the host (HB_HOST_EMU).
// (1) The ChaCha20 block function of k_rlc_draw (kernels.cuh chacha20_block_dev) and the host stream's (chacha20.hpp).
// (2) The scaling kernels and k_group_insert fed their coefficients / salt through the device-pointer sources (rlc_coeffs_dev,
// rlc_block_coeffs_dev, grp_salt_dev) and through the by-value sources on the same values: the outputs must agree byte for byte.
// Reuses emu_kernels.cpp's host shims and launchers.  Never linked into libhbls.so; the product has no CPU path.
#include "emu_kernels.cpp"
static inline unsigned atomicCAS(unsigned* p, unsigned cmp, unsigned v) { unsigned o = *p; if (o == cmp) *p = v; return o; }
static inline unsigned atomicMin(unsigned* p, unsigned v) { unsigned o = *p; if (v < o) *p = v; return o; }
#include "../../harmony_b200/csrc/device_forms.cuh"
#include "../../harmony_b200/csrc/chacha20.hpp"

namespace {
struct Rounds { std::vector<g1> apk; std::vector<g2a> sig, hm; std::vector<uint8_t> okp, oks, okh; };
Rounds decode_rounds(size_t n, const uint8_t* pks48, const uint8_t* sigs96, const uint8_t* msgs, uint32_t len) {
    Rounds r; r.apk.resize(n); r.sig.resize(n); r.hm.resize(n); r.okp.resize(n); r.oks.resize(n); r.okh.resize(n);
    run_seq(1, (unsigned)n, [&] { k_g1_decode_jac(n, pks48, r.apk.data(), r.okp.data(), 1); });
    run_seq(1, (unsigned)n, [&] { k_g2_decode(n, sigs96, r.sig.data(), r.oks.data(), 1); });
    run_seq(1, (unsigned)n, [&] { k_hash_to_g2(n, msgs, len, r.hm.data(), r.okh.data()); });
    return r;
}
template <class T> int differ(const std::vector<T>& a, const std::vector<T>& b) {
    return a.size() != b.size() || std::memcmp(a.data(), b.data(), a.size() * sizeof(T)) != 0 ? 1 : 0;
}
// every scaling kernel hbls.cu launches, once per source; returns the number of outputs (arrays) that differ in any byte
template <int G, class CO, class CB> struct Out { std::vector<g1a> pk1, pk2; std::vector<g2> s1, s3, sg; std::vector<uint8_t> b1, b3, bg; };
template <int G, class CO, class CB> Out<G, CO, CB> scale_all(const Rounds& r, size_t ng, CO co, CB cb, size_t S, const unsigned* gp) {
    const size_t nr = ng * G;
    Out<G, CO, CB> o;
    o.pk1.assign(nr, g1a{}); o.pk2.assign(nr, g1a{}); o.s1.assign(nr, g2{}); o.s3.assign(nr, g2{}); o.sg.assign(ng, g2{});
    o.b1.assign(nr, 0xee); o.b3.assign(nr, 0xee); o.bg.assign(nr, 0xee);
    run_seq(2, 3, [&] { k_rlc_scale(nr, ng, r.apk.data(), r.sig.data(), r.hm.data(), r.oks.data(), r.okh.data(), r.okp.data(), co, (const uint64_t*)nullptr,
                                    o.pk1.data(), o.s1.data(), o.b1.data(), S, cb, gp); });
    run_seq(2, 3, [&] { k_rlc_scale_g1(nr, ng, r.apk.data(), co, o.pk2.data(), S, cb, gp); });
    run_pair([&] { k_rlc_scale_g2_pair(nr, ng, r.apk.data(), r.sig.data(), r.hm.data(), r.oks.data(), r.okh.data(), r.okp.data(), co, o.s3.data(), o.b3.data(), S, cb, gp); });
    run_pair([&] { k_rlc_group_scale_g2_pair<G>(ng, r.apk.data(), r.sig.data(), r.hm.data(), r.oks.data(), r.okh.data(), r.okp.data(), co, o.sg.data(), o.bg.data(), S, cb, gp); });
    return o;
}
template <int G> int scale_sources(size_t n, const uint8_t* pks48, const uint8_t* sigs96, const uint8_t* msgs, uint32_t len, size_t ng,
                                   const uint64_t* coeffs, int blocks, int gate) {
    const Rounds r = decode_rounds(n, pks48, sigs96, msgs, len);
    rlc_coeffs co; rlc_block_coeffs cb;
    std::memcpy(co.c, coeffs, sizeof co.c); std::memcpy(cb.c, coeffs + HB_RLC_GMAX, sizeof cb.c);
    const size_t S = blocks ? (((ng + HB_RLC_M - 1) / HB_RLC_M + 31) & ~(size_t)31) : 0;      // hbls.cu launch_verify_tail
    unsigned gv = gate < 0 ? 0u : (unsigned)gate; const unsigned* gp = gate < 0 ? nullptr : &gv;
    const auto v = scale_all<G>(r, ng, co, cb, S, gp);
    const auto d = scale_all<G>(r, ng, rlc_coeffs_dev{co.c}, rlc_block_coeffs_dev{cb.c}, S, gp);
    return differ(v.pk1, d.pk1) + differ(v.pk2, d.pk2) + differ(v.s1, d.s1) + differ(v.s3, d.s3) + differ(v.sg, d.sg)
         + differ(v.b1, d.b1) + differ(v.b3, d.b3) + differ(v.bg, d.bg);
}
}  // namespace

extern "C" {
// the device block function on a whole 16-word state
void emu_chacha_dev(const uint32_t st[16], uint32_t out[16]) { chacha20_block_dev(st, out); }
// the host stream's block `block` of call `counter`
void emu_chacha_host(const uint32_t key[8], uint64_t counter, uint32_t block, uint32_t out[16]) { chacha20_block(key, counter, out, block); }
// the device draw's nonce word (k_rlc_draw's HB_RLC_DRAW_NONCE)
uint32_t emu_draw_nonce(void) { return HB_RLC_DRAW_NONCE; }
// n = ng G rounds, coefficients = 8 per-position draws then 8 x 16 per-(position, member) draws; blocks != 0: hbls.cu's member stride;
// gate < 0: no device gate, else its value.  Returns the number of outputs that differ between the two sources (0: identical).
int emu_scale_sources(int G, size_t n, const uint8_t* pks48, const uint8_t* sigs96, const uint8_t* msgs, uint32_t len, size_t ng,
                      const uint64_t* coeffs, int blocks, int gate) {
    if (n != ng * (size_t)G) return -1;
    return G == 8 ? scale_sources<8>(n, pks48, sigs96, msgs, len, ng, coeffs, blocks, gate) : scale_sources<4>(n, pks48, sigs96, msgs, len, ng, coeffs, blocks, gate);
}
// k_group_insert over k messages, by value under salt (k0, k1) and through grp_salt_dev pointing at (j0, j1); returns the number of
// output arrays (slot items, slot representatives, item slots) that differ: 0 when the two runs agree
int emu_group_sources(size_t k, const uint8_t* msgs, uint32_t msg_len, uint64_t k0, uint64_t k1, uint64_t j0, uint64_t j1) {
    size_t T = 64; while (T < 2 * k) T <<= 1;
    std::vector<uint32_t> si[2], sr[2], is[2];
    const uint64_t salt[2] = {j0, j1};
    for (int src = 0; src < 2; src++) {
        si[src].assign(T, HB_GRP_EMPTY); sr[src].assign(T, HB_GRP_EMPTY); is[src].assign(k, 0);
        gridDim = {1, 1, 1}; blockDim = {(unsigned)k, 1, 1};
        for (size_t u = 0; u < k; u++) {
            threadIdx = {(unsigned)u, 0, 0};
            if (src == 0) k_group_insert(k, msgs, msg_len, (uint32_t)(T - 1), k0, k1, si[0].data(), sr[0].data(), is[0].data());
            else k_group_insert(k, msgs, msg_len, (uint32_t)(T - 1), grp_salt_dev{&salt[0]}, grp_salt_dev{&salt[1]}, si[1].data(), sr[1].data(), is[1].data());
        }
        blockDim = {1, 1, 1}; threadIdx = {0, 0, 0};
    }
    return differ(si[0], si[1]) + differ(sr[0], sr[1]) + differ(is[0], is[1]);
}
}
