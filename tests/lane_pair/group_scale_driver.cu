// tests/lane_pair/group_scale_driver.cu -- TEST HARNESS ONLY (compiled by tests/test_group_scale.py): the joint per-group ladder of the
// coefficient stage (k_rlc_group_scale_g2_pair + k_g2_normalize_batch) against the per-round form (k_rlc_scale_g2_pair +
// k_rlc_group_sum<G>) on the device, each kernel launched with the geometry hbls.cu gives it.  Returns the number of groups whose affine
// sums differ in any byte plus the number of rounds whose bad flags differ, or -1 on a CUDA error.
#include <cuda_runtime.h>
#include <cstring>
#include <vector>
#include "../../harmony_b200/csrc/kernels.cuh"
using namespace hb;

namespace {
int sms() { int d = 0, n = 0; cudaGetDevice(&d); cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, d); return n; }
unsigned thread_grid(size_t n, unsigned per_sm) { size_t need = (n + 63) / 64, cap = (size_t)sms() * (per_sm / 64); return (unsigned)(need < cap ? need : cap); }
unsigned pair_grid(size_t n) { size_t need = (2 * n + 511) / 512; return (unsigned)(need < (size_t)sms() ? need : sms()); }
template <class T> T* up(const void* h, size_t n) { T* d = nullptr; cudaMalloc(&d, n * sizeof(T)); if (h) cudaMemcpy(d, h, n * sizeof(T), cudaMemcpyHostToDevice); return d; }
template <class T> std::vector<T> down(const T* d, size_t n) { std::vector<T> h(n); cudaMemcpy(h.data(), d, n * sizeof(T), cudaMemcpyDeviceToHost); return h; }
template <class T> int count_diff(const std::vector<T>& a, const std::vector<T>& b) {
    int diff = 0;
    for (size_t i = 0; i < a.size(); i++) diff += std::memcmp(&a[i], &b[i], sizeof(T)) != 0 ? 1 : 0;
    return diff;
}
template <int G> void per_round(size_t ng, const g1* apk, const g2a* sig, const g2a* hm, const uint8_t* okp, const uint8_t* oks, const uint8_t* okh,
                                const rlc_coeffs& co, const rlc_block_coeffs& cb, size_t S, g2* s1, g2a* sg, uint8_t* bad) {
    k_rlc_scale_g2_pair<<<pair_grid(ng * G), 512>>>(ng * G, ng, apk, sig, hm, oks, okh, okp, co, s1, bad, S, cb, nullptr);
    k_rlc_group_sum<G><<<thread_grid(ng, 384), 64>>>(ng, s1, sg);
}
template <int G> void joint(size_t ng, const g1* apk, const g2a* sig, const g2a* hm, const uint8_t* okp, const uint8_t* oks, const uint8_t* okh,
                            const rlc_coeffs& co, const rlc_block_coeffs& cb, size_t S, g2* j, g2a* sg, uint8_t* bad) {
    k_rlc_group_scale_g2_pair<G><<<pair_grid(ng), 512>>>(ng, apk, sig, hm, oks, okh, okp, co, j, bad, S, cb, nullptr);
    k_g2_normalize_batch<<<thread_grid(ng, 384), 64>>>(ng, j, sg);
}
}  // namespace

// n rounds (keys, signatures, messages) in ng groups of G = n / ng; coeffs = 8 per-position coefficients followed by 8 x 16
// per-(position, member) ones; blocks != 0 selects the block stride
extern "C" int gs_compare(size_t n, const uint8_t* pks48, const uint8_t* sigs96, const uint8_t* msgs, uint32_t len, size_t ng,
                          const uint64_t* coeffs, int blocks) {
    const size_t G = n / ng, nr = ng * G;
    if (G != 4 && G != 8) return -2;
    uint8_t *dk = up<uint8_t>(pks48, 48 * n), *ds = up<uint8_t>(sigs96, 96 * n), *dm = up<uint8_t>(msgs, (size_t)len * n);
    g1* apk = up<g1>(nullptr, n); g2a *sig = up<g2a>(nullptr, n), *hm = up<g2a>(nullptr, n), *sg1 = up<g2a>(nullptr, ng), *sg2 = up<g2a>(nullptr, ng);
    uint8_t *okp = up<uint8_t>(nullptr, n), *oks = up<uint8_t>(nullptr, n), *okh = up<uint8_t>(nullptr, n), *b1 = up<uint8_t>(nullptr, n), *b2 = up<uint8_t>(nullptr, n);
    g2 *s1 = up<g2>(nullptr, n), *j2 = up<g2>(nullptr, ng);
    cudaMemset(b1, 0xee, n); cudaMemset(b2, 0xee, n);
    k_g1_decode_jac<<<thread_grid(n, 384), 64>>>(n, dk, apk, okp, 1);
    k_g2_decode<<<thread_grid(n, 512), 64>>>(n, ds, sig, oks, 1);
    k_hash_to_g2<<<thread_grid(n, 384), 64>>>(n, dm, len, hm, okh);
    rlc_coeffs co; rlc_block_coeffs cb;
    std::memcpy(co.c, coeffs, sizeof co.c); std::memcpy(cb.c, coeffs + HB_RLC_GMAX, sizeof cb.c);
    const size_t S = blocks ? (((ng + HB_RLC_M - 1) / HB_RLC_M + 31) & ~(size_t)31) : 0;
    if (G == 8) { per_round<8>(ng, apk, sig, hm, okp, oks, okh, co, cb, S, s1, sg1, b1); joint<8>(ng, apk, sig, hm, okp, oks, okh, co, cb, S, j2, sg2, b2); }
    else { per_round<4>(ng, apk, sig, hm, okp, oks, okh, co, cb, S, s1, sg1, b1); joint<4>(ng, apk, sig, hm, okp, oks, okh, co, cb, S, j2, sg2, b2); }
    const bool ok = cudaDeviceSynchronize() == cudaSuccess && cudaGetLastError() == cudaSuccess;
    const int r = ok ? count_diff(down(sg1, ng), down(sg2, ng)) + count_diff(down(b1, nr), down(b2, nr)) : -1;
    for (void* p : {(void*)dk, (void*)ds, (void*)dm, (void*)apk, (void*)sig, (void*)hm, (void*)sg1, (void*)sg2, (void*)okp, (void*)oks, (void*)okh,
                    (void*)b1, (void*)b2, (void*)s1, (void*)j2}) cudaFree(p);
    return r;
}
