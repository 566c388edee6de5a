// tests/lane_pair/ladders_driver.cu -- TEST HARNESS ONLY (compiled by tests/test_lane_pair_ladders.py): the large-batch lane-pair
// ladder kernels against the thread-per-item kernels they replace in hbls.cu, on the device, with the launch geometry hbls.cu uses
// for each.  Every entry point returns the number of items whose outputs differ in any byte, or -1 on a CUDA error.
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
int done(int diff) { return cudaDeviceSynchronize() == cudaSuccess && cudaGetLastError() == cudaSuccess ? diff : -1; }
}  // namespace

// n signatures decoded without the order test, then k_g2_subgroup against k_g2_subgroup_pair (zeroing): points and flags
extern "C" int lp_subgroup(size_t n, const uint8_t* sigs96, uint8_t* ok_out) {
    uint8_t* din = up<uint8_t>(sigs96, 96 * n);
    g2a *p1 = up<g2a>(nullptr, n), *p2 = up<g2a>(nullptr, n); uint8_t *o1 = up<uint8_t>(nullptr, n), *o2 = up<uint8_t>(nullptr, n);
    k_g2_decode<<<thread_grid(n, 512), 64>>>(n, din, p1, o1, 0);
    cudaMemcpy(p2, p1, n * sizeof(g2a), cudaMemcpyDeviceToDevice); cudaMemcpy(o2, o1, n, cudaMemcpyDeviceToDevice);
    k_g2_subgroup<<<thread_grid(n, 512), 64>>>(n, p1, o1);
    k_g2_subgroup_pair<<<pair_grid(n), 512>>>(n, p2, o2, o2, 1);
    const int r = done(count_diff(down(p1, n), down(p2, n)) + count_diff(down(o1, n), down(o2, n)));
    cudaMemcpy(ok_out, o2, n, cudaMemcpyDeviceToHost);
    cudaFree(din); cudaFree(p1); cudaFree(p2); cudaFree(o1); cudaFree(o2);
    return r;
}

// n messages through k_hash_sw; items with drop[i] lose their ok flag; then k_hash_cofactor_jac against k_hash_cofactor_pair
extern "C" int lp_cofactor(size_t n, const uint8_t* msgs, uint32_t len, const uint8_t* drop) {
    uint8_t* dm = up<uint8_t>(msgs, (size_t)len * n);
    g2a* pts = up<g2a>(nullptr, n); uint8_t* ok = up<uint8_t>(nullptr, n); g2 *h1 = up<g2>(nullptr, n), *h2 = up<g2>(nullptr, n);
    k_hash_sw<<<thread_grid(n, 512), 64>>>(n, dm, len, pts, ok);
    std::vector<uint8_t> okh = down(ok, n);
    for (size_t i = 0; i < n; i++) if (drop[i]) okh[i] = 0;
    cudaMemcpy(ok, okh.data(), n, cudaMemcpyHostToDevice);
    k_hash_cofactor_jac<<<thread_grid(n, 512), 64>>>(n, pts, ok, h1);
    k_hash_cofactor_pair<<<pair_grid(n), 512>>>(n, pts, ok, h2);
    const int r = done(count_diff(down(h1, n), down(h2, n)));
    cudaFree(dm); cudaFree(pts); cudaFree(ok); cudaFree(h1); cudaFree(h2);
    return r;
}

// n rounds (keys, signatures, messages) in groups of n / ng: k_rlc_scale_g2 against k_rlc_scale_g2_pair, S and the bad flags.
// coeffs = 8 per-position coefficients followed by 8 x 16 per-(position, member) ones; blocks != 0 selects the block stride.
extern "C" int lp_scale(size_t n, const uint8_t* pks48, const uint8_t* sigs96, const uint8_t* msgs, uint32_t len, size_t ng,
                        const uint64_t* coeffs, int blocks) {
    uint8_t *dk = up<uint8_t>(pks48, 48 * n), *ds = up<uint8_t>(sigs96, 96 * n), *dm = up<uint8_t>(msgs, (size_t)len * n);
    g1* apk = up<g1>(nullptr, n); g2a *sig = up<g2a>(nullptr, n), *hm = up<g2a>(nullptr, n);
    uint8_t *okp = up<uint8_t>(nullptr, n), *oks = up<uint8_t>(nullptr, n), *okh = up<uint8_t>(nullptr, n), *b1 = up<uint8_t>(nullptr, n), *b2 = up<uint8_t>(nullptr, n);
    g2 *s1 = up<g2>(nullptr, n), *s2 = up<g2>(nullptr, n);
    k_g1_decode_jac<<<thread_grid(n, 384), 64>>>(n, dk, apk, okp, 1);
    k_g2_decode<<<thread_grid(n, 512), 64>>>(n, ds, sig, oks, 1);
    k_hash_to_g2<<<thread_grid(n, 384), 64>>>(n, dm, len, hm, okh);
    rlc_coeffs co; rlc_block_coeffs cb;
    std::memcpy(co.c, coeffs, sizeof co.c); std::memcpy(cb.c, coeffs + HB_RLC_GMAX, sizeof cb.c);
    const size_t S = blocks ? (((ng + HB_RLC_M - 1) / HB_RLC_M + 31) & ~(size_t)31) : 0, nr = ng * (n / ng);
    k_rlc_scale_g2<<<thread_grid(nr, 384), 64>>>(nr, ng, apk, sig, hm, oks, okh, okp, co, s1, b1, S, cb, nullptr);
    k_rlc_scale_g2_pair<<<pair_grid(nr), 512>>>(nr, ng, apk, sig, hm, oks, okh, okp, co, s2, b2, S, cb, nullptr);
    const int r = done(count_diff(down(s1, nr), down(s2, nr)) + count_diff(down(b1, nr), down(b2, nr)));
    for (void* p : {(void*)dk, (void*)ds, (void*)dm, (void*)apk, (void*)sig, (void*)hm, (void*)okp, (void*)oks, (void*)okh, (void*)b1, (void*)b2, (void*)s1, (void*)s2}) cudaFree(p);
    return r;
}
