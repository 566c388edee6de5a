// tests/zladders/zladders_driver.cu -- TEST HARNESS ONLY (compiled by tests/test_zladders.py): the |z| ladders hbls.cu runs with an
// affine base, on the device with the launch geometry hbls.cu gives them (one lock-stepped CTA per SM, `cta` resident threads): the
// subgroup test k_g2_subgroup_pair against the thread kernel k_g2_subgroup, and the cofactor clearing k_hash_cofactor_z1_pair +
// k_hash_cofactor_z2_pair against k_hash_cofactor_pair, both followed by k_g2_normalize_batch.  Every entry point returns the number of
// items whose outputs differ in any byte, or -1 on a CUDA error.
#include <cuda_runtime.h>
#include <cstring>
#include <vector>
#include "../../harmony_b200/csrc/kernels.cuh"
using namespace hb;

namespace {
int sms() { int d = 0, n = 0; cudaGetDevice(&d); cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, d); return n; }
unsigned thread_grid(size_t n, unsigned per_sm) { size_t need = (n + 63) / 64, cap = (size_t)sms() * (per_sm / 64); return (unsigned)(need < cap ? need : cap); }
unsigned pair_grid(size_t n, unsigned cta) { size_t need = (2 * n + cta - 1) / cta; return (unsigned)(need < (size_t)sms() ? need : sms()); }
template <class T> T* up(const void* h, size_t n) { T* d = nullptr; cudaMalloc(&d, n * sizeof(T)); if (h) cudaMemcpy(d, h, n * sizeof(T), cudaMemcpyHostToDevice); return d; }
template <class T> std::vector<T> down(const T* d, size_t n) { std::vector<T> h(n); cudaMemcpy(h.data(), d, n * sizeof(T), cudaMemcpyDeviceToHost); return h; }
template <class T> int count_diff(const std::vector<T>& a, const std::vector<T>& b) {
    int diff = 0;
    for (size_t i = 0; i < a.size(); i++) diff += std::memcmp(&a[i], &b[i], sizeof(T)) != 0 ? 1 : 0;
    return diff;
}
int done(int diff) { return cudaDeviceSynchronize() == cudaSuccess && cudaGetLastError() == cudaSuccess ? diff : -1; }
// the items' ok flags on the device, with those of drop[i] cleared
void drop_flags(uint8_t* ok, const uint8_t* drop, size_t n) {
    std::vector<uint8_t> h = down(ok, n);
    for (size_t i = 0; i < n; i++) if (drop[i]) h[i] = 0;
    cudaMemcpy(ok, h.data(), n, cudaMemcpyHostToDevice);
}
}  // namespace

// n serialized points decoded without the order test; items with drop[i] lose their ok flag; then k_g2_subgroup against
// k_g2_subgroup_pair (zeroing): points and flags.  ok_out = the pair kernel's flags
extern "C" int zl_subgroup(size_t n, const uint8_t* pts96, const uint8_t* drop, unsigned cta, uint8_t* ok_out) {
    uint8_t* din = up<uint8_t>(pts96, 96 * n);
    g2a *p1 = up<g2a>(nullptr, n), *p2 = up<g2a>(nullptr, n); uint8_t *o1 = up<uint8_t>(nullptr, n), *o2 = up<uint8_t>(nullptr, n);
    k_g2_decode<<<thread_grid(n, 512), 64>>>(n, din, p1, o1, 0);
    drop_flags(o1, drop, n);
    cudaMemcpy(p2, p1, n * sizeof(g2a), cudaMemcpyDeviceToDevice); cudaMemcpy(o2, o1, n, cudaMemcpyDeviceToDevice);
    k_g2_subgroup<<<thread_grid(n, 512), 64>>>(n, p1, o1);
    k_g2_subgroup_pair<<<pair_grid(n, cta), cta>>>(n, p2, o2, o2, 1);
    const int r = done(count_diff(down(p1, n), down(p2, n)) + count_diff(down(o1, n), down(o2, n)));
    cudaMemcpy(ok_out, o2, n, cudaMemcpyDeviceToHost);
    cudaFree(din); cudaFree(p1); cudaFree(p2); cudaFree(o1); cudaFree(o2);
    return r;
}

// np serialized points decoded without the order test (items 0 .. np) and nm messages through k_hash_sw (items np .. np + nm); items
// with drop[i] lose their ok flag; then k_hash_cofactor_pair against k_hash_cofactor_z1_pair + _z2_pair, each followed by
// k_g2_normalize_batch: the affine points.  ok_out = the flags the clearings saw
extern "C" int zl_cofactor(size_t np, const uint8_t* pts96, size_t nm, const uint8_t* msgs, uint32_t len, const uint8_t* drop, unsigned cta,
                           uint8_t* ok_out) {
    const size_t n = np + nm;
    uint8_t *din = up<uint8_t>(pts96, 96 * np), *dm = up<uint8_t>(msgs, (size_t)len * nm);
    g2a *pts = up<g2a>(nullptr, n), *a1 = up<g2a>(nullptr, n), *a2 = up<g2a>(nullptr, n); uint8_t* ok = up<uint8_t>(nullptr, n);
    g2 *h1 = up<g2>(nullptr, n), *h2 = up<g2>(nullptr, n);
    k_g2_decode<<<thread_grid(np, 512), 64>>>(np, din, pts, ok, 0);
    k_hash_sw<<<thread_grid(nm, 512), 64>>>(nm, dm, len, pts + np, ok + np);
    drop_flags(ok, drop, n);
    k_hash_cofactor_pair<<<pair_grid(n, cta), cta>>>(n, pts, ok, h1);
    k_hash_cofactor_z1_pair<<<pair_grid(n, cta), cta>>>(n, pts, ok, h2);
    k_hash_cofactor_z2_pair<<<pair_grid(n, cta), cta>>>(n, pts, ok, h2);
    k_g2_normalize_batch<<<thread_grid(n, 512), 64>>>(n, h1, a1);
    k_g2_normalize_batch<<<thread_grid(n, 512), 64>>>(n, h2, a2);
    const int r = done(count_diff(down(a1, n), down(a2, n)));
    cudaMemcpy(ok_out, ok, n, cudaMemcpyDeviceToHost);
    for (void* p : {(void*)din, (void*)dm, (void*)pts, (void*)a1, (void*)a2, (void*)ok, (void*)h1, (void*)h2}) cudaFree(p);
    return r;
}
