// tests/ct/ct_driver.cu -- TEST / MEASUREMENT HARNESS ONLY: the four secret-scalar kernels of kernels.cuh on the device.
// Built by tests/test_constant_time.py with -DHB_CT_PROBE_DEVICE: every HB_CT_PROBE the kernels execute (complete formulas, table reads,
// ladder steps) records, per thread, how many probes it passed, a hash of their tags and whether __activemask() was ever short of the
// full warp -- on the code nvcc emitted for sm_90a.  Built without it by tools/sign_timing.py, which times the kernels against the
// variable-time ladders they replaced (restated below as k_vt_*) with CUDA events.
#include <cuda_runtime.h>
#include <cstring>
#include <vector>
#include "../../harmony_b200/csrc/kernels.cuh"
using namespace hb;

struct CtRec { uint32_t count, partial; uint64_t hash; };
__device__ CtRec* ct_rec;
#ifdef HB_CT_PROBE_DEVICE
namespace hb {
__device__ void hb_ct_probe(uint32_t tag) {
    const unsigned m = __activemask();
    CtRec& r = ct_rec[blockIdx.x * blockDim.x + threadIdx.x];
    r.count++; r.partial |= m != 0xffffffffu ? 1u : 0u; r.hash = (r.hash ^ tag) * 0x100000001b3ull;
}
}
#endif

// ---- the variable-time ladders of the previous kernels (reference for timing only): pt_mul's fixed window with skipped zero windows,
// and the psi ladder that added the subset sum of each bit column when it was non-zero
__global__ void k_vt_g1_mul_gen(size_t n, const uint8_t* sk32, g1* out) {
    size_t i = HB_TID; if (i >= n) return;
    uint32_t k[8]; load_words(k, sk32 + 32 * i, 8);
    g1 g, r; g1_generator(g); pt_mul(r, g, k, 8); out[i] = r;
}
__global__ void k_vt_sign_hm_pair(size_t n, const uint8_t* sk32, const g2a* hm, g2* out) {
    const size_t i = HB_TID >> 1; if (i >= n) return;
    uint32_t k[8]; load_words(k, sk32 + 32 * i, 8);
    const g2a h = hm[0];
    jac<fp2h> H, R; fp2h_pack(H.x, h.x); fp2h_pack(H.y, h.y); fp2_one(H.z);
    pt_mul(R, H, k, 8);
    g2 r; fp2h_unpack(r.x, R.x); fp2h_unpack(r.y, R.y); fp2h_unpack(r.z, R.z);
    if ((threadIdx.x & 1) == 0) out[i] = r;
}
__global__ void k_vt_sign_hm_gls_pair(size_t n, const uint64_t* digits, const g2a* hm, g2* out) {
    const size_t i = HB_TID >> 1; if (i >= n) return;
    const uint64_t d0 = digits[4 * i], d1 = digits[4 * i + 1], d2 = digits[4 * i + 2], d3 = digits[4 * i + 3];
    const g2a h = hm[0];
    jac<fp2h> T[16], R;
    pt_set_inf(T[0]);
    fp2h_pack(T[1].x, h.x); fp2h_pack(T[1].y, h.y); fp2_one(T[1].z);
    g2_psi(T[2], T[1]); pt_neg(T[2], T[2]);
    g2_psi2(T[4], T[1]);
    g2_psi(T[8], T[4]); pt_neg(T[8], T[8]);
    for (int m = 3; m < 16; m++) if (m & (m - 1)) pt_add(T[m], T[m & (m - 1)], T[m & -m]);
    pt_set_inf(R);
    for (int b = 63; b >= 0; b--) {
        pt_dbl(R, R);
        const int m = (int)((d0 >> b) & 1) | (int)((d1 >> b) & 1) << 1 | (int)((d2 >> b) & 1) << 2 | (int)((d3 >> b) & 1) << 3;
        if (m) pt_add(R, R, T[m]);
    }
    g2 r; fp2h_unpack(r.x, R.x); fp2h_unpack(r.y, R.y); fp2h_unpack(r.z, R.z);
    if ((threadIdx.x & 1) == 0) out[i] = r;
}

namespace {
template <class T> T* dalloc(size_t n) { T* d = nullptr; cudaMalloc(&d, (n ? n : 1) * sizeof(T)); cudaMemset(d, 0, (n ? n : 1) * sizeof(T)); return d; }
template <class T> T* up(const void* h, size_t n) { T* d = dalloc<T>(n); cudaMemcpy(d, h, n * sizeof(T), cudaMemcpyHostToDevice); return d; }
int status() { return cudaDeviceSynchronize() == cudaSuccess && cudaGetLastError() == cudaSuccess ? 0 : -1; }
unsigned grid(size_t threads) { return (unsigned)((threads + 31) / 32); }
// H(m) of one message (public; every item signs it)
g2a* hash_one(const uint8_t* msg, uint32_t len, uint8_t** okh) {
    uint8_t* dm = up<uint8_t>(msg, len ? len : 1); g2a* hm = dalloc<g2a>(1); *okh = dalloc<uint8_t>(1);
    k_hash_to_g2<<<1, 32>>>(1, dm, len, hm, *okh);
    cudaFree(dm);
    return hm;
}
}  // namespace

// Runs kernel (0 k_g1_mul_gen, 1 k_sign_hash, 2 k_sign_hm_pair, 3 k_sign_hm_gls_pair) over n items in CTAs of 32 threads (the Part-1
// geometry of hbls.cu): keys sk32 (n x 32 bytes; kernel 3: digits, n x 4 u64), every item on message msg.  out: the serialized results
// (48 or 96 bytes each); ok: the kernels' flags; rec: one CtRec per thread (probe builds).  Returns 0, or -1 on a CUDA error.
extern "C" int ct_run(int kernel, size_t n, const uint8_t* sk32, const uint64_t* digits, const uint8_t* msg, uint32_t len,
                      uint8_t* out, uint8_t* ok, CtRec* rec) {
    const bool pair = kernel >= 2;
    const size_t threads = pair ? 2 * n : n;
    CtRec* drec = dalloc<CtRec>(grid(threads) * 32);
    cudaMemcpyToSymbol(ct_rec, &drec, sizeof drec);
    uint8_t* dsk = up<uint8_t>(sk32, 32 * n); uint64_t* ddig = kernel == 3 ? up<uint64_t>(digits, 4 * n) : nullptr;
    uint8_t* dm = up<uint8_t>(msg, (size_t)len * n + 1);
    uint8_t* dok = dalloc<uint8_t>(n); uint8_t* dser = dalloc<uint8_t>(96 * n);
    uint8_t* okh = nullptr; g2a* hm = pair ? hash_one(msg, len, &okh) : nullptr;
    if (kernel == 0) {
        g1* p = dalloc<g1>(n);
        k_g1_mul_gen<<<grid(threads), 32>>>(n, dsk, p);
        k_g1_serialize<<<grid(n), 32>>>(n, p, dser);
        cudaMemset(dok, 1, n);
        cudaFree(p);
    } else {
        std::vector<uint8_t> msgs((size_t)len * n + 1);
        for (size_t i = 0; i < n; i++) std::memcpy(&msgs[(size_t)len * i], msg, len);
        cudaMemcpy(dm, msgs.data(), (size_t)len * n, cudaMemcpyHostToDevice);
        g2* p = dalloc<g2>(n);
        if (kernel == 1) k_sign_hash<<<grid(threads), 32>>>(n, dsk, dm, len, p, dok);
        else if (kernel == 2) k_sign_hm_pair<<<grid(threads), 32>>>(n, dsk, hm, okh, 0, p, dok);
        else k_sign_hm_gls_pair<<<grid(threads), 32>>>(n, ddig, hm, okh, 0, p, dok);
        k_g2_serialize<<<grid(n), 32>>>(n, p, dser);
        cudaFree(p);
    }
    int rc = status();
    cudaMemcpy(out, dser, (kernel == 0 ? 48 : 96) * n, cudaMemcpyDeviceToHost);
    cudaMemcpy(ok, dok, n, cudaMemcpyDeviceToHost);
    if (rec) cudaMemcpy(rec, drec, threads * sizeof(CtRec), cudaMemcpyDeviceToHost);
    for (void* q : {(void*)drec, (void*)dsk, (void*)ddig, (void*)dm, (void*)dok, (void*)dser, (void*)okh, (void*)hm}) if (q) cudaFree(q);
    return rc ? rc : status();
}

// CUDA-event time (ms per launch, mean over reps after one warm-up launch) of one ladder kernel over n items in CTAs of 32 threads:
// which = 0 / 1 G1 generator (variable-time / constant-time), 2 / 3 the 256-bit G2 ladder on lane pairs, 4 / 5 the psi ladder on lane
// pairs.  sk32: n keys; digits: their base-|z| digits (n x 4 u64).  Returns 0, or -1 on a CUDA error.
extern "C" int ct_time(int which, size_t n, const uint8_t* sk32, const uint64_t* digits, const uint8_t* msg, uint32_t len, int reps, float* ms) {
    uint8_t* dsk = up<uint8_t>(sk32, 32 * n); uint64_t* ddig = up<uint64_t>(digits, 4 * n);
    uint8_t* okh = nullptr; g2a* hm = hash_one(msg, len, &okh);
    g1* p1 = dalloc<g1>(n); g2* p2 = dalloc<g2>(n); uint8_t* dok = dalloc<uint8_t>(n);
    auto launch = [&] {
        switch (which) {
        case 0: k_vt_g1_mul_gen<<<grid(n), 32>>>(n, dsk, p1); break;
        case 1: k_g1_mul_gen<<<grid(n), 32>>>(n, dsk, p1); break;
        case 2: k_vt_sign_hm_pair<<<grid(2 * n), 32>>>(n, dsk, hm, p2); break;
        case 3: k_sign_hm_pair<<<grid(2 * n), 32>>>(n, dsk, hm, okh, 0, p2, dok); break;
        case 4: k_vt_sign_hm_gls_pair<<<grid(2 * n), 32>>>(n, ddig, hm, p2); break;
        default: k_sign_hm_gls_pair<<<grid(2 * n), 32>>>(n, ddig, hm, okh, 0, p2, dok); break;
        }
    };
    cudaEvent_t e0, e1; cudaEventCreate(&e0); cudaEventCreate(&e1);
    launch();
    cudaEventRecord(e0);
    for (int r = 0; r < reps; r++) launch();
    cudaEventRecord(e1); cudaEventSynchronize(e1);
    float t = 0; cudaEventElapsedTime(&t, e0, e1); *ms = t / (reps > 0 ? reps : 1);
    cudaEventDestroy(e0); cudaEventDestroy(e1);
    for (void* q : {(void*)dsk, (void*)ddig, (void*)okh, (void*)hm, (void*)p1, (void*)p2, (void*)dok}) cudaFree(q);
    return status();
}
