// tests/arith/arith_driver.cu -- TEST HARNESS ONLY (compiled by tests/test_arith_primitives.py with build.py's NVCC_FLAGS): the
// op table of arith_ops.cuh on the device, one kernel per (op, aliasing form).  Thread ops run in 64-thread CTAs, lane-pair ops in
// the 512-thread CTAs of the pair kernels (they may reach CTA barriers, so items are padded to whole CTAs and no thread returns
// early), step-machine ops on one warp with its slots in shared memory.
#include <cuda_runtime.h>
#include <vector>
#include "arith_ops.cuh"
using namespace ar;

namespace {
template <int OP, int A> __global__ void __launch_bounds__(512) k_item(const uint32_t* in, uint32_t* out) {
    constexpr int IW = AR_IN[OP], OW = AR_OUT[OP], C = AR_CARRIER[OP];
    const size_t t = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
    const size_t i = C == C_PAIR ? t >> 1 : t;
    ar_item<OP, A>(in + i * IW, out + i * OW);
}
template <int OP, int A> __global__ void __launch_bounds__(32) k_vm(const uint32_t* in, uint32_t* out) {
    __shared__ uint32_t slots[(16 * VM_ITEM_SLOTS + 1) * VM_SLOT_WORDS];
    constexpr int IW = AR_IN[OP], OW = AR_OUT[OP];
    const int lane = threadIdx.x, pair = lane >> 1, im = lane & 1;
    const int base = pair * VM_ITEM_SLOTS, zero = 16 * VM_ITEM_SLOTS;
    const size_t i = blockIdx.x * (size_t)16 + pair;
    const uint32_t z[12] = {0};
    if (lane < 2) vm_st(slots, zero, im, z);
    ar_vm_load(OP, slots, base, in + i * IW, im);
    __syncwarp();
    ar_vm_exec<OP, A>(slots, base, zero, in + i * IW, im);
    __syncwarp();
    ar_vm_store(slots, base, out + i * OW, im);
}

template <int OP, int A> int go(size_t n, const uint32_t* in, uint32_t* out) {
    if constexpr (!((AR_FORMS[OP] >> A) & 1)) return -2;
    else {
        constexpr int C = AR_CARRIER[OP], IW = AR_IN[OP], OW = AR_OUT[OP];
        const size_t per = C == C_THR ? 64 : (C == C_PAIR ? 256 : 16);      // items per CTA
        const size_t np = (n + per - 1) / per * per;
        // padding items repeat item 0 (valid operands for every op)
        std::vector<uint32_t> hin(np * IW + 1);
        for (size_t k = 0; k < np; k++)
            for (int j = 0; j < IW; j++) hin[k * IW + j] = in[(k < n ? k : 0) * IW + j];
        uint32_t *din = nullptr, *dout = nullptr;
        if (cudaMalloc(&din, hin.size() * 4) != cudaSuccess || cudaMalloc(&dout, np * OW * 4) != cudaSuccess) return -1;
        cudaMemcpy(din, hin.data(), hin.size() * 4, cudaMemcpyHostToDevice);
        cudaMemset(dout, 0xee, np * OW * 4);
        if (C == C_VM) k_vm<OP, A><<<(unsigned)(np / 16), 32>>>(din, dout);
        else k_item<OP, A><<<(unsigned)(np / per), C == C_THR ? 64 : 512>>>(din, dout);
        const bool ok = cudaDeviceSynchronize() == cudaSuccess && cudaGetLastError() == cudaSuccess &&
                        cudaMemcpy(out, dout, n * OW * 4, cudaMemcpyDeviceToHost) == cudaSuccess;
        cudaFree(din); cudaFree(dout);
        return ok ? 0 : -1;
    }
}
template <int OP> int run_op(int a, size_t n, const uint32_t* in, uint32_t* out) {
    switch (a) {
    case 0: return go<OP, 0>(n, in, out);
    case 1: return go<OP, 1>(n, in, out);
    case 2: return go<OP, 2>(n, in, out);
    case 3: return go<OP, 3>(n, in, out);
    case 4: return go<OP, 4>(n, in, out);
    }
    return -2;
}
template <int I> int dispatch(int op, int a, size_t n, const uint32_t* in, uint32_t* out) {
    if constexpr (I == AR_NOPS) return -2;
    else return op == I ? run_op<I>(a, n, in, out) : dispatch<I + 1>(op, a, n, in, out);
}
}  // namespace

// 0, -1 on a CUDA error, -2 for an unknown op or an aliasing form the op does not have
extern "C" int ar_run(int op, int alias, size_t n, const uint32_t* in, uint32_t* out) { return dispatch<0>(op, alias, n, in, out); }
extern "C" int ar_op_count() { return AR_NOPS; }
extern "C" const char* ar_op_name(int i) { return i >= 0 && i < AR_NOPS ? AR_NAME[i] : nullptr; }
// carrier, alias-form mask, input words, output words of one item
extern "C" void ar_op_info(int i, int* v) { v[0] = AR_CARRIER[i]; v[1] = AR_FORMS[i]; v[2] = AR_IN[i]; v[3] = AR_OUT[i]; }
