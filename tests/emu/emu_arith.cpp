// tests/emu/emu_arith.cpp -- TEST HARNESS ONLY: the op table of tests/arith/arith_ops.cuh under HB_HOST_EMU (software carry
// flags): thread ops one item after the other, lane-pair ops on two host threads (a shuffle is a rendezvous, as in
// emu_kernels.cpp), step-machine ops lane by lane on one slot array.  Same entry points as tests/arith/arith_driver.cu.
#define HB_HOST_EMU 1
#include <cstdint>
#include <cstddef>
#include <thread>
#include <vector>
struct hb_dim3 { unsigned x, y, z; };
static thread_local hb_dim3 threadIdx = {0, 0, 0}, blockIdx = {0, 0, 0}, blockDim = {1, 1, 1}, gridDim = {1, 1, 1};
#define __global__
#define __shared__ static
#define __restrict__
#define __launch_bounds__(...)
struct uint4 { unsigned x, y, z, w; };
static inline void __syncwarp() {}
static inline unsigned __funnelshift_l(unsigned lo, unsigned hi, unsigned sh) { sh &= 31; return sh ? (hi << sh) | (lo >> (32 - sh)) : hi; }
static inline unsigned __ballot_sync(unsigned, bool p) { return p ? 1u : 0u; }
#include "../arith/arith_ops.cuh"
using namespace ar;

namespace {
template <int OP, int A> int go(size_t n, const uint32_t* in, uint32_t* out) {
    if constexpr (!((AR_FORMS[OP] >> A) & 1)) return -2;
    else {
        constexpr int C = AR_CARRIER[OP], IW = AR_IN[OP], OW = AR_OUT[OP];
        if constexpr (C == C_THR) {
            for (size_t i = 0; i < n; i++) ar_item<OP, A>(in + i * IW, out + i * OW);
        } else if constexpr (C == C_PAIR) {
            hb_emu_pair_reset();
            auto lane = [&](int role) {
                hb_emu.role = role; hb_emu.seq = 0;
                for (size_t i = 0; i < n; i++) ar_item<OP, A>(in + i * IW, out + i * OW);
                hb_emu.role = 0;
            };
            std::thread th(lane, 1); lane(0); th.join();
        } else {
            std::vector<uint32_t> slots((VM_ITEM_SLOTS + 1) * VM_SLOT_WORDS, 0);
            for (size_t i = 0; i < n; i++) {
                for (int im = 0; im < 2; im++) ar_vm_load(OP, slots.data(), 0, in + i * IW, im);
                for (int im = 0; im < 2; im++) ar_vm_exec<OP, A>(slots.data(), 0, VM_ITEM_SLOTS, in + i * IW, im);
                for (int im = 0; im < 2; im++) ar_vm_store(slots.data(), 0, out + i * OW, im);
            }
        }
        return 0;
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

extern "C" int ar_run(int op, int alias, size_t n, const uint32_t* in, uint32_t* out) { return dispatch<0>(op, alias, n, in, out); }
extern "C" int ar_op_count() { return AR_NOPS; }
extern "C" const char* ar_op_name(int i) { return i >= 0 && i < AR_NOPS ? AR_NAME[i] : nullptr; }
extern "C" void ar_op_info(int i, int* v) { v[0] = AR_CARRIER[i]; v[1] = AR_FORMS[i]; v[2] = AR_IN[i]; v[3] = AR_OUT[i]; }
