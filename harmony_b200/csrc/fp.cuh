// harmony_b200/csrc/fp.cuh -- BLS12-381 base field on sm_90a: 12 x 32-bit limbs, Montgomery form (R = 2^384).
//
// Replaces the Fp layer of libmcl that Harmony links through github.com/harmony-one/bls (reference go.mod:27,
// Makefile:68-70).  One thread owns one field element; every 32x32+64->64 multiply-accumulate is a single
// IMAD.WIDE.U32(.X) (ptxas fuses the mad.lo.cc / madc.hi.cc pairs below and keeps carries in predicates), so a
// Montgomery product costs 288 wide MACs + 12 IMAD.LO for the quotient digits.
//
// Multiplication layout: two accumulators X (64-bit lanes at even limb positions) and Y (lanes at odd positions)
// so that no lane ever straddles an aligned register pair; the modulus is folded in two quotient digits (64 bits)
// per round, and the half-lane of Y that falls off the window is rippled into X once per round.
#pragma once
#include <stdint.h>

// HB_HOST_EMU: tests/emu compiles these headers with g++ and software carry flags so that the device LOGIC can be
// checked against the oracle on the CPU-only build box (test harness only -- never part of libhbls.so).
#ifdef HB_HOST_EMU
#define __device__
#define __forceinline__ inline
#define __noinline__
#define __constant__
#endif

#define HB_DEV __device__ __forceinline__
#define HB_NOINLINE __device__ __noinline__
// code-size knobs (the pairing kernels are instruction-fetch sensitive): outline the cheap field ops
#ifndef HB_OUTLINE_FP
#define HB_OUTLINE_FP 0
#endif
// CTA-wide re-alignment points inside the uniform ladders / exponentiation loops of the thread-per-item kernels: with one
// large CTA per SM all of its warps then walk the same instruction-cache lines (same idea as hb_lockstep in the pairing kernels).
// Threads that left the kernel do not block a barrier; every call site is reached by whole CTAs in the common case.
#ifndef HB_LOCKSTEP_T
#define HB_LOCKSTEP_T 0
#endif
#if HB_LOCKSTEP_T && !defined(HB_HOST_EMU)
#define HB_USYNC() __syncthreads()
#else
#define HB_USYNC() ((void)0)
#endif
#ifndef HB_OUTLINE_FP2
#define HB_OUTLINE_FP2 1
#endif
#if HB_OUTLINE_FP
#define HB_FPFN __device__ __noinline__
#else
#define HB_FPFN __device__ __forceinline__
#endif
#if HB_OUTLINE_FP2
#define HB_FP2FN __device__ __noinline__
#else
#define HB_FP2FN __device__ __forceinline__
#endif


namespace hb {

// natural (4-byte) alignment: forcing 16 bytes (128-bit local-memory moves) measured no faster, and the sm_90a build of it
// rejected valid public keys; buffers that are read with 128-bit accesses are aligned by their allocation (line_store)
struct fp { uint32_t l[12]; };

// modulus limbs as immediates (little-endian 32-bit)
#define HB_P0  0xffffaaabu
#define HB_P1  0xb9feffffu
#define HB_P2  0xb153ffffu
#define HB_P3  0x1eabfffeu
#define HB_P4  0xf6b0f624u
#define HB_P5  0x6730d2a0u
#define HB_P6  0xf38512bfu
#define HB_P7  0x64774b84u
#define HB_P8  0x434bacd7u
#define HB_P9  0x4b1ba7b6u
#define HB_P10 0x397fe69au
#define HB_P11 0x1a0111eau
#define HB_N0  0xfffcfffdu      // -p^{-1} mod 2^32

HB_DEV uint32_t p_limb(int i) {
    switch (i) {
    case 0: return HB_P0; case 1: return HB_P1; case 2: return HB_P2; case 3: return HB_P3;
    case 4: return HB_P4; case 5: return HB_P5; case 6: return HB_P6; case 7: return HB_P7;
    case 8: return HB_P8; case 9: return HB_P9; case 10: return HB_P10; default: return HB_P11;
    }
}

#ifdef HB_HOST_EMU
static thread_local uint32_t hb_cf = 0;
inline void hb_acc3(uint32_t& d, uint64_t x, uint64_t y, uint64_t z) { uint64_t t = x + y + z; d = (uint32_t)t; hb_cf = (uint32_t)(t >> 32); }
inline void mad_lo_cc(uint32_t& d, uint32_t a, uint32_t b, uint32_t c)  { hb_acc3(d, (uint32_t)((uint64_t)a * b), c, 0); }
inline void madc_lo_cc(uint32_t& d, uint32_t a, uint32_t b, uint32_t c) { hb_acc3(d, (uint32_t)((uint64_t)a * b), c, hb_cf); }
inline void madc_hi_cc(uint32_t& d, uint32_t a, uint32_t b, uint32_t c) { hb_acc3(d, (uint32_t)(((uint64_t)a * b) >> 32), c, hb_cf); }
inline void add_cc(uint32_t& d, uint32_t a, uint32_t b)  { hb_acc3(d, a, b, 0); }
inline void addc_cc(uint32_t& d, uint32_t a, uint32_t b) { hb_acc3(d, a, b, hb_cf); }
inline void addc(uint32_t& d, uint32_t a, uint32_t b)    { d = a + b + hb_cf; }
inline void hb_sub3(uint32_t& d, uint32_t a, uint32_t b, uint32_t bin) { uint64_t t = (uint64_t)a - b - bin; d = (uint32_t)t; hb_cf = (uint32_t)(t >> 63); }
inline void sub_cc(uint32_t& d, uint32_t a, uint32_t b)  { hb_sub3(d, a, b, 0); }
inline void subc_cc(uint32_t& d, uint32_t a, uint32_t b) { hb_sub3(d, a, b, hb_cf); }
inline void subc(uint32_t& d, uint32_t a, uint32_t b)    { d = a - b - hb_cf; }
#else
// ---- single-instruction PTX wrappers; CC.CF flows between consecutive volatile asm statements
HB_DEV void mad_lo_cc(uint32_t& d, uint32_t a, uint32_t b, uint32_t c)  { asm volatile("mad.lo.cc.u32 %0, %1, %2, %3;"  : "=r"(d) : "r"(a), "r"(b), "r"(c)); }
HB_DEV void madc_lo_cc(uint32_t& d, uint32_t a, uint32_t b, uint32_t c) { asm volatile("madc.lo.cc.u32 %0, %1, %2, %3;" : "=r"(d) : "r"(a), "r"(b), "r"(c)); }
HB_DEV void madc_hi_cc(uint32_t& d, uint32_t a, uint32_t b, uint32_t c) { asm volatile("madc.hi.cc.u32 %0, %1, %2, %3;" : "=r"(d) : "r"(a), "r"(b), "r"(c)); }
HB_DEV void add_cc(uint32_t& d, uint32_t a, uint32_t b)  { asm volatile("add.cc.u32 %0, %1, %2;"  : "=r"(d) : "r"(a), "r"(b)); }
HB_DEV void addc_cc(uint32_t& d, uint32_t a, uint32_t b) { asm volatile("addc.cc.u32 %0, %1, %2;" : "=r"(d) : "r"(a), "r"(b)); }
HB_DEV void addc(uint32_t& d, uint32_t a, uint32_t b)    { asm volatile("addc.u32 %0, %1, %2;"    : "=r"(d) : "r"(a), "r"(b)); }
HB_DEV void sub_cc(uint32_t& d, uint32_t a, uint32_t b)  { asm volatile("sub.cc.u32 %0, %1, %2;"  : "=r"(d) : "r"(a), "r"(b)); }
HB_DEV void subc_cc(uint32_t& d, uint32_t a, uint32_t b) { asm volatile("subc.cc.u32 %0, %1, %2;" : "=r"(d) : "r"(a), "r"(b)); }
HB_DEV void subc(uint32_t& d, uint32_t a, uint32_t b)    { asm volatile("subc.u32 %0, %1, %2;"    : "=r"(d) : "r"(a), "r"(b)); }

#endif

// acc[0..11] (six 64-bit lanes) += {a[0], a[2], ..., a[10]} * b ; carry rippled into acc[12], acc[13]
HB_DEV void lane_mad(uint32_t* acc, const uint32_t* a, uint32_t b) {
    mad_lo_cc(acc[0], a[0], b, acc[0]);
    madc_hi_cc(acc[1], a[0], b, acc[1]);
#pragma unroll
    for (int j = 2; j < 12; j += 2) {
        madc_lo_cc(acc[j], a[j], b, acc[j]);
        madc_hi_cc(acc[j + 1], a[j], b, acc[j + 1]);
    }
    // the carry ripples two limbs up: the windows accumulate several rows, and a single limb measured wrong results on the
    // device (tests/test_arith_primitives.py)
    addc_cc(acc[12], acc[12], 0);
    addc(acc[13], acc[13], 0);
}
// same with the modulus (limbs become immediates), PAR = 0 even limbs, 1 odd limbs
template <int PAR> HB_DEV void lane_mad_p(uint32_t* acc, uint32_t m) {
    mad_lo_cc(acc[0], p_limb(PAR), m, acc[0]);
    madc_hi_cc(acc[1], p_limb(PAR), m, acc[1]);
#pragma unroll
    for (int j = 2; j < 12; j += 2) {
        madc_lo_cc(acc[j], p_limb(PAR + j), m, acc[j]);
        madc_hi_cc(acc[j + 1], p_limb(PAR + j), m, acc[j + 1]);
    }
    addc_cc(acc[12], acc[12], 0);
    addc(acc[13], acc[13], 0);
}

// r = a*b/R mod p, inputs and output canonical in [0, p)
HB_DEV void fp_mul_regs(uint32_t* r, const uint32_t* a, const uint32_t* b) {
    uint32_t x[28], y[28];
#pragma unroll
    for (int i = 0; i < 28; i++) { x[i] = 0; y[i] = 0; }
#pragma unroll
    for (int k = 0; k < 6; k++) {
        const int q = 2 * k;
        const uint32_t b0 = b[q], b1 = b[q + 1];
        lane_mad(x + q, a, b0);              // a_even * b0 -> positions q + even
        lane_mad(y + q + 1, a + 1, b0);      // a_odd  * b0 -> positions q + odd
        lane_mad(y + q + 1, a, b1);          // a_even * b1 -> positions q + 1 + even
        lane_mad(x + q + 2, a + 1, b1);      // a_odd  * b1 -> positions q + 1 + odd
        const uint32_t m0 = x[q] * HB_N0;
        lane_mad_p<0>(x + q, m0);
        lane_mad_p<1>(y + q + 1, m0);
        const uint32_t m1 = (x[q + 1] + y[q + 1]) * HB_N0;
        lane_mad_p<0>(y + q + 1, m1);
        lane_mad_p<1>(x + q + 2, m1);
        // positions q, q+1 are now 0 mod 2^64: x[q] == 0, x[q+1] + y[q+1] in {0, 2^32}.  Fold that carry and the
        // orphaned upper half of Y's lowest lane (position q+2) into X, rippling to the top of the window.
        uint32_t dead;
        add_cc(dead, x[q + 1], y[q + 1]);
        addc_cc(x[q + 2], x[q + 2], y[q + 2]);
#pragma unroll
        for (int j = q + 3; j < q + 15; j++) addc_cc(x[j], x[j], 0);
        addc(x[q + 15], x[q + 15], 0);
        (void)dead;
    }
    // T / 2^384 = X[12..] + Y[13..]  (Y's position-12 half was folded above)
    add_cc(x[13], x[13], y[13]);
#pragma unroll
    for (int j = 14; j < 24; j++) addc_cc(x[j], x[j], y[j]);
    // result < 2p < 2^382: conditional subtract
    uint32_t s[12];
    sub_cc(s[0], x[12], HB_P0);
#pragma unroll
    for (int j = 1; j < 12; j++) subc_cc(s[j], x[12 + j], p_limb(j));
    uint32_t borrow;
    subc(borrow, 0, 0);
#pragma unroll
    for (int j = 0; j < 12; j++) r[j] = borrow ? x[12 + j] : s[j];
}

HB_DEV void fp_add_regs(uint32_t* r, const uint32_t* a, const uint32_t* b) {
    uint32_t t[12], s[12];
    add_cc(t[0], a[0], b[0]);
#pragma unroll
    for (int j = 1; j < 12; j++) addc_cc(t[j], a[j], b[j]);
    sub_cc(s[0], t[0], HB_P0);
#pragma unroll
    for (int j = 1; j < 12; j++) subc_cc(s[j], t[j], p_limb(j));
    uint32_t borrow;
    subc(borrow, 0, 0);
#pragma unroll
    for (int j = 0; j < 12; j++) r[j] = borrow ? t[j] : s[j];
}
HB_DEV void fp_sub_regs(uint32_t* r, const uint32_t* a, const uint32_t* b) {
    uint32_t t[12];
    sub_cc(t[0], a[0], b[0]);
#pragma unroll
    for (int j = 1; j < 12; j++) subc_cc(t[j], a[j], b[j]);
    uint32_t borrow;
    subc(borrow, 0, 0);            // 0xffffffff when a < b
    add_cc(r[0], t[0], HB_P0 & borrow);
#pragma unroll
    for (int j = 1; j < 12; j++) addc_cc(r[j], t[j], p_limb(j) & borrow);
}

// ------------------------------------------------------------------ struct-level API
HB_FPFN void fp_add(fp& r, const fp& a, const fp& b) { fp_add_regs(r.l, a.l, b.l); }
HB_FPFN void fp_sub(fp& r, const fp& a, const fp& b) { fp_sub_regs(r.l, a.l, b.l); }
HB_FPFN void fp_dbl(fp& r, const fp& a) { fp_add_regs(r.l, a.l, a.l); }
// r = a / 2 mod p: (a + (a odd ? p : 0)) >> 1.  a < p < 2^381, so the sum fits the 12 limbs; linear, hence valid on Montgomery forms.
// (replaces multiplications by the constant 1/2 in the Miller doubling step: ~40 ALU instructions instead of 300 IMAD)
HB_DEV void fp_half(fp& r, const fp& a) {
    const uint32_t m = 0u - (a.l[0] & 1u);
    uint32_t t[12];
    add_cc(t[0], a.l[0], HB_P0 & m);
#pragma unroll
    for (int j = 1; j < 11; j++) addc_cc(t[j], a.l[j], p_limb(j) & m);
    addc(t[11], a.l[11], HB_P11 & m);
#pragma unroll
    for (int j = 0; j < 11; j++) r.l[j] = (t[j] >> 1) | (t[j + 1] << 31);
    r.l[11] = t[11] >> 1;
}
HB_DEV bool fp_is_zero(const fp& a) {
    uint32_t o = 0;
#pragma unroll
    for (int j = 0; j < 12; j++) o |= a.l[j];
    return o == 0;
}
HB_DEV bool fp_eq(const fp& a, const fp& b) {
    uint32_t o = 0;
#pragma unroll
    for (int j = 0; j < 12; j++) o |= a.l[j] ^ b.l[j];
    return o == 0;
}
HB_DEV void fp_zero(fp& r) {
#pragma unroll
    for (int j = 0; j < 12; j++) r.l[j] = 0;
}
HB_FPFN void fp_neg(fp& r, const fp& a) {
    // p - a, forced to 0 when a == 0 (a is canonical, so p - a never borrows)
    uint32_t t[12], nz = 0;
#pragma unroll
    for (int j = 0; j < 12; j++) nz |= a.l[j];
    sub_cc(t[0], HB_P0, a.l[0]);
#pragma unroll
    for (int j = 1; j < 11; j++) subc_cc(t[j], p_limb(j), a.l[j]);
    subc(t[11], HB_P11, a.l[11]);
    const uint32_t m = nz ? 0xffffffffu : 0u;
#pragma unroll
    for (int j = 0; j < 12; j++) r.l[j] = t[j] & m;
}
HB_DEV void fp_set(fp& r, const uint32_t* k) {
#pragma unroll
    for (int j = 0; j < 12; j++) r.l[j] = k[j];
}
HB_DEV void fp_cmov(fp& r, const fp& a, bool c) {
#pragma unroll
    for (int j = 0; j < 12; j++) r.l[j] = c ? a.l[j] : r.l[j];
}

// out-of-line multipliers keep the instruction footprint of the pairing kernels inside the L1.5 I-cache
#ifdef HB_HOST_EMU
static thread_local uint64_t hb_emu_cnt_mul = 0, hb_emu_cnt_sqr = 0;      // executed-work counters (tests / bench bookkeeping)
#define HB_EMU_COUNT(x) (++(x))
#else
#define HB_EMU_COUNT(x) ((void)0)
#endif
#ifndef HB_KARATSUBA
#define HB_KARATSUBA 0
#endif
// The out-of-line field operations receive their operands' addresses through hb_opaque (an empty asm): the optimiser then has
// to treat every local passed to them as escaped.  Without it the sm_90a build merged locals whose addresses were still passed
// to later calls (fp2_sqrt read its operand's slot after fp_pow had written its result there) and computed wrong points.
// (DESIGN.md "Toolchain notes": compiler version and the PTX pattern.)
template <class T> HB_DEV T* hb_opaque(T* p) {
#ifndef HB_HOST_EMU
    asm("" : "+l"(p));
#endif
    return p;
}
#if HB_KARATSUBA
HB_NOINLINE void fp_mul_ool(fp& r, const fp& a, const fp& b);      // fp_wide.cuh: Karatsuba product + separate reduction
#else
HB_NOINLINE void fp_mul_ool(fp& r, const fp& a, const fp& b) {
    HB_EMU_COUNT(hb_emu_cnt_mul);
    uint32_t ra[12], rb[12], rr[12];
#pragma unroll
    for (int j = 0; j < 12; j++) { ra[j] = a.l[j]; rb[j] = b.l[j]; }
    fp_mul_regs(rr, ra, rb);
#pragma unroll
    for (int j = 0; j < 12; j++) r.l[j] = rr[j];
}
#endif
HB_DEV void fp_mul(fp& r, const fp& a, const fp& b) { fp_mul_ool(*hb_opaque(&r), *hb_opaque(&a), *hb_opaque(&b)); }
// fp_sqr lives in fp_wide.cuh (dedicated 78-product squaring + one reduction)

}  // namespace hb
