// tests/arith/arith_ops.cuh -- TEST HARNESS ONLY: one body per arithmetic primitive of csrc/ (fp.cuh, fp_wide.cuh, tower.cuh,
// curve.cuh, pairing.cuh, vm.cuh), written once and compiled both for sm_90a (arith_driver.cu) and for the host emulation
// (tests/emu/emu_arith.cpp).  tests/test_arith_primitives.py feeds every op stored limbs (12 x u32 Montgomery words per Fp, raw
// words for the 768-bit layer) and checks the outputs against big-integer arithmetic.
//
// Every op is a template instance ar_item<OP, A>: A picks the aliasing form, and the operands are LOCALS of the item function
// passed by reference -- the historical device faults came from the optimiser giving two live locals one stack slot, which
// operands in global memory could not show.  Binary forms: 0 distinct, 1 r == x, 2 r == y, 3 x == y, 4 r == x == y; unary forms:
// 0 distinct, 1 r == x.  AR_FORMS holds the forms that apply to an op as a bit mask.
//
// Carriers: 0 one item per thread; 1 one item per lane pair (fp2h: every Fp2 value split, the even lane holds the real halves);
// 2 one item per lane pair of the step machine (vm.cuh: Fp2 slots in shared memory).  Item layouts are the same for the thread
// and the pair form of an op: a value built of Fp2 elements lists them whole (real, imaginary), and a pair lane reads its half.
// A verdict takes two words: a pair's lanes write one each, a thread writes both.
#pragma once
#include <type_traits>
#include "../../harmony_b200/csrc/pairing.cuh"
#include "../../harmony_b200/csrc/vm.cuh"

namespace ar {
using namespace hb;

enum { W_F = 12, W_F2 = 24, W_F6 = 72, W_F12 = 144, W_FL = 2 };
enum { M_BIN = 0x1f, M_UN = 0x3, M_ONE = 0x1, M_XY = 0x9 };
enum { C_THR = 0, C_PAIR = 1, C_VM = 2 };

// X(name, carrier, alias forms, input words, output words)
#define AR_FIELD_OPS(X) \
    X(fp_mul, C_THR, M_BIN, 2 * W_F, W_F) X(fp_sqr, C_THR, M_UN, W_F, W_F) X(fp_add, C_THR, M_BIN, 2 * W_F, W_F) \
    X(fp_sub, C_THR, M_BIN, 2 * W_F, W_F) X(fp_dbl, C_THR, M_UN, W_F, W_F) X(fp_neg, C_THR, M_UN, W_F, W_F) \
    X(fp_half, C_THR, M_UN, W_F, W_F) X(fp_inv, C_THR, M_UN, W_F, W_F) X(fp_inv_gcd, C_THR, M_UN, W_F, W_F) \
    X(fp_sqrt, C_THR, M_UN, W_F, W_F + W_FL) X(fp_sqrt_inv, C_THR, M_UN, W_F, 2 * W_F + W_FL) \
    X(fp_legendre, C_THR, M_ONE, W_F, W_FL) X(fp_legendre_pow, C_THR, M_ONE, W_F, W_FL) \
    X(fp_from_int, C_THR, M_UN, W_F, W_F) X(fp_to_int, C_THR, M_UN, W_F, W_F) X(fp_int_geq_p, C_THR, M_ONE, W_F, W_FL) \
    X(mul_wide, C_THR, M_XY, 2 * W_F, 2 * W_F) X(mul_wide_k, C_THR, M_XY, 2 * W_F, 2 * W_F) \
    X(mul_wide2, C_THR, M_XY, 4 * W_F, 2 * W_F) X(sqr_wide, C_THR, M_ONE, W_F, 2 * W_F) X(redc_wide, C_THR, M_ONE, 2 * W_F, W_F) \
    X(fp2_mul_regs, C_THR, M_BIN, 2 * W_F2, W_F2) X(fp2_mul_regs_cios, C_THR, M_BIN, 2 * W_F2, W_F2) \
    X(fp2_sqr_regs, C_THR, M_UN, W_F2, W_F2) X(fp2_sqr_regs_cios, C_THR, M_UN, W_F2, W_F2) \
    X(fp2_sqrt, C_THR, M_UN, W_F2, W_F2 + W_FL) X(fp2_sqrt_anysign, C_THR, M_UN, W_F2, W_F2 + W_FL) \
    X(fp2_norm, C_THR, M_ONE, W_F2, W_F)

// the Fp2-and-above ops exist on both carriers: fp2_* on one thread, fp2h_* on a lane pair
#define AR_TOWER_OPS(X, P, C) \
    X(P##_mul, C, M_BIN, 2 * W_F2, W_F2) X(P##_sqr, C, M_UN, W_F2, W_F2) X(P##_add, C, M_BIN, 2 * W_F2, W_F2) \
    X(P##_sub, C, M_BIN, 2 * W_F2, W_F2) X(P##_neg, C, M_UN, W_F2, W_F2) X(P##_dbl, C, M_UN, W_F2, W_F2) \
    X(P##_inv, C, M_UN, W_F2, W_F2) X(P##_inv_gcd, C, M_UN, W_F2, W_F2) X(P##_mul_xi, C, M_UN, W_F2, W_F2) \
    X(P##_conj, C, M_UN, W_F2, W_F2) X(P##_mul_fp, C, M_UN, W_F2 + W_F, W_F2) X(P##_half, C, M_UN, W_F2, W_F2) \
    X(P##_mul_twist3b, C, M_UN, W_F2, W_F2) X(P##_is_zero, C, M_ONE, W_F2, W_FL) X(P##_eq, C, M_XY, 2 * W_F2, W_FL) \
    X(P##_one, C, M_ONE, 0, W_F2) X(P##_const, C, M_ONE, 0, W_F2) \
    X(P##_fp6_mul, C, M_BIN, 2 * W_F6, W_F6) X(P##_fp6_inv, C, M_UN, W_F6, W_F6) \
    X(P##_fp6_mul_by_01, C, M_UN, W_F6 + 2 * W_F2, W_F6) X(P##_fp6_mul_by_1, C, M_UN, W_F6 + W_F2, W_F6) \
    X(P##_fp6_mul_by_12, C, M_UN, W_F6 + 2 * W_F2, W_F6) \
    X(P##_fp12_mul, C, M_BIN, 2 * W_F12, W_F12) X(P##_fp12_sqr, C, M_UN, W_F12, W_F12) X(P##_fp12_inv, C, M_UN, W_F12, W_F12) \
    X(P##_fp12_conj, C, M_UN, W_F12, W_F12) X(P##_fp12_mul_by_014, C, M_UN, W_F12 + 3 * W_F2, W_F12) \
    X(P##_fp12_mul_by_two_lines, C, M_UN, W_F12 + 6 * W_F2, W_F12) X(P##_fp12_frob, C, M_UN, W_F12, W_F12) \
    X(P##_fp12_frob2, C, M_UN, W_F12, W_F12) X(P##_fp12_is_one, C, M_ONE, W_F12, W_FL) \
    X(P##_fp12_cyc_sqr, C, M_UN, W_F12, W_F12) X(P##_fp12_cyc_exp_z, C, M_UN, W_F12, W_F12) \
    X(P##_final_exp, C, M_UN, W_F12, W_F12)

// the group law on G1 (g1_), G2 over fp2 (g2_) and G2 over the lane pair (g2h_); W = words of one coordinate
#define AR_GROUP_OPS(X, P, C, W) \
    X(P##_pt_dbl, C, M_UN, 3 * W, 3 * W) X(P##_pt_add, C, M_BIN, 6 * W, 3 * W) X(P##_pt_add_mixed, C, M_UN, 5 * W, 3 * W) \
    X(P##_pt_eq, C, M_XY, 6 * W, W_FL) X(P##_pt_to_aff, C, M_ONE, 3 * W, 2 * W) X(P##_pt_to_aff_zinv, C, M_ONE, 4 * W, 2 * W) \
    X(P##_batch_inv, C, M_ONE, 4 * W + 4, 4 * W)

// the step machine's three instruction classes: slot values, then (vm_lin) the two lanes' atom rows and the atom count
#define AR_VM_OPS(X) \
    X(vm_mul, C_VM, M_XY, 2 * W_F2, W_F2) X(vm_sqr, C_VM, M_ONE, W_F2, W_F2) X(vm_lin, C_VM, M_ONE, 8 * W_F2 + 9, W_F2)

#define AR_OPS(X) AR_FIELD_OPS(X) AR_TOWER_OPS(X, fp2, C_THR) AR_TOWER_OPS(X, fp2h, C_PAIR) \
    AR_GROUP_OPS(X, g1, C_THR, W_F) AR_GROUP_OPS(X, g2, C_THR, W_F2) AR_GROUP_OPS(X, g2h, C_PAIR, W_F2) AR_VM_OPS(X)

#define AR_ENUM(n, c, m, i, o) OP_##n,
enum { AR_OPS(AR_ENUM) AR_NOPS };
#define AR_CARRIER_OF(n, c, m, i, o) c,
#define AR_FORMS_OF(n, c, m, i, o) m,
#define AR_IN_OF(n, c, m, i, o) i,
#define AR_OUT_OF(n, c, m, i, o) o,
#define AR_NAME_OF(n, c, m, i, o) #n,
constexpr int AR_CARRIER[] = {AR_OPS(AR_CARRIER_OF)};
constexpr int AR_FORMS[] = {AR_OPS(AR_FORMS_OF)};
constexpr int AR_IN[] = {AR_OPS(AR_IN_OF)};
constexpr int AR_OUT[] = {AR_OPS(AR_OUT_OF)};
static const char* const AR_NAME[] = {AR_OPS(AR_NAME_OF)};

// ------------------------------------------------------------------ loads / stores between the item layout and kernel locals
struct w4 { uint32_t l[4]; };
struct w24 { uint32_t l[24]; };
typedef fp6_t<fp2h> fp6h; typedef fp12_t<fp2h> fp12h;
template <class T> struct split { static constexpr bool v = false; };          // built of lane-pair halves?
template <> struct split<fp2h> { static constexpr bool v = true; };
template <> struct split<fp6h> { static constexpr bool v = true; };
template <> struct split<fp12h> { static constexpr bool v = true; };
template <> struct split<jac<fp2h>> { static constexpr bool v = true; };
template <> struct split<aff<fp2h>> { static constexpr bool v = true; };

template <class T> HB_DEV void ld(T& v, const uint32_t* in, int& o) {
    uint32_t* w = reinterpret_cast<uint32_t*>(&v);
    if constexpr (split<T>::v) {               // this lane's half of every Fp2 element
        const int r = fp2h_role();
        for (int k = 0; k < (int)(sizeof(T) / 48); k++)
            for (int j = 0; j < 12; j++) w[12 * k + j] = in[o + 24 * k + 12 * r + j];
        o += (int)(sizeof(T) / 2);
    } else {
        for (int j = 0; j < (int)(sizeof(T) / 4); j++) w[j] = in[o + j];
        o += (int)(sizeof(T) / 4);
    }
}
template <class T> HB_DEV void st(uint32_t* out, int& o, const T& v) {
    const uint32_t* w = reinterpret_cast<const uint32_t*>(&v);
    if constexpr (split<T>::v) {
        const int r = fp2h_role();
        for (int k = 0; k < (int)(sizeof(T) / 48); k++)
            for (int j = 0; j < 12; j++) out[o + 24 * k + 12 * r + j] = w[12 * k + j];
        o += (int)(sizeof(T) / 2);
    } else {
        for (int j = 0; j < (int)(sizeof(T) / 4); j++) out[o + j] = w[j];
        o += (int)(sizeof(T) / 4);
    }
}
template <int C> HB_DEV void st_flag(uint32_t* out, int& o, uint32_t f) {
    if (C == C_PAIR) out[o + fp2h_role()] = f;
    else { out[o] = f; out[o + 1] = f; }
    o += W_FL;
}

// ------------------------------------------------------------------ aliasing forms over kernel locals
template <int A, class T, class F> HB_DEV void bin(T& r, T& x, T& y, F f) {
    if constexpr (A == 0) f(r, x, y);
    else if constexpr (A == 1) { f(x, x, y); r = x; }
    else if constexpr (A == 2) { f(y, x, y); r = y; }
    else if constexpr (A == 3) f(r, x, x);
    else { f(x, x, x); r = x; }
}
template <int A, class T, class F> HB_DEV void un(T& r, T& x, F f) {
    if constexpr (A == 0) f(r, x);
    else { f(x, x); r = x; }
}

#define AR_BIN(N, T, BODY) if constexpr (OP == OP_##N) { \
    T x, y, r; int i = 0, o = 0; ld(x, in, i); ld(y, in, i); \
    bin<A>(r, x, y, [](T& r, const T& x, const T& y) { BODY; }); st(out, o, r); }
#define AR_UN(N, T, BODY) if constexpr (OP == OP_##N) { \
    T x, r; int i = 0, o = 0; ld(x, in, i); un<A>(r, x, [](T& r, const T& x) { BODY; }); st(out, o, r); }
#define AR_PRED(N, T, EXPR) if constexpr (OP == OP_##N) { \
    T x; int i = 0, o = 0; ld(x, in, i); st_flag<AR_CARRIER[OP]>(out, o, (uint32_t)(EXPR)); }

// ---- the Fp2-and-above ops, generic over the carrier E (fp2 / fp2h); ID = OP_<P>_<op> for this carrier
template <int OP, int A, class E, int B> HB_DEV void ar_tower(const uint32_t* in, uint32_t* out) {
    typedef fp6_t<E> F6; typedef fp12_t<E> F12;
#define T_OP(n) (B + (OP_fp2_##n - OP_fp2_mul))
#define T_BIN(n, T, BODY) if constexpr (OP == T_OP(n)) { \
    T x, y, r; int i = 0, o = 0; ld(x, in, i); ld(y, in, i); bin<A>(r, x, y, [](T& r, const T& x, const T& y) { BODY; }); st(out, o, r); }
#define T_UN(n, T, BODY) if constexpr (OP == T_OP(n)) { \
    T x, r; int i = 0, o = 0; ld(x, in, i); un<A>(r, x, [](T& r, const T& x) { BODY; }); st(out, o, r); }
#define T_UN_K(n, T, K, NK, CALL) if constexpr (OP == T_OP(n)) { \
    T x, r; K k[NK]; int i = 0, o = 0; ld(x, in, i); for (int j = 0; j < NK; j++) ld(k[j], in, i); \
    if constexpr (A == 0) { CALL(r, x); } else { CALL(x, x); r = x; } st(out, o, r); }
    T_BIN(mul, E, fp2_mul(r, x, y))
    T_UN(sqr, E, fp2_sqr(r, x))
    T_BIN(add, E, fp2_add(r, x, y))
    T_BIN(sub, E, fp2_sub(r, x, y))
    T_UN(neg, E, fp2_neg(r, x))
    T_UN(dbl, E, fp2_dbl(r, x))
    T_UN(inv, E, fp2_inv(r, x))
    T_UN(inv_gcd, E, fp2_inv_gcd(r, x))
    T_UN(mul_xi, E, fp2_mul_xi(r, x))
    T_UN(conj, E, fp2_conj(r, x))
#define C_MULFP(R, X) fp2_mul_fp(R, X, k[0])
    T_UN_K(mul_fp, E, fp, 1, C_MULFP)
    T_UN(half, E, fp2_half(r, x))
    T_UN(mul_twist3b, E, fp2_mul_twist3b(r, x))
    if constexpr (OP == T_OP(is_zero)) { E x; int i = 0, o = 0; ld(x, in, i); st_flag<AR_CARRIER[OP]>(out, o, fp2_is_zero(x) ? 1u : 0u); }
    if constexpr (OP == T_OP(eq)) {
        E x, y; int i = 0, o = 0; ld(x, in, i); ld(y, in, i);
        bool v; if constexpr (A == 0) v = fp2_eq(x, y); else v = fp2_eq(x, x);
        st_flag<AR_CARRIER[OP]>(out, o, v ? 1u : 0u);
    }
    if constexpr (OP == T_OP(one)) { E r; int o = 0; fp2_one(r); st(out, o, r); }
    if constexpr (OP == T_OP(const)) { E r; int o = 0; fp2_const(r, K_FROB1[1]); st(out, o, r); }
    T_BIN(fp6_mul, F6, fp6_mul(r, x, y))
    T_UN(fp6_inv, F6, fp6_inv(r, x))
#define C_BY01(R, X) fp6_mul_by_01(R, X, k[0], k[1])
#define C_BY1(R, X) fp6_mul_by_1(R, X, k[0])
#define C_BY12(R, X) fp6_mul_by_12(R, X, k[0], k[1])
    T_UN_K(fp6_mul_by_01, F6, E, 2, C_BY01)
    T_UN_K(fp6_mul_by_1, F6, E, 1, C_BY1)
    T_UN_K(fp6_mul_by_12, F6, E, 2, C_BY12)
    T_BIN(fp12_mul, F12, fp12_mul(r, x, y))
    T_UN(fp12_sqr, F12, fp12_sqr(r, x))
    T_UN(fp12_inv, F12, fp12_inv(r, x))
    T_UN(fp12_conj, F12, fp12_conj(r, x))
#define C_BY014(R, X) fp12_mul_by_014(R, X, k[0], k[1], k[2])
#define C_BY2L(R, X) fp12_mul_by_two_lines(R, X, k[0], k[1], k[2], k[3], k[4], k[5])
    T_UN_K(fp12_mul_by_014, F12, E, 3, C_BY014)
    T_UN_K(fp12_mul_by_two_lines, F12, E, 6, C_BY2L)
    T_UN(fp12_frob, F12, fp12_frob(r, x))
    T_UN(fp12_frob2, F12, fp12_frob2(r, x))
    if constexpr (OP == T_OP(fp12_is_one)) { F12 x; int i = 0, o = 0; ld(x, in, i); st_flag<AR_CARRIER[OP]>(out, o, fp12_is_one(x) ? 1u : 0u); }
    T_UN(fp12_cyc_sqr, F12, fp12_cyc_sqr(r, x))
    T_UN(fp12_cyc_exp_z, F12, fp12_cyc_exp_z(r, x))
    T_UN(final_exp, F12, final_exp(r, x))
#undef T_OP
#undef T_BIN
#undef T_UN
#undef T_UN_K
}

// ---- the group law over the coordinate field F; ID = OP_<P>_pt_dbl for this field
template <int OP, int A, class F, int B> HB_DEV void ar_group(const uint32_t* in, uint32_t* out) {
    typedef jac<F> J; typedef aff<F> Af;
#define G_OP(n) (B + (OP_g1_##n - OP_g1_pt_dbl))
    if constexpr (OP == G_OP(pt_dbl)) { J x, r; int i = 0, o = 0; ld(x, in, i); un<A>(r, x, [](J& r, const J& x) { pt_dbl(r, x); }); st(out, o, r); }
    if constexpr (OP == G_OP(pt_add)) {
        J x, y, r; int i = 0, o = 0; ld(x, in, i); ld(y, in, i);
        bin<A>(r, x, y, [](J& r, const J& x, const J& y) { pt_add(r, x, y); }); st(out, o, r);
    }
    if constexpr (OP == G_OP(pt_add_mixed)) {
        J x, r; Af q; int i = 0, o = 0; ld(x, in, i); ld(q, in, i);
        if constexpr (A == 0) pt_add_mixed(r, x, q); else { pt_add_mixed(x, x, q); r = x; }
        st(out, o, r);
    }
    if constexpr (OP == G_OP(pt_eq)) {
        J x, y; int i = 0, o = 0; ld(x, in, i); ld(y, in, i);
        bool v; if constexpr (A == 0) v = pt_eq(x, y); else v = pt_eq(x, x);
        st_flag<AR_CARRIER[OP]>(out, o, v ? 1u : 0u);
    }
    if constexpr (OP == G_OP(pt_to_aff)) { J x; Af r; int i = 0, o = 0; ld(x, in, i); pt_to_aff(r, x); st(out, o, r); }
    if constexpr (OP == G_OP(pt_to_aff_zinv)) { J x; F zi; Af r; int i = 0, o = 0; ld(x, in, i); ld(zi, in, i); pt_to_aff_zinv(r, x, zi); st(out, o, r); }
    if constexpr (OP == G_OP(batch_inv)) {
        F z[4]; w4 s; bool skip[4]; int i = 0, o = 0;
        for (int k = 0; k < 4; k++) ld(z[k], in, i);
        ld(s, in, i);
        for (int k = 0; k < 4; k++) skip[k] = s.l[k] != 0;
        f_batch_inv<F, 4>(z, skip);
        for (int k = 0; k < 4; k++) st(out, o, z[k]);
    }
#undef G_OP
}

template <int OP, int A> HB_DEV void ar_item(const uint32_t* in, uint32_t* out) {
    AR_BIN(fp_mul, fp, fp_mul(r, x, y))
    AR_UN(fp_sqr, fp, fp_sqr(r, x))
    AR_BIN(fp_add, fp, fp_add(r, x, y))
    AR_BIN(fp_sub, fp, fp_sub(r, x, y))
    AR_UN(fp_dbl, fp, fp_dbl(r, x))
    AR_UN(fp_neg, fp, fp_neg(r, x))
    AR_UN(fp_half, fp, fp_half(r, x))
    AR_UN(fp_inv, fp, fp_inv(r, x))
    AR_UN(fp_inv_gcd, fp, fp_inv_gcd(r, x))
    if constexpr (OP == OP_fp_sqrt) {
        fp x, r; int i = 0, o = 0; ld(x, in, i); fp_zero(r);
        bool ok; if constexpr (A == 0) ok = fp_sqrt(r, x); else { ok = fp_sqrt(x, x); r = x; }
        st(out, o, r); st_flag<C_THR>(out, o, ok ? 1u : 0u);
    }
    if constexpr (OP == OP_fp_sqrt_inv) {
        fp x, r, u; int i = 0, o = 0; ld(x, in, i); fp_zero(r); fp_zero(u);
        bool ok; if constexpr (A == 0) ok = fp_sqrt_inv(r, u, x); else { ok = fp_sqrt_inv(x, u, x); r = x; }
        st(out, o, r); st(out, o, u); st_flag<C_THR>(out, o, ok ? 1u : 0u);
    }
    AR_PRED(fp_legendre, fp, fp_legendre(x))
    AR_PRED(fp_legendre_pow, fp, fp_legendre_pow(x))
    AR_UN(fp_from_int, fp, fp_from_int(r, x))
    AR_UN(fp_to_int, fp, fp_to_int(r, x))
    AR_PRED(fp_int_geq_p, fp, fp_int_geq_p(x) ? 1u : 0u)
    if constexpr (OP == OP_mul_wide || OP == OP_mul_wide_k) {
        fp x, y; w24 r; int i = 0, o = 0; ld(x, in, i); ld(y, in, i);
        const uint32_t* b = A == 0 ? y.l : x.l;
        if constexpr (OP == OP_mul_wide) mul_wide(r.l, x.l, b); else mul_wide_k(r.l, x.l, b);
        st(out, o, r);
    }
    if constexpr (OP == OP_mul_wide2) {
        fp a1, b1, a2, b2; w24 r; int i = 0, o = 0; ld(a1, in, i); ld(b1, in, i); ld(a2, in, i); ld(b2, in, i);
        if constexpr (A == 0) mul_wide2(r.l, a1.l, b1.l, a2.l, b2.l); else mul_wide2(r.l, a1.l, a1.l, a2.l, a2.l);
        st(out, o, r);
    }
    if constexpr (OP == OP_sqr_wide) { fp x; w24 r; int i = 0, o = 0; ld(x, in, i); sqr_wide(r.l, x.l); st(out, o, r); }
    if constexpr (OP == OP_redc_wide) { w24 t; fp r; int i = 0, o = 0; ld(t, in, i); redc_wide(r.l, t.l); st(out, o, r); }
    AR_BIN(fp2_mul_regs, fp2, fp2_mul_regs(r.a.l, r.b.l, x.a.l, x.b.l, y.a.l, y.b.l))
    AR_BIN(fp2_mul_regs_cios, fp2, fp2_mul_regs_cios(r.a.l, r.b.l, x.a.l, x.b.l, y.a.l, y.b.l))
    AR_UN(fp2_sqr_regs, fp2, fp2_sqr_regs(r.a.l, r.b.l, x.a.l, x.b.l))
    AR_UN(fp2_sqr_regs_cios, fp2, fp2_sqr_regs_cios(r.a.l, r.b.l, x.a.l, x.b.l))
    if constexpr (OP == OP_fp2_sqrt || OP == OP_fp2_sqrt_anysign) {
        fp2 x, r; int i = 0, o = 0; ld(x, in, i); fp2_zero(r);
        bool ok;
        if constexpr (OP == OP_fp2_sqrt) { if constexpr (A == 0) ok = fp2_sqrt(r, x); else { ok = fp2_sqrt(x, x); r = x; } }
        else { if constexpr (A == 0) ok = fp2_sqrt_anysign(r, x); else { ok = fp2_sqrt_anysign(x, x); r = x; } }
        st(out, o, r); st_flag<C_THR>(out, o, ok ? 1u : 0u);
    }
    if constexpr (OP == OP_fp2_norm) { fp2 x; fp r; int i = 0, o = 0; ld(x, in, i); fp2_norm(r, x); st(out, o, r); }
    if constexpr (OP >= OP_fp2_mul && OP <= OP_fp2_final_exp) ar_tower<OP, A, fp2, OP_fp2_mul>(in, out);
    if constexpr (OP >= OP_fp2h_mul && OP <= OP_fp2h_final_exp) ar_tower<OP, A, fp2h, OP_fp2h_mul>(in, out);
    if constexpr (OP >= OP_g1_pt_dbl && OP <= OP_g1_batch_inv) ar_group<OP, A, fp, OP_g1_pt_dbl>(in, out);
    if constexpr (OP >= OP_g2_pt_dbl && OP <= OP_g2_batch_inv) ar_group<OP, A, fp2, OP_g2_pt_dbl>(in, out);
    if constexpr (OP >= OP_g2h_pt_dbl && OP <= OP_g2h_batch_inv) ar_group<OP, A, fp2h, OP_g2h_pt_dbl>(in, out);
}

// ------------------------------------------------------------------ step-machine ops: one lane pair, slots base .. base + 9 and
// the shared zero slot.  Three phases separated by the caller's warp barrier: each lane stores its halves of the operands, both
// lanes run the step, each lane stores its half of the destination.
enum { VM_ITEM_SLOTS = 10 };
HB_DEV void ar_vm_load(int op, uint32_t* slots, int base, const uint32_t* in, int im) {
    const int nsrc = op == OP_vm_lin ? 8 : (op == OP_vm_mul ? 2 : 1);
    for (int s = 0; s < nsrc; s++) vm_st(slots, base + s, im, in + 24 * s + 12 * im);
}
template <int OP, int A> HB_DEV void ar_vm_exec(uint32_t* slots, int base, int zero, const uint32_t* in, int im) {
    const int dst = base + 9;
    if constexpr (OP == OP_vm_mul) vm_mul(slots, dst, base, A == 0 ? base + 1 : base, im);
    if constexpr (OP == OP_vm_sqr) vm_sqr(slots, dst, base, im);
    if constexpr (OP == OP_vm_lin) {
        // atoms name item-local slots 0..7, or 8 for the zero slot: rebase them to this pair's slots
        const uint32_t* rw = in + 8 * 24 + 4 * im;
        uint32_t w[4];
        for (int k = 0; k < 4; k++) {
            uint32_t v = 0;
            for (int h = 0; h < 2; h++) {
                const uint32_t at = (rw[k] >> (16 * h)) & 0xffffu, s = at & 0xffu;
                const uint32_t g = s == 8 ? (uint32_t)zero : (uint32_t)base + s;
                v |= ((at & 0xff00u) | g) << (16 * h);
            }
            w[k] = v;
        }
        uint4 row; row.x = w[0]; row.y = w[1]; row.z = w[2]; row.w = w[3];
        vm_lin(slots, dst, row, (int)in[8 * 24 + 8], im);
    }
}
HB_DEV void ar_vm_store(uint32_t* slots, int base, uint32_t* out, int im) { vm_ld(out + 12 * im, slots, base + 9, im); }

}  // namespace ar
