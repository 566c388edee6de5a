// harmony_b200/csrc/tower.cuh -- Fp2 = Fp[i]/(i^2+1), Fp6 = Fp2[v]/(v^3 - xi), Fp12 = Fp6[w]/(w^2 - v), xi = 1 + i.
// Replaces mcl's Fp2/Fp6/Fp12 tower used by Sign.VerifyHash (reference call sites: consensus/leader.go:173,287,
// internal/chain/engine.go:638).  Pairing values are never exposed by the reference API (only booleans), so the
// tower basis and formulas are free; results are checked as booleans against oracle/.
#pragma once
#include "fp.cuh"
#include "fp_wide.cuh"
#include "hbls_constants.cuh"

#ifdef HB_HOST_EMU
#include <atomic>
#include <thread>
#endif
namespace hb {
// per-helper outlining switches (code size vs call overhead); -DHB_OL_<NAME>=0/1, default = HB_OUTLINE_FP2
#ifndef HB_OL_ADD
#define HB_OL_ADD HB_OUTLINE_FP2
#endif
#if HB_OL_ADD
#define HB_ATTR_ADD __device__ __noinline__
#else
#define HB_ATTR_ADD __device__ __forceinline__
#endif
#ifndef HB_OL_SUB
#define HB_OL_SUB HB_OUTLINE_FP2
#endif
#if HB_OL_SUB
#define HB_ATTR_SUB __device__ __noinline__
#else
#define HB_ATTR_SUB __device__ __forceinline__
#endif
#ifndef HB_OL_NEG
#define HB_OL_NEG HB_OUTLINE_FP2
#endif
#if HB_OL_NEG
#define HB_ATTR_NEG __device__ __noinline__
#else
#define HB_ATTR_NEG __device__ __forceinline__
#endif
#ifndef HB_OL_CONJ
#define HB_OL_CONJ HB_OUTLINE_FP2
#endif
#if HB_OL_CONJ
#define HB_ATTR_CONJ __device__ __noinline__
#else
#define HB_ATTR_CONJ __device__ __forceinline__
#endif
#ifndef HB_OL_DBL
#define HB_OL_DBL HB_OUTLINE_FP2
#endif
#if HB_OL_DBL
#define HB_ATTR_DBL __device__ __noinline__
#else
#define HB_ATTR_DBL __device__ __forceinline__
#endif
#ifndef HB_OL_MULFP
#define HB_OL_MULFP HB_OUTLINE_FP2
#endif
#if HB_OL_MULFP
#define HB_ATTR_MULFP __device__ __noinline__
#else
#define HB_ATTR_MULFP __device__ __forceinline__
#endif
#ifndef HB_OL_MULXI
#define HB_OL_MULXI HB_OUTLINE_FP2
#endif
#if HB_OL_MULXI
#define HB_ATTR_MULXI __device__ __noinline__
#else
#define HB_ATTR_MULXI __device__ __forceinline__
#endif

struct fp2 { fp a, b; };

HB_DEV void fp_const(fp& r, const uint32_t* k) { fp_set(r, k); }
// Constants reach out-of-line functions by reference straight from constant memory.  A stack copy made only to be passed
// (fp c; fp_set(c, K); f(.., c)) was given the stack slot of a live local by the sm_90a build -- fp_to_int's 1 took the slot of
// the value being converted, fp2_sqrt's 1/2 that of its operand -- and silently corrupted both.
HB_DEV const fp& fp_k(const uint32_t* k) { return *reinterpret_cast<const fp*>(k); }
HB_DEV const fp2& fp2_k(const uint32_t k[2][12]) { return *reinterpret_cast<const fp2*>(k); }
static __device__ __constant__ const uint32_t K_INT_ONE[12] = {1u};      // the integer 1 (Montgomery form -> canonical)
HB_DEV void fp_one(fp& r) { fp_set(r, K_ONE); }

// ------------------------------------------------------------------ Fp exponentiation (fixed public exponents)
// r = a^e, e = 12 x u32 plain integer in constant memory; 4-bit fixed window (uniform control flow across the warp)
HB_NOINLINE void fp_pow_ool(fp& r, const fp& a, const uint32_t* e) {
    fp tbl[16];
    fp_one(tbl[0]); tbl[1] = a;
    for (int i = 2; i < 16; i++) fp_mul(tbl[i], tbl[i - 1], a);
    fp acc; fp_one(acc);
    bool started = false;
    for (int i = 95; i >= 0; i--) {
        uint32_t w = (e[i >> 3] >> (4 * (i & 7))) & 15u;
        if ((i & 3) == 3) HB_USYNC();
        if (started) { fp_sqr(acc, acc); fp_sqr(acc, acc); fp_sqr(acc, acc); fp_sqr(acc, acc); }
        if (w) { if (started) fp_mul(acc, acc, tbl[w]); else { acc = tbl[w]; started = true; } }
    }
    r = acc;
}
HB_DEV void fp_pow(fp& r, const fp& a, const uint32_t* e) { fp_pow_ool(*hb_opaque(&r), *hb_opaque(&a), e); }
HB_DEV void fp_inv(fp& r, const fp& a) { fp_pow(r, a, K_P_MINUS_2); }
// mcl Fp::squareRoot (p = 3 mod 4): candidate a^((p+1)/4), accepted iff it squares back (SURVEY A.1)
HB_DEV bool fp_sqrt(fp& r, const fp& a) {
    fp y, y2; fp_pow(y, a, K_P_PLUS_1_DIV_4); fp_sqr(y2, y);
    if (!fp_eq(y2, a)) return false;
    r = y; return true;
}
// one exponentiation for BOTH the square root and its inverse: u = a^((p-3)/4) => a*u = a^((p+1)/4) (exactly the
// candidate mcl's Fp::squareRoot produces) and, when a is a square, u = 1/sqrt(a).  false iff a is a non-residue.
HB_DEV bool fp_sqrt_inv(fp& root, fp& inv_root, const fp& a) {
    fp u, c, c2; fp_pow(u, a, K_P_MINUS_3_DIV_4); fp_mul(c, u, a); fp_sqr(c2, c);
    if (!fp_eq(c2, a)) return false;
    root = c; inv_root = u; return true;
}
HB_DEV int fp_legendre_pow(const fp& a) {
    if (fp_is_zero(a)) return 0;
    fp t, one; fp_pow(t, a, K_P_MINUS_1_DIV_2); fp_one(one);
    return fp_eq(t, one) ? 1 : -1;
}
// Legendre symbol as a binary Jacobi symbol: ~540 shift/subtract steps on 12 limbs (no multiplications), about a fifth
// of the instructions of the a^((p-1)/2) exponentiation.  The Montgomery factor R = (2^192)^2 is a square, so the
// symbol of the stored value a R mod p is the symbol of a.  Each step is branch-free (selects), only the trip count
// depends on the data.
HB_NOINLINE int fp_legendre(const fp& x) {
    uint32_t a[12], n[12], d[12], e[12];
    uint32_t nz = 0;
#pragma unroll
    for (int j = 0; j < 12; j++) { a[j] = x.l[j]; n[j] = p_limb(j); nz |= a[j]; }
    if (!nz) return 0;
    uint32_t t = 0;
    for (int it = 0; it < 800 && nz; it++) {
        const uint32_t odd = 0u - (a[0] & 1u);                       // all-ones when a is odd
        uint32_t bw;
        sub_cc(d[0], a[0], n[0]);
#pragma unroll
        for (int j = 1; j < 12; j++) subc_cc(d[j], a[j], n[j]);
        subc(bw, 0, 0);                                              // all-ones when a < n
        sub_cc(e[0], n[0], a[0]);
#pragma unroll
        for (int j = 1; j < 11; j++) subc_cc(e[j], n[j], a[j]);
        subc(e[11], n[11], a[11]);
        const uint32_t swp = odd & bw;                               // odd and a < n: (a, n) <- (n - a, a)
        t ^= swp & (((a[0] & n[0] & 3u) == 3u) ? 1u : 0u);
        const uint32_t keep = ~odd;                                  // even: a unchanged
        nz = 0;
#pragma unroll
        for (int j = 0; j < 12; j++) {
            const uint32_t na = (a[j] & keep) | (odd & ((e[j] & swp) | (d[j] & ~swp)));
            n[j] = (a[j] & swp) | (n[j] & ~swp);
            a[j] = na;
        }
#pragma unroll
        for (int j = 0; j < 11; j++) { a[j] = (a[j] >> 1) | (a[j + 1] << 31); nz |= a[j]; }
        a[11] >>= 1; nz |= a[11];
        const uint32_t r = n[0] & 7u;
        t ^= (r == 3u || r == 5u) ? 1u : 0u;
    }
    uint32_t rest = n[0] ^ 1u;
#pragma unroll
    for (int j = 1; j < 12; j++) rest |= n[j];
    return rest ? 0 : ((t & 1u) ? -1 : 1);
}
// Modular inverse by the binary extended Euclidean algorithm: ~570 branch-free iterations of 12-limb shifts / subtractions (ALU
// pipe only, no multiplications) + one product -- about a tenth of the FMA-pipe time of the a^(p-2) chain, and roughly a quarter of
// its latency on a single thread.  Used where an inversion sits on a latency-critical path (the warp-cooperative pairing).
// x is the Montgomery value a R; the loop inverts that integer (y = a^-1 R^-1) and one product by R^3 returns a^-1 R.  x = 0 -> 0.
HB_NOINLINE void fp_inv_gcd(fp& r, const fp& x) {
    uint32_t u[12], v[12], x1[12], x2[12];
    uint32_t nz = 0;
#pragma unroll
    for (int j = 0; j < 12; j++) { u[j] = x.l[j]; v[j] = p_limb(j); x1[j] = j == 0; x2[j] = 0; nz |= u[j]; }
    if (!nz) { fp_zero(r); return; }
    // invariants: x1 * a == u, x2 * a == v (mod p); u, v > 0; gcd(u, v) = 1.  Every iteration removes at least one bit from u + v.
    for (int it = 0; it < 1600; it++) {
        uint32_t u1 = u[0] ^ 1u, v1 = v[0] ^ 1u;
#pragma unroll
        for (int j = 1; j < 12; j++) { u1 |= u[j]; v1 |= v[j]; }
        if (u1 == 0 || v1 == 0) break;                                // u == 1 or v == 1
        const uint32_t ue = 0u - ((u[0] & 1u) ^ 1u), ve = 0u - ((v[0] & 1u) ^ 1u);     // all-ones when even
        // d = u - v, e = v - u and the borrow of u - v (all-ones when u < v)
        uint32_t d[12], e[12], bw;
        sub_cc(d[0], u[0], v[0]);
#pragma unroll
        for (int j = 1; j < 12; j++) subc_cc(d[j], u[j], v[j]);
        subc(bw, 0, 0);
        sub_cc(e[0], v[0], u[0]);
#pragma unroll
        for (int j = 1; j < 11; j++) subc_cc(e[j], v[j], u[j]);
        subc(e[11], v[11], u[11]);
        // odd/odd: the larger one absorbs the difference (which is even) and is halved in the same iteration
        const uint32_t both_odd = ~ue & ~ve;
        const uint32_t upd_u = ue | (both_odd & ~bw);                  // u changes: u even, or both odd and u >= v
        const uint32_t upd_v = ~ue & (ve | (both_odd & bw));           // v changes: (u odd and v even), or both odd and u < v
        const uint32_t sub_u = both_odd & ~bw, sub_v = both_odd & bw;
        // coefficient updates: x1 -= x2 (mod p) when u -= v; x2 -= x1 (mod p) when v -= u
        uint32_t s1[12], s2[12], b1, b2;
        sub_cc(s1[0], x1[0], x2[0]);
#pragma unroll
        for (int j = 1; j < 12; j++) subc_cc(s1[j], x1[j], x2[j]);
        subc(b1, 0, 0);
        add_cc(s1[0], s1[0], HB_P0 & b1);
#pragma unroll
        for (int j = 1; j < 12; j++) addc_cc(s1[j], s1[j], p_limb(j) & b1);
        sub_cc(s2[0], x2[0], x1[0]);
#pragma unroll
        for (int j = 1; j < 12; j++) subc_cc(s2[j], x2[j], x1[j]);
        subc(b2, 0, 0);
        add_cc(s2[0], s2[0], HB_P0 & b2);
#pragma unroll
        for (int j = 1; j < 12; j++) addc_cc(s2[j], s2[j], p_limb(j) & b2);
#pragma unroll
        for (int j = 0; j < 12; j++) {
            u[j] = (d[j] & sub_u) | (u[j] & ~sub_u); x1[j] = (s1[j] & sub_u) | (x1[j] & ~sub_u);
            v[j] = (e[j] & sub_v) | (v[j] & ~sub_v); x2[j] = (s2[j] & sub_v) | (x2[j] & ~sub_v);
        }
        // halve the updated side: value >>= 1 ; coefficient = (coefficient + (odd ? p : 0)) >> 1
        const uint32_t o1 = 0u - (x1[0] & 1u), o2 = 0u - (x2[0] & 1u);
        uint32_t h1[12], h2[12];
        add_cc(h1[0], x1[0], HB_P0 & o1);
#pragma unroll
        for (int j = 1; j < 11; j++) addc_cc(h1[j], x1[j], p_limb(j) & o1);
        addc(h1[11], x1[11], HB_P11 & o1);
        add_cc(h2[0], x2[0], HB_P0 & o2);
#pragma unroll
        for (int j = 1; j < 11; j++) addc_cc(h2[j], x2[j], p_limb(j) & o2);
        addc(h2[11], x2[11], HB_P11 & o2);
#pragma unroll
        for (int j = 0; j < 12; j++) {
            const uint32_t un = j < 11 ? u[j + 1] : 0u, vn = j < 11 ? v[j + 1] : 0u, h1n = j < 11 ? h1[j + 1] : 0u, h2n = j < 11 ? h2[j + 1] : 0u;
            const uint32_t uh = (u[j] >> 1) | (un << 31), vh = (v[j] >> 1) | (vn << 31);
            const uint32_t x1h = (h1[j] >> 1) | (h1n << 31), x2h = (h2[j] >> 1) | (h2n << 31);
            u[j] = (uh & upd_u) | (u[j] & ~upd_u); x1[j] = (x1h & upd_u) | (x1[j] & ~upd_u);
            v[j] = (vh & upd_v) | (v[j] & ~upd_v); x2[j] = (x2h & upd_v) | (x2[j] & ~upd_v);
        }
    }
    uint32_t u1 = u[0] ^ 1u;
#pragma unroll
    for (int j = 1; j < 12; j++) u1 |= u[j];
    fp y;
#pragma unroll
    for (int j = 0; j < 12; j++) y.l[j] = u1 == 0 ? x1[j] : x2[j];
    fp_mul(r, y, fp_k(K_R3));
}
// Montgomery <-> canonical integer limbs
HB_DEV void fp_from_int(fp& r, const fp& v) { fp_mul(r, v, fp_k(K_R2)); }
HB_DEV void fp_to_int(fp& v, const fp& a) { fp_mul(v, a, fp_k(K_INT_ONE)); }
HB_DEV bool fp_int_geq_p(const fp& v) {
    uint32_t s, borrow;
    sub_cc(s, v.l[0], HB_P0);
#pragma unroll
    for (int j = 1; j < 12; j++) subc_cc(s, v.l[j], p_limb(j));
    subc(borrow, 0, 0);
    return borrow == 0;
}

// ------------------------------------------------------------------ Fp2
HB_DEV void fp2_zero(fp2& r) { fp_zero(r.a); fp_zero(r.b); }
HB_DEV void fp2_one(fp2& r) { fp_one(r.a); fp_zero(r.b); }
HB_DEV bool fp2_is_zero(const fp2& x) { return fp_is_zero(x.a) && fp_is_zero(x.b); }
HB_DEV bool fp2_eq(const fp2& x, const fp2& y) { return fp_eq(x.a, y.a) && fp_eq(x.b, y.b); }
HB_ATTR_ADD void fp2_add(fp2& r, const fp2& x, const fp2& y) { fp_add(r.a, x.a, y.a); fp_add(r.b, x.b, y.b); }
HB_ATTR_SUB void fp2_sub(fp2& r, const fp2& x, const fp2& y) { fp_sub(r.a, x.a, y.a); fp_sub(r.b, x.b, y.b); }
HB_ATTR_NEG void fp2_neg(fp2& r, const fp2& x) { fp_neg(r.a, x.a); fp_neg(r.b, x.b); }
HB_ATTR_CONJ void fp2_conj(fp2& r, const fp2& x) { r.a = x.a; fp_neg(r.b, x.b); }
HB_ATTR_DBL void fp2_dbl(fp2& r, const fp2& x) { fp_dbl(r.a, x.a); fp_dbl(r.b, x.b); }
HB_DEV void fp2_half(fp2& r, const fp2& x) { fp_half(r.a, x.a); fp_half(r.b, x.b); }
HB_DEV void fp2_const(fp2& r, const uint32_t k[2][12]) { fp_set(r.a, k[0]); fp_set(r.b, k[1]); }
HB_DEV void fp2_cmov(fp2& r, const fp2& x, bool c) { fp_cmov(r.a, x.a, c); fp_cmov(r.b, x.b, c); }

#ifndef HB_FUSED_FP2
#define HB_FUSED_FP2 0      // 0: three out-of-line CIOS products (fastest measured); 1: lazy-reduction fused; 2: fused CIOS
#endif
#if HB_FUSED_FP2
// register-resident Karatsuba with lazy reduction (fp_wide.cuh): 744 IMAD.WIDE, operands touched once
HB_NOINLINE void fp2_mul(fp2& r, const fp2& x, const fp2& y) {
    uint32_t xa[12], xb[12], ya[12], yb[12], ra[12], rb[12];
#pragma unroll
    for (int j = 0; j < 12; j++) { xa[j] = x.a.l[j]; xb[j] = x.b.l[j]; ya[j] = y.a.l[j]; yb[j] = y.b.l[j]; }
#if HB_FUSED_FP2 == 2
    fp2_mul_regs_cios(ra, rb, xa, xb, ya, yb);
#else
    fp2_mul_regs(ra, rb, xa, xb, ya, yb);
#endif
#pragma unroll
    for (int j = 0; j < 12; j++) { r.a.l[j] = ra[j]; r.b.l[j] = rb[j]; }
}
HB_NOINLINE void fp2_sqr(fp2& r, const fp2& x) {
    uint32_t xa[12], xb[12], ra[12], rb[12];
#pragma unroll
    for (int j = 0; j < 12; j++) { xa[j] = x.a.l[j]; xb[j] = x.b.l[j]; }
#if HB_FUSED_FP2 == 2
    fp2_sqr_regs_cios(ra, rb, xa, xb);
#else
    fp2_sqr_regs(ra, rb, xa, xb);
#endif
#pragma unroll
    for (int j = 0; j < 12; j++) { r.a.l[j] = ra[j]; r.b.l[j] = rb[j]; }
}
#else
HB_NOINLINE void fp2_mul(fp2& r, const fp2& x, const fp2& y) {
    fp t0, t1, t2, s0, s1;
    fp_mul(t0, x.a, y.a); fp_mul(t1, x.b, y.b);
    fp_add(s0, x.a, x.b); fp_add(s1, y.a, y.b); fp_mul(t2, s0, s1);
    fp_sub(r.a, t0, t1); fp_sub(t2, t2, t0); fp_sub(r.b, t2, t1);
}
HB_NOINLINE void fp2_sqr(fp2& r, const fp2& x) {
    fp s, d, m;
    fp_add(s, x.a, x.b); fp_sub(d, x.a, x.b); fp_mul(m, x.a, x.b);
    fp_mul(r.a, s, d); fp_dbl(r.b, m);
}
#endif
HB_ATTR_MULFP void fp2_mul_fp(fp2& r, const fp2& x, const fp& k) { fp_mul(r.a, x.a, k); fp_mul(r.b, x.b, k); }
HB_ATTR_MULXI void fp2_mul_xi(fp2& r, const fp2& x) { fp t; fp_sub(t, x.a, x.b); fp_add(r.b, x.a, x.b); r.a = t; }
HB_DEV void fp2_norm(fp& r, const fp2& x) { fp t; fp_sqr(r, x.a); fp_sqr(t, x.b); fp_add(r, r, t); }
HB_NOINLINE void fp2_inv(fp2& r, const fp2& x) {
    fp n; fp2_norm(n, x); fp_inv(n, n);
    fp_mul(r.a, x.a, n); fp_mul(r.b, x.b, n); fp_neg(r.b, r.b);
}
// mcl Fp2::squareRoot (SURVEY A.4): fixes WHICH root is produced -- bit-exactness of hash-to-G2 and of
// signature decompression depends on it
HB_NOINLINE bool fp2_sqrt(fp2& r, const fp2& x) {
    fp t1, t2;
    if (fp_is_zero(x.b)) {
        if (fp_sqrt(t1, x.a)) { r.a = t1; fp_zero(r.b); }
        else { fp_neg(t2, x.a); if (!fp_sqrt(t1, t2)) return false; fp_zero(r.a); r.b = t1; }
        return true;
    }
    fp2_norm(t1, x);
    if (!fp_sqrt(t1, t1)) return false;
    const fp& inv2 = fp_k(K_INV2);
    // mcl: c = sqrt((a + s)/2), or sqrt((a - s)/2) when the first is a non-residue, always the root t^((p+1)/4)
    // (the one that is itself a residue); then (c, b / 2c).  One exponentiation serves both cases: with
    // u = t^((p-3)/4), c = t u:  c^2 == t -> (c, b u / 2).  Otherwise c^2 == -t and u == -1/c, the other half is
    // (b u / 2)^2, its residue root is sigma * (-b u / 2) with sigma = Legendre(-b u / 2), and b / 2c' = sigma c.
    fp u, c, c2, h;
    fp_add(t2, x.a, t1); fp_mul(t2, t2, inv2);
    fp_pow(u, t2, K_P_MINUS_3_DIV_4); fp_mul(c, u, t2); fp_sqr(c2, c);
    fp_mul(h, x.b, u); fp_mul(h, h, inv2);                    // b u / 2
    if (fp_eq(c2, t2)) { r.a = c; r.b = h; return true; }
    fp_neg(c2, c2);
    if (!fp_eq(c2, t2)) return false;
    fp_neg(h, h);
    if (fp_legendre(h) < 0) { fp_neg(h, h); fp_neg(c, c); }
    r.a = h; r.b = c;
    return true;
}

// A square root of x with NO promise about which of the two (callers fix the sign themselves, e.g. point
// decompression by the parity bit): two exponentiations instead of three.  With t = (a + sqrt(N))/2 and
// u = t^((p-3)/4), c = t u:  c^2 == t  -> root (c, b u / 2);  otherwise c^2 == -t, u == -1/c, the other half
// t' = (a - sqrt(N))/2 = (b / 2c)^2 is the square and the root is (-b u / 2, c).
HB_NOINLINE bool fp2_sqrt_anysign(fp2& r, const fp2& x) {
    if (fp_is_zero(x.b)) return fp2_sqrt(r, x);
    fp n, t, u, c, c2, h;
    fp2_norm(n, x);
    if (!fp_sqrt(n, n)) return false;
    const fp& inv2 = fp_k(K_INV2);
    fp_add(t, x.a, n); fp_mul(t, t, inv2);
    fp_pow(u, t, K_P_MINUS_3_DIV_4); fp_mul(c, u, t); fp_sqr(c2, c);
    fp_mul(h, x.b, u); fp_mul(h, h, inv2);                    // b u / 2
    if (fp_eq(c2, t)) { r.a = c; r.b = h; return true; }
    fp_neg(c2, c2);
    if (!fp_eq(c2, t)) return false;                            // t == 0 cannot happen for b != 0
    fp_neg(r.a, h); r.b = c;
    return true;
}

// ------------------------------------------------------------------ Fp2 split across a lane pair (fp2h)
// Two adjacent lanes (2k, 2k+1) co-own every Fp2 value of one pairing: the even lane holds the real part, the odd lane
// the imaginary part.  Per-thread state (and stack traffic) of the Miller loop / final exponentiation halves, so twice
// as many warps fit the same L1/L2 footprint; products exchange 24 words by __shfl_xor and cost 2 wide products + 1
// reduction per lane (schoolbook, perfectly balanced); squarings cost 1 + 1.  All role-dependent choices are selects,
// so the instruction stream is identical in both lanes.  Control flow must be pair-uniform (it is: the pairing code is
// data-oblivious), because the exchanges use full-warp shuffles.
struct fp2h { fp c; };
#ifdef HB_HOST_EMU
// host emulation (tests/emu): two host threads play the two lanes of ONE pair; role = lane parity, and a shuffle with the
// partner lane is a rendezvous through a pair of slots (sequence numbers: publish, wait for the partner's value of the same
// exchange, acknowledge so the partner may overwrite its slot at the next exchange)
struct fp2h_emu_ctx { int role; uint64_t seq; };
static thread_local fp2h_emu_ctx hb_emu = {0, 0};
struct hb_emu_pair_t { std::atomic<uint32_t> slot[2]; std::atomic<uint64_t> pub[2], ack[2]; };
static hb_emu_pair_t hb_emu_pair;
static inline void hb_emu_pair_reset() { for (int i = 0; i < 2; i++) { hb_emu_pair.pub[i] = 0; hb_emu_pair.ack[i] = 0; } }
static inline uint32_t hb_emu_exchange(uint32_t v) {
    const int me = hb_emu.role, other = me ^ 1;
    const uint64_t n = ++hb_emu.seq;
    while (hb_emu_pair.ack[other].load(std::memory_order_acquire) < n - 1) std::this_thread::yield();   // partner consumed my previous value
    hb_emu_pair.slot[me].store(v, std::memory_order_relaxed);
    hb_emu_pair.pub[me].store(n, std::memory_order_release);
    while (hb_emu_pair.pub[other].load(std::memory_order_acquire) < n) std::this_thread::yield();
    const uint32_t got = hb_emu_pair.slot[other].load(std::memory_order_relaxed);
    hb_emu_pair.ack[me].store(n, std::memory_order_release);
    return got;
}
template <class T> static inline T __shfl_xor_sync(unsigned, T v, int) { return (T)hb_emu_exchange((uint32_t)v); }
#endif
// Exchanges between the two lanes of a pair name only those two lanes in the shuffle mask: pairs of one warp may then diverge
// (data-dependent branches of the point arithmetic on hostile inputs) without leaving a shuffle short of participants.
#ifdef HB_HOST_EMU
#define HB_PAIR_MASK 0u
#else
#define HB_PAIR_MASK (3u << (threadIdx.x & 30u))
#endif
HB_DEV int fp2h_role() {
#ifdef HB_HOST_EMU
    return hb_emu.role;
#else
    return threadIdx.x & 1;
#endif
}
HB_DEV void fp2h_partner(fp& r, const fp& x) {
#pragma unroll
    for (int j = 0; j < 12; j++) r.l[j] = __shfl_xor_sync(HB_PAIR_MASK, x.l[j], 1);
}
HB_DEV void fp2_zero(fp2h& r) { fp_zero(r.c); }
HB_DEV void fp2_one(fp2h& r) { fp o; fp_one(o); fp z; fp_zero(z); r.c = z; fp_cmov(r.c, o, fp2h_role() == 0); }
HB_DEV bool fp2_is_zero(const fp2h& x) {
    bool mine = fp_is_zero(x.c);
    bool other = __shfl_xor_sync(HB_PAIR_MASK, mine ? 1 : 0, 1) != 0;
    return mine && other;
}
HB_DEV void fp2_const(fp2h& r, const uint32_t k[2][12]) { fp_set(r.c, k[fp2h_role()]); }
// fp2_k for either carrier (see fp_k): the whole constant, or this lane's half of it
template <class E> HB_DEV const E& fp2_k(const uint32_t k[2][12]);
template <> HB_DEV const fp2& fp2_k<fp2>(const uint32_t k[2][12]) { return fp2_k(k); }
template <> HB_DEV const fp2h& fp2_k<fp2h>(const uint32_t k[2][12]) { return *reinterpret_cast<const fp2h*>(k[fp2h_role()]); }
// both lanes always reach the exchange: with `mine && shfl(..)` a lane whose own half differs skipped it, and its partner then
// waited on a shuffle the pair did not execute together (a difference confined to one half, e.g. in pt_eq of the subgroup test)
HB_DEV bool fp2_eq(const fp2h& x, const fp2h& y) {
    const int mine = fp_eq(x.c, y.c) ? 1 : 0;
    const int other = __shfl_xor_sync(HB_PAIR_MASK, mine, 1);
    return mine && other;
}
HB_DEV void fp2_cmov(fp2h& r, const fp2h& x, bool c) { fp_cmov(r.c, x.c, c); }
// whole value <-> the pair's halves (both lanes end up holding the full Fp2 element / each lane keeps its own half)
HB_DEV void fp2h_unpack(fp2& r, const fp2h& x) {
    fp o; 
#pragma unroll
    for (int j = 0; j < 12; j++) o.l[j] = __shfl_xor_sync(HB_PAIR_MASK, x.c.l[j], 1);
    const bool im = fp2h_role() == 1;
    r.a = im ? o : x.c; r.b = im ? x.c : o;
}
HB_DEV void fp2h_pack(fp2h& r, const fp2& x) { r.c = fp2h_role() == 1 ? x.b : x.a; }
#ifndef HB_SPLIT_INLINE
#define HB_SPLIT_INLINE 1
#endif
#if HB_SPLIT_INLINE
#define HB_ATTR_H __device__ __forceinline__
#else
#define HB_ATTR_H __device__ __noinline__
#endif
HB_ATTR_H void fp2_add(fp2h& r, const fp2h& x, const fp2h& y) { fp_add(r.c, x.c, y.c); }
HB_ATTR_H void fp2_sub(fp2h& r, const fp2h& x, const fp2h& y) { fp_sub(r.c, x.c, y.c); }
HB_ATTR_H void fp2_neg(fp2h& r, const fp2h& x) { fp_neg(r.c, x.c); }
HB_ATTR_H void fp2_dbl(fp2h& r, const fp2h& x) { fp_dbl(r.c, x.c); }
HB_ATTR_H void fp2_conj(fp2h& r, const fp2h& x) { fp n; fp_neg(n, x.c); r.c = x.c; fp_cmov(r.c, n, fp2h_role() == 1); }
HB_ATTR_MULFP void fp2_mul_fp(fp2h& r, const fp2h& x, const fp& k) { fp_mul(r.c, x.c, k); }
HB_DEV void fp2_half(fp2h& r, const fp2h& x) { fp_half(r.c, x.c); }
// xi * (a + b i) = (a - b) + (a + b) i
HB_ATTR_H void fp2_mul_xi(fp2h& r, const fp2h& x) {
    fp o, s, d; fp2h_partner(o, x.c);
    fp_add(s, x.c, o);                 // role 1 result
    fp_sub(d, x.c, o);                 // role 0 result (a - b)
    r.c = s; fp_cmov(r.c, d, fp2h_role() == 0);
}
// real: xo*yo + xp*(p - yp) ; imag: xo*yp + xp*yo   (o = own, p = partner): both lanes ADD two wide products that share
// one accumulator pair (mul_wide2), then reduce once -- 288 + 156 IMAD.WIDE per lane
HB_NOINLINE void fp2_mul(fp2h& r, const fp2h& x, const fp2h& y) {
    const bool im = fp2h_role() == 1;
    uint32_t xo[12], yo[12], xp[12], yp[12], A[12], B[12], T[24], rr[12];
#pragma unroll
    for (int j = 0; j < 12; j++) { xo[j] = x.c.l[j]; yo[j] = y.c.l[j]; }
#pragma unroll
    for (int j = 0; j < 12; j++) { xp[j] = __shfl_xor_sync(HB_PAIR_MASK, xo[j], 1); yp[j] = __shfl_xor_sync(HB_PAIR_MASK, yo[j], 1); }
    uint32_t ny[12];                                   // p - yp in (0, p]
    sub_cc(ny[0], HB_P0, yp[0]);
#pragma unroll
    for (int j = 1; j < 11; j++) subc_cc(ny[j], p_limb(j), yp[j]);
    subc(ny[11], HB_P11, yp[11]);
#pragma unroll
    for (int j = 0; j < 12; j++) { A[j] = im ? yp[j] : yo[j]; B[j] = im ? yo[j] : ny[j]; }
    HB_MUL_WIDE2(T, xo, A, xp, B);                     // < 2 p^2 < p R
    redc_wide(rr, T);
#pragma unroll
    for (int j = 0; j < 12; j++) r.c.l[j] = rr[j];
}
// real: (xo + xp)(xo - xp) ; imag: 2 xo xp -- 1 wide product + 1 reduction per lane
HB_NOINLINE void fp2_sqr(fp2h& r, const fp2h& x) {
    const bool im = fp2h_role() == 1;
    uint32_t xo[12], xp[12], s[12], d[12], t[12], A[12], B[12], T[24], rr[12];
#pragma unroll
    for (int j = 0; j < 12; j++) xo[j] = x.c.l[j];
#pragma unroll
    for (int j = 0; j < 12; j++) xp[j] = __shfl_xor_sync(HB_PAIR_MASK, xo[j], 1);
    limbs_add12(s, xo, xp);            // < 2p
    limbs_sub12_plus_p(d, xo, xp);     // in (0, 2p)
    limbs_add12(t, xp, xp);            // 2 xp < 2p
#pragma unroll
    for (int j = 0; j < 12; j++) { A[j] = im ? xo[j] : s[j]; B[j] = im ? t[j] : d[j]; }
    HB_MUL_WIDE(T, A, B);              // < 4 p^2 < p R
    redc_wide(rr, T);
#pragma unroll
    for (int j = 0; j < 12; j++) r.c.l[j] = rr[j];
}
HB_NOINLINE void fp2_inv(fp2h& r, const fp2h& x) {
    fp sq, o, n; fp_sqr(sq, x.c); fp2h_partner(o, sq); fp_add(n, sq, o);      // a^2 + b^2 (both lanes)
    fp_inv(n, n);
    fp t, m; fp_mul(t, x.c, n); fp_neg(m, t);
    r.c = t; fp_cmov(r.c, m, fp2h_role() == 1);
}

// latency-path inversion: same as fp2_inv with the binary-GCD Fp inverse
HB_NOINLINE void fp2_inv_gcd(fp2& r, const fp2& x) {
    fp n; fp2_norm(n, x); fp_inv_gcd(n, n);
    fp_mul(r.a, x.a, n); fp_mul(r.b, x.b, n); fp_neg(r.b, r.b);
}
HB_NOINLINE void fp2_inv_gcd(fp2h& r, const fp2h& x) {
    fp sq, o, n; fp_sqr(sq, x.c); fp2h_partner(o, sq); fp_add(n, sq, o);
    fp_inv_gcd(n, n);
    fp t, m; fp_mul(t, x.c, n); fp_neg(m, t);
    r.c = t; fp_cmov(r.c, m, fp2h_role() == 1);
}

// Lock-step hint: with many resident warps the pairing is instruction-fetch bound because warps drift through ~60 KB of
// hot code.  The lane-pair kernels keep every thread of a
// CTA alive with identical trip counts, so a CTA barrier per Fp12 operation keeps its warps on the same cache lines.
template <class E> HB_DEV void hb_lockstep() {}
#ifndef HB_HOST_EMU
#ifndef HB_LOCKSTEP
#define HB_LOCKSTEP 1
#endif
#if HB_LOCKSTEP
template <> HB_DEV void hb_lockstep<fp2h>() { __syncthreads(); }
#endif
#endif
// finer-grained barriers (HB_LOCKSTEP >= 2: every Fp12-level operation, >= 3: every Fp6 product)
template <class E> HB_DEV void hb_lockstep2() {
#if defined(HB_LOCKSTEP) && HB_LOCKSTEP >= 2
    hb_lockstep<E>();
#endif
}
template <class E> HB_DEV void hb_lockstep3() {
#if defined(HB_LOCKSTEP) && HB_LOCKSTEP >= 3
    hb_lockstep<E>();
#endif
}

// ------------------------------------------------------------------ Fp6 / Fp12, generic over the Fp2 carrier E (fp2 or fp2h)
template <class E> struct fp6_t { E c0, c1, c2; };
// 3 b' x for the twist constant b' = 4 (1 + i): 12 (1 + i) x by additions only (mul_xi, three doublings, one addition) instead of an
// Fp2 product by a constant
template <class E> HB_DEV void fp2_mul_twist3b(E& r, const E& x) { E t, u; fp2_mul_xi(t, x); fp2_dbl(t, t); fp2_dbl(t, t); fp2_dbl(u, t); fp2_add(r, t, u); }
template <class E> struct fp12_t { fp6_t<E> c0, c1; };
typedef fp6_t<fp2> fp6;
typedef fp12_t<fp2> fp12;

template <class E> HB_DEV void fp6_add(fp6_t<E>& r, const fp6_t<E>& x, const fp6_t<E>& y) { fp2_add(r.c0, x.c0, y.c0); fp2_add(r.c1, x.c1, y.c1); fp2_add(r.c2, x.c2, y.c2); }
template <class E> HB_DEV void fp6_sub(fp6_t<E>& r, const fp6_t<E>& x, const fp6_t<E>& y) { fp2_sub(r.c0, x.c0, y.c0); fp2_sub(r.c1, x.c1, y.c1); fp2_sub(r.c2, x.c2, y.c2); }
template <class E> HB_DEV void fp6_neg(fp6_t<E>& r, const fp6_t<E>& x) { fp2_neg(r.c0, x.c0); fp2_neg(r.c1, x.c1); fp2_neg(r.c2, x.c2); }
template <class E> HB_DEV void fp6_mul_v(fp6_t<E>& r, const fp6_t<E>& x) { E t; fp2_mul_xi(t, x.c2); r.c2 = x.c1; r.c1 = x.c0; r.c0 = t; }
template <class E> HB_NOINLINE void fp6_mul(fp6_t<E>& r, const fp6_t<E>& x, const fp6_t<E>& y) {
    hb_lockstep3<E>();
    E v0, v1, v2, t0, t1, t2, s;
    fp2_mul(v0, x.c0, y.c0); fp2_mul(v1, x.c1, y.c1); fp2_mul(v2, x.c2, y.c2);
    fp2_add(t0, x.c1, x.c2); fp2_add(s, y.c1, y.c2); fp2_mul(t0, t0, s);
    fp2_sub(t0, t0, v1); fp2_sub(t0, t0, v2); fp2_mul_xi(t0, t0); fp2_add(t0, t0, v0);
    fp2_add(t1, x.c0, x.c1); fp2_add(s, y.c0, y.c1); fp2_mul(t1, t1, s);
    fp2_sub(t1, t1, v0); fp2_sub(t1, t1, v1); fp2_mul_xi(s, v2); fp2_add(t1, t1, s);
    fp2_add(t2, x.c0, x.c2); fp2_add(s, y.c0, y.c2); fp2_mul(t2, t2, s);
    fp2_sub(t2, t2, v0); fp2_sub(t2, t2, v2); fp2_add(t2, t2, v1);
    r.c0 = t0; r.c1 = t1; r.c2 = t2;
}
// x * (b0 + b1 v)
template <class E> HB_NOINLINE void fp6_mul_by_01(fp6_t<E>& r, const fp6_t<E>& x, const E& b0, const E& b1) {
    E v0, v1, t0, t1, t2, s;
    fp2_mul(v0, x.c0, b0); fp2_mul(v1, x.c1, b1);
    fp2_mul(t0, x.c2, b1); fp2_mul_xi(t0, t0); fp2_add(t0, t0, v0);
    fp2_add(t1, x.c0, x.c1); fp2_add(s, b0, b1); fp2_mul(t1, t1, s); fp2_sub(t1, t1, v0); fp2_sub(t1, t1, v1);
    fp2_mul(t2, x.c2, b0); fp2_add(t2, t2, v1);
    r.c0 = t0; r.c1 = t1; r.c2 = t2;
}
// x * (b1 v)
template <class E> HB_NOINLINE void fp6_mul_by_1(fp6_t<E>& r, const fp6_t<E>& x, const E& b1) {
    E t0, t1, t2;
    fp2_mul(t0, x.c2, b1); fp2_mul_xi(t0, t0);
    fp2_mul(t1, x.c0, b1); fp2_mul(t2, x.c1, b1);
    r.c0 = t0; r.c1 = t1; r.c2 = t2;
}
template <class E> HB_NOINLINE void fp6_inv(fp6_t<E>& r, const fp6_t<E>& x) {
    E t0, t1, t2, s, d;
    fp2_sqr(t0, x.c0); fp2_mul(s, x.c1, x.c2); fp2_mul_xi(s, s); fp2_sub(t0, t0, s);
    fp2_sqr(t1, x.c2); fp2_mul_xi(t1, t1); fp2_mul(s, x.c0, x.c1); fp2_sub(t1, t1, s);
    fp2_sqr(t2, x.c1); fp2_mul(s, x.c0, x.c2); fp2_sub(t2, t2, s);
    fp2_mul(d, x.c2, t1); fp2_mul(s, x.c1, t2); fp2_add(d, d, s); fp2_mul_xi(d, d);
    fp2_mul(s, x.c0, t0); fp2_add(d, d, s);
    fp2_inv(d, d);
    fp2_mul(r.c0, t0, d); fp2_mul(r.c1, t1, d); fp2_mul(r.c2, t2, d);
}

template <class E> HB_DEV void fp12_one(fp12_t<E>& r) {
    fp2_one(r.c0.c0); fp2_zero(r.c0.c1); fp2_zero(r.c0.c2); fp2_zero(r.c1.c0); fp2_zero(r.c1.c1); fp2_zero(r.c1.c2);
}
template <class E> HB_DEV bool fp12_is_one(const fp12_t<E>& x) {
    // every term is evaluated (no short-circuit): for the lane-pair carrier fp2_is_zero contains a full-warp shuffle,
    // which must be executed by all lanes even when another round in the warp already knows its answer
    E d = x.c0.c0; fp_sub(d.a, d.a, fp_k(K_ONE));
    const bool z0 = fp2_is_zero(d), z1 = fp2_is_zero(x.c0.c1), z2 = fp2_is_zero(x.c0.c2);
    const bool z3 = fp2_is_zero(x.c1.c0), z4 = fp2_is_zero(x.c1.c1), z5 = fp2_is_zero(x.c1.c2);
    return z0 & z1 & z2 & z3 & z4 & z5;
}
// lane-pair carrier: each lane tests its own six components, ONE shuffle combines the pair's verdicts
HB_DEV bool fp12_is_one(const fp12_t<fp2h>& x) {
    fp one; fp_one(one);
    const bool re = fp2h_role() == 0;
    uint32_t acc = 0;
#pragma unroll
    for (int j = 0; j < 12; j++) {
        acc |= x.c0.c0.c.l[j] ^ (re ? one.l[j] : 0u);
        acc |= x.c0.c1.c.l[j] | x.c0.c2.c.l[j] | x.c1.c0.c.l[j] | x.c1.c1.c.l[j] | x.c1.c2.c.l[j];
    }
    const int mine = acc == 0;
    const int other = __shfl_xor_sync(HB_PAIR_MASK, mine, 1);
    return mine && other;
}
template <class E> HB_NOINLINE void fp12_mul(fp12_t<E>& r, const fp12_t<E>& x, const fp12_t<E>& y) {
    hb_lockstep2<E>();
    fp6_t<E> v0, v1, s, t;
    fp6_mul(v0, x.c0, y.c0); fp6_mul(v1, x.c1, y.c1);
    fp6_add(s, x.c0, x.c1); fp6_add(t, y.c0, y.c1); fp6_mul(s, s, t);
    fp6_sub(s, s, v0); fp6_sub(s, s, v1);
    fp6_mul_v(t, v1); fp6_add(r.c0, v0, t); r.c1 = s;
}
template <class E> HB_NOINLINE void fp12_sqr(fp12_t<E>& r, const fp12_t<E>& x) {
    hb_lockstep2<E>();
    fp6_t<E> ab, s, t;
    fp6_mul(ab, x.c0, x.c1);
    fp6_add(s, x.c0, x.c1); fp6_mul_v(t, x.c1); fp6_add(t, t, x.c0); fp6_mul(s, s, t);
    fp6_sub(s, s, ab); fp6_mul_v(t, ab); fp6_sub(r.c0, s, t);
    fp6_add(r.c1, ab, ab);
}
template <class E> HB_DEV void fp12_conj(fp12_t<E>& r, const fp12_t<E>& x) { r.c0 = x.c0; fp6_neg(r.c1, x.c1); }
template <class E> HB_NOINLINE void fp12_inv(fp12_t<E>& r, const fp12_t<E>& x) {
    fp6_t<E> t0, t1;
    fp6_mul(t0, x.c0, x.c0); fp6_mul(t1, x.c1, x.c1); fp6_mul_v(t1, t1); fp6_sub(t0, t0, t1);
    fp6_inv(t0, t0);
    fp6_mul(r.c0, x.c0, t0); fp6_mul(t1, x.c1, t0); fp6_neg(r.c1, t1);
}
// sparse multiply by a Miller line (o0 + o1 v) + (o4 v) w : non-zero coefficients at w^0, w^2, w^3
template <class E> HB_NOINLINE void fp12_mul_by_014(fp12_t<E>& r, const fp12_t<E>& x, const E& o0, const E& o1, const E& o4) {
    hb_lockstep2<E>();
    fp6_t<E> aa, bb, s; E o14;
    fp6_mul_by_01(aa, x.c0, o0, o1);
    fp6_mul_by_1(bb, x.c1, o4);
    fp2_add(o14, o1, o4);
    fp6_add(s, x.c0, x.c1); fp6_mul_by_01(s, s, o0, o14);
    fp6_sub(s, s, aa); fp6_sub(s, s, bb);
    fp6_mul_v(bb, bb); fp6_add(r.c0, aa, bb); r.c1 = s;
}
// x * (d1 v + d2 v^2): 5 products
template <class E> HB_NOINLINE void fp6_mul_by_12(fp6_t<E>& r, const fp6_t<E>& x, const E& d1, const E& d2) {
    E m1, m2, m12, s, t, u0, u1;
    fp2_mul(m1, x.c1, d1); fp2_mul(m2, x.c2, d2);
    fp2_add(s, x.c1, x.c2); fp2_add(t, d1, d2); fp2_mul(m12, s, t); fp2_sub(m12, m12, m1); fp2_sub(m12, m12, m2);      // x1 d2 + x2 d1
    fp2_mul(u0, x.c0, d1); fp2_mul(u1, x.c0, d2);
    fp2_mul_xi(r.c0, m12);
    fp2_mul_xi(s, m2); fp2_add(r.c1, u0, s);
    fp2_add(r.c2, u1, m1);
}
// x * (la * lb) for two Miller lines la = (a0 + a1 v) + (a4 v) w, lb likewise: the product of the lines first (6 products: it has five
// non-zero coefficients), then ONE multiplication by it (17) -- 23 Fp2 products instead of 2 x 13
template <class E> HB_NOINLINE void fp12_mul_by_two_lines(fp12_t<E>& r, const fp12_t<E>& x, const E& a0, const E& a1, const E& a4, const E& b0, const E& b1, const E& b4) {
    hb_lockstep2<E>();
    E t00, t11, t44, s, t, d1, d2;
    fp6_t<E> C0;
    fp2_mul(t00, a0, b0); fp2_mul(t11, a1, b1); fp2_mul(t44, a4, b4);
    fp2_add(s, a0, a1); fp2_add(t, b0, b1); fp2_mul(C0.c1, s, t); fp2_sub(C0.c1, C0.c1, t00); fp2_sub(C0.c1, C0.c1, t11);   // a0 b1 + a1 b0
    fp2_add(s, a0, a4); fp2_add(t, b0, b4); fp2_mul(d1, s, t); fp2_sub(d1, d1, t00); fp2_sub(d1, d1, t44);                  // a0 b4 + a4 b0
    fp2_add(s, a1, a4); fp2_add(t, b1, b4); fp2_mul(d2, s, t); fp2_sub(d2, d2, t11); fp2_sub(d2, d2, t44);                  // a1 b4 + a4 b1
    fp2_mul_xi(s, t44); fp2_add(C0.c0, t00, s); C0.c2 = t11;
    // x * (C0 + (d1 v + d2 v^2) w)
    fp6_t<E> v0, v1, sx, sc;
    fp6_mul(v0, x.c0, C0);
    fp6_mul_by_12(v1, x.c1, d1, d2);
    fp6_add(sx, x.c0, x.c1);
    sc.c0 = C0.c0; fp2_add(sc.c1, C0.c1, d1); fp2_add(sc.c2, C0.c2, d2);
    fp6_mul(sx, sx, sc);
    fp6_sub(sx, sx, v0); fp6_sub(sx, sx, v1);
    fp6_mul_v(sc, v1); fp6_add(r.c0, v0, sc); r.c1 = sx;
}
// coefficient of w^k (k = 2i + j) <-> tower slot
template <class E> HB_DEV E& fp12_slot(fp12_t<E>& x, int k) {
    fp6_t<E>& h = (k & 1) ? x.c1 : x.c0;
    int i = k >> 1;
    return i == 0 ? h.c0 : (i == 1 ? h.c1 : h.c2);
}
template <class E> HB_NOINLINE void fp12_frob(fp12_t<E>& r, const fp12_t<E>& x) {
    fp12_t<E> t = x;
    for (int k = 0; k < 6; k++) {
        E& s = fp12_slot(t, k);
        fp2_conj(s, s); fp2_mul(s, s, fp2_k<E>(K_FROB1[k]));
    }
    r = t;
}
template <class E> HB_NOINLINE void fp12_frob2(fp12_t<E>& r, const fp12_t<E>& x) {
    fp12_t<E> t = x;
    for (int k = 0; k < 6; k++) { E& s = fp12_slot(t, k); fp2_mul_fp(s, s, fp_k(K_FROB2[k])); }
    r = t;
}
// Granger-Scott squaring in the cyclotomic subgroup (valid after the easy part of the final exponentiation)
template <class E> HB_DEV void fp4_sqr(E& c0, E& c1, const E& a, const E& b) {
    E t0, t1, t2;
    fp2_sqr(t0, a); fp2_sqr(t1, b);
    fp2_mul_xi(t2, t1); fp2_add(c0, t2, t0);
    fp2_add(t2, a, b); fp2_sqr(t2, t2); fp2_sub(t2, t2, t0); fp2_sub(c1, t2, t1);
}
template <class E> HB_NOINLINE void fp12_cyc_sqr(fp12_t<E>& r, const fp12_t<E>& x) {
    hb_lockstep2<E>();
    E z0 = x.c0.c0, z4 = x.c0.c1, z3 = x.c0.c2, z2 = x.c1.c0, z1 = x.c1.c1, z5 = x.c1.c2;
    E t0, t1, t2, t3;
    fp4_sqr(t0, t1, z0, z1);
    fp2_sub(z0, t0, z0); fp2_dbl(z0, z0); fp2_add(z0, z0, t0);
    fp2_add(z1, t1, z1); fp2_dbl(z1, z1); fp2_add(z1, z1, t1);
    fp4_sqr(t0, t1, z2, z3);
    fp4_sqr(t2, t3, z4, z5);
    fp2_sub(z4, t0, z4); fp2_dbl(z4, z4); fp2_add(z4, z4, t0);
    fp2_add(z5, t1, z5); fp2_dbl(z5, z5); fp2_add(z5, z5, t1);
    fp2_mul_xi(t0, t3);
    fp2_add(z2, t0, z2); fp2_dbl(z2, z2); fp2_add(z2, z2, t0);
    fp2_sub(z3, t2, z3); fp2_dbl(z3, z3); fp2_add(z3, z3, t2);
    r.c0.c0 = z0; r.c0.c1 = z4; r.c0.c2 = z3; r.c1.c0 = z2; r.c1.c1 = z1; r.c1.c2 = z5;
}
// r = x^z, z = -0xd201000000010000, x in the cyclotomic subgroup
template <class E> HB_NOINLINE void fp12_cyc_exp_z(fp12_t<E>& r, const fp12_t<E>& x) {
    fp12_t<E> acc = x;
    for (int i = 62; i >= 0; i--) {
        hb_lockstep<E>();
        fp12_cyc_sqr(acc, acc);
        if ((K_Z_ABS >> i) & 1) fp12_mul(acc, acc, x);
    }
    fp12_conj(r, acc);
}

}  // namespace hb
