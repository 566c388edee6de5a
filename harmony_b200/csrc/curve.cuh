// harmony_b200/csrc/curve.cuh -- G1 = E(Fp): y^2 = x^3 + 4 and G2 = E'(Fp2): y^2 = x^3 + 4(1+i), Jacobian coordinates.
// SWAP_G layout of the reference: public keys live in G1 (48 B), signatures in G2 (96 B)
// (reference crypto/bls/bls.go:18-21).  The all-zero struct is the identity, matching the zero-value Go structs
// the reference starts every aggregate from (crypto/bls/mask.go:59,88).
#pragma once
#include "tower.cuh"

namespace hb {

// ---- overloads so the point arithmetic is written once for both coordinate fields
HB_DEV void f_add(fp& r, const fp& a, const fp& b) { fp_add(r, a, b); }
HB_DEV void f_sub(fp& r, const fp& a, const fp& b) { fp_sub(r, a, b); }
HB_DEV void f_dbl(fp& r, const fp& a) { fp_dbl(r, a); }
HB_DEV void f_neg(fp& r, const fp& a) { fp_neg(r, a); }
HB_DEV void f_mul(fp& r, const fp& a, const fp& b) { fp_mul(r, a, b); }
HB_DEV void f_sqr(fp& r, const fp& a) { fp_sqr(r, a); }
HB_DEV void f_inv(fp& r, const fp& a) { fp_inv(r, a); }
HB_DEV bool f_is_zero(const fp& a) { return fp_is_zero(a); }
HB_DEV bool f_eq(const fp& a, const fp& b) { return fp_eq(a, b); }
HB_DEV void f_zero(fp& r) { fp_zero(r); }
HB_DEV void f_one(fp& r) { fp_one(r); }
HB_DEV void f_cmov(fp& r, const fp& a, bool c) { fp_cmov(r, a, c); }

HB_DEV void f_add(fp2& r, const fp2& a, const fp2& b) { fp2_add(r, a, b); }
HB_DEV void f_sub(fp2& r, const fp2& a, const fp2& b) { fp2_sub(r, a, b); }
HB_DEV void f_dbl(fp2& r, const fp2& a) { fp2_dbl(r, a); }
HB_DEV void f_neg(fp2& r, const fp2& a) { fp2_neg(r, a); }
HB_DEV void f_mul(fp2& r, const fp2& a, const fp2& b) { fp2_mul(r, a, b); }
HB_DEV void f_sqr(fp2& r, const fp2& a) { fp2_sqr(r, a); }
HB_DEV void f_inv(fp2& r, const fp2& a) { fp2_inv(r, a); }
HB_DEV bool f_is_zero(const fp2& a) { return fp2_is_zero(a); }
HB_DEV bool f_eq(const fp2& a, const fp2& b) { return fp2_eq(a, b); }
HB_DEV void f_zero(fp2& r) { fp2_zero(r); }
HB_DEV void f_one(fp2& r) { fp2_one(r); }
HB_DEV void f_cmov(fp2& r, const fp2& a, bool c) { fp2_cmov(r, a, c); }

// lane-pair carrier (tower.cuh fp2h): the same point arithmetic with every Fp2 coordinate split over two lanes
HB_DEV void f_add(fp2h& r, const fp2h& a, const fp2h& b) { fp2_add(r, a, b); }
HB_DEV void f_sub(fp2h& r, const fp2h& a, const fp2h& b) { fp2_sub(r, a, b); }
HB_DEV void f_dbl(fp2h& r, const fp2h& a) { fp2_dbl(r, a); }
HB_DEV void f_neg(fp2h& r, const fp2h& a) { fp2_neg(r, a); }
HB_DEV void f_mul(fp2h& r, const fp2h& a, const fp2h& b) { fp2_mul(r, a, b); }
HB_DEV void f_sqr(fp2h& r, const fp2h& a) { fp2_sqr(r, a); }
HB_DEV void f_inv(fp2h& r, const fp2h& a) { fp2_inv(r, a); }
HB_DEV bool f_is_zero(const fp2h& a) { return fp2_is_zero(a); }
HB_DEV bool f_eq(const fp2h& a, const fp2h& b) { return fp2_eq(a, b); }
HB_DEV void f_zero(fp2h& r) { fp2_zero(r); }
HB_DEV void f_one(fp2h& r) { fp2_one(r); }
HB_DEV void f_cmov(fp2h& r, const fp2h& a, bool c) { fp2_cmov(r, a, c); }

template <class F> struct jac { F x, y, z; };     // Jacobian: (X/Z^2, Y/Z^3); z == 0 <=> identity
template <class F> struct aff { F x, y; };        // affine; x == y == 0 encodes the identity (not on either curve)
typedef jac<fp> g1; typedef jac<fp2> g2;
typedef aff<fp> g1a; typedef aff<fp2> g2a;

template <class F> HB_DEV bool pt_is_inf(const jac<F>& p) { return f_is_zero(p.z); }
template <class F> HB_DEV void pt_set_inf(jac<F>& p) { f_zero(p.x); f_zero(p.y); f_zero(p.z); }
template <class F> HB_DEV void pt_neg(jac<F>& r, const jac<F>& p) { r.x = p.x; f_neg(r.y, p.y); r.z = p.z; }
template <class F> HB_DEV bool aff_is_inf(const aff<F>& p) { return f_is_zero(p.x) && f_is_zero(p.y); }
template <class F> HB_DEV void pt_from_aff(jac<F>& r, const aff<F>& a) {
    if (aff_is_inf(a)) { pt_set_inf(r); return; }
    r.x = a.x; r.y = a.y; f_one(r.z);
}

template <class F> HB_NOINLINE void pt_dbl(jac<F>& r, const jac<F>& p) {
    if (pt_is_inf(p)) { pt_set_inf(r); return; }
    F A, B, C, D, E, Fq, t;
    f_sqr(A, p.x); f_sqr(B, p.y); f_sqr(C, B);
    f_add(D, p.x, B); f_sqr(D, D); f_sub(D, D, A); f_sub(D, D, C); f_dbl(D, D);
    f_dbl(E, A); f_add(E, E, A);
    f_sqr(Fq, E);
    f_mul(t, p.y, p.z); f_dbl(r.z, t);
    f_dbl(t, D); f_sub(r.x, Fq, t);
    f_sub(t, D, r.x); f_mul(t, t, E);
    f_dbl(C, C); f_dbl(C, C); f_dbl(C, C);
    f_sub(r.y, t, C);
}

template <class F> HB_NOINLINE void pt_add(jac<F>& r, const jac<F>& p, const jac<F>& q) {
    if (pt_is_inf(p)) { r = q; return; }
    if (pt_is_inf(q)) { r = p; return; }
    F Z1Z1, Z2Z2, U1, U2, S1, S2, H, R, HH, HHH, V, t;
    f_sqr(Z1Z1, p.z); f_sqr(Z2Z2, q.z);
    f_mul(U1, p.x, Z2Z2); f_mul(U2, q.x, Z1Z1);
    f_mul(S1, p.y, q.z); f_mul(S1, S1, Z2Z2);
    f_mul(S2, q.y, p.z); f_mul(S2, S2, Z1Z1);
    f_sub(H, U2, U1); f_sub(R, S2, S1);
    if (f_is_zero(H)) {
        if (f_is_zero(R)) { pt_dbl(r, p); return; }
        pt_set_inf(r); return;
    }
    f_sqr(HH, H); f_mul(HHH, H, HH); f_mul(V, U1, HH);
    f_mul(t, p.z, q.z); f_mul(r.z, t, H);
    f_sqr(t, R); f_sub(t, t, HHH); f_sub(t, t, V); f_sub(r.x, t, V);
    f_sub(t, V, r.x); f_mul(t, t, R); f_mul(S1, S1, HHH); f_sub(r.y, t, S1);
}

// r = p + q with q affine (the committee table is stored affine: 8 M + 3 S instead of 12 M + 4 S)
template <class F> HB_NOINLINE void pt_add_mixed(jac<F>& r, const jac<F>& p, const aff<F>& q) {
    if (aff_is_inf(q)) { r = p; return; }
    if (pt_is_inf(p)) { r.x = q.x; r.y = q.y; f_one(r.z); return; }
    F Z1Z1, U2, S2, H, R, HH, HHH, V, t;
    f_sqr(Z1Z1, p.z);
    f_mul(U2, q.x, Z1Z1);
    f_mul(S2, q.y, p.z); f_mul(S2, S2, Z1Z1);
    f_sub(H, U2, p.x); f_sub(R, S2, p.y);
    if (f_is_zero(H)) {
        if (f_is_zero(R)) { pt_dbl(r, p); return; }
        pt_set_inf(r); return;
    }
    f_sqr(HH, H); f_mul(HHH, H, HH); f_mul(V, p.x, HH);
    F y1 = p.y;
    f_mul(r.z, p.z, H);
    f_sqr(t, R); f_sub(t, t, HHH); f_sub(t, t, V); f_sub(r.x, t, V);
    f_sub(t, V, r.x); f_mul(t, t, R); f_mul(y1, y1, HHH); f_sub(r.y, t, y1);
}

template <class F> HB_NOINLINE bool pt_eq(const jac<F>& p, const jac<F>& q) {
    if (pt_is_inf(p) || pt_is_inf(q)) return pt_is_inf(p) && pt_is_inf(q);
    F Z1Z1, Z2Z2, a, b;
    f_sqr(Z1Z1, p.z); f_sqr(Z2Z2, q.z);
    f_mul(a, p.x, Z2Z2); f_mul(b, q.x, Z1Z1);
    if (!f_eq(a, b)) return false;
    f_mul(a, p.y, q.z); f_mul(a, a, Z2Z2);
    f_mul(b, q.y, p.z); f_mul(b, b, Z1Z1);
    return f_eq(a, b);
}

// no branch for the identity: 1/0 = 0 here (a^(p-2)), so it maps to (0, 0) like the affine identity.  With an early return for
// it, the sm_90a build returned wrong affine points for the OTHER lanes of a warp that held one identity (a batch of triples
// with an undecodable key then rejected its 31 neighbours: tests/test_gpu_parity.py::test_config4_*); the cost is one
// inversion for an identity input, which honest input never has.
template <class F> HB_NOINLINE void pt_to_aff(aff<F>& r, const jac<F>& p) {
    F zi, zi2;
    f_inv(zi, p.z); f_sqr(zi2, zi);
    f_mul(r.x, p.x, zi2); f_mul(zi2, zi2, zi); f_mul(r.y, p.y, zi2);
}

// Montgomery's trick over K elements held by ONE thread: z[k] <- 1/z[k] with a single inversion (3 (K - 1) extra products);
// entries flagged skip are left untouched.  A persistent thread that handles several items in turn shares their inversions.
template <class F, int K> HB_NOINLINE void f_batch_inv(F* z, const bool* skip) {
    F pre[K], acc; f_one(acc);
    for (int k = 0; k < K; k++) { pre[k] = acc; if (!skip[k]) f_mul(acc, acc, z[k]); }
    F inv; f_inv(inv, acc);
    for (int k = K - 1; k >= 0; k--) if (!skip[k]) { F t; f_mul(t, inv, pre[k]); f_mul(inv, inv, z[k]); z[k] = t; }
}
// affine form of p given zi = 1 / p.z (identity -> the all-zero encoding)
template <class F> HB_DEV void pt_to_aff_zinv(aff<F>& r, const jac<F>& p, const F& zi) {
    if (pt_is_inf(p)) { f_zero(r.x); f_zero(r.y); return; }
    F zi2; f_sqr(zi2, zi);
    f_mul(r.x, p.x, zi2); f_mul(zi2, zi2, zi); f_mul(r.y, p.y, zi2);
}

// r = [k]p, k = nw little-endian 32-bit words; 4-bit fixed window, uniform control flow
template <class F> HB_NOINLINE void pt_mul(jac<F>& r, const jac<F>& p, const uint32_t* k, int nw) {
    jac<F> tbl[16];
    pt_set_inf(tbl[0]); tbl[1] = p;
    for (int i = 2; i < 16; i++) pt_add(tbl[i], tbl[i - 1], p);
    jac<F> acc; pt_set_inf(acc);
    for (int i = nw * 8 - 1; i >= 0; i--) {
        uint32_t w = (k[i >> 3] >> (4 * (i & 7))) & 15u;
        pt_dbl(acc, acc); pt_dbl(acc, acc); pt_dbl(acc, acc); pt_dbl(acc, acc);
        if (w) pt_add(acc, acc, tbl[w]);
    }
    r = acc;
}
// r = [|z|]p, |z| = 0xd201000000010000 (sparse: 63 doublings + 5 additions)
template <class F> HB_NOINLINE void pt_mul_zabs(jac<F>& r, const jac<F>& p) {
    jac<F> acc = p;
    for (int i = 62; i >= 0; i--) {
        HB_USYNC();
        pt_dbl(acc, acc);
        if ((K_Z_ABS >> i) & 1) pt_add(acc, acc, p);
    }
    r = acc;
}
// the same ladder for an affine base: mixed additions (8 M + 3 S instead of 12 M + 4 S).  The all-zero encoding gives the identity,
// acc == +-p takes pt_add_mixed's doubling / identity branches as pt_add's, so the result is the group element pt_mul_zabs gives.
template <class F> HB_NOINLINE void pt_mul_zabs_aff(jac<F>& r, const aff<F>& p) {
    jac<F> acc; pt_from_aff(acc, p);
    for (int i = 62; i >= 0; i--) {
        HB_USYNC();
        pt_dbl(acc, acc);
        if ((K_Z_ABS >> i) & 1) pt_add_mixed(acc, acc, p);
    }
    r = acc;
}

// r = [k]p for a 64-bit k (random-linear-combination coefficients): plain MSB-first double-and-add
template <class F> HB_NOINLINE void pt_mul_u64(jac<F>& r, const jac<F>& p, uint64_t k) {
    jac<F> acc; pt_set_inf(acc);
    for (int i = 63; i >= 0; i--) { pt_dbl(acc, acc); if ((k >> i) & 1) pt_add(acc, acc, p); }
    r = acc;
}
template <class F> HB_NOINLINE void pt_mul_u64_aff(jac<F>& r, const aff<F>& p, uint64_t k) {
    jac<F> acc; pt_set_inf(acc);
    for (int i = 63; i >= 0; i--) { pt_dbl(acc, acc); if ((k >> i) & 1) pt_add_mixed(acc, acc, p); }
    r = acc;
}

// [a + b lambda] P from P and P2 = [lambda] P with one shared 32-step ladder (a, b 32-bit): 32 doublings + <= 32 additions
template <class F> HB_NOINLINE void pt_mul_2d(jac<F>& r, const jac<F>& p, const jac<F>& p2, uint32_t a, uint32_t b) {
    jac<F> t; pt_add(t, p, p2);
    jac<F> acc; pt_set_inf(acc);
    for (int i = 31; i >= 0; i--) {
        HB_USYNC();
        pt_dbl(acc, acc);
        const int sel = ((a >> i) & 1) | (((b >> i) & 1) << 1);
        if (sel) pt_add(acc, acc, sel == 1 ? p : (sel == 2 ? p2 : t));
    }
    r = acc;
}
template <class F> HB_NOINLINE void pt_mul_2d_aff(jac<F>& r, const aff<F>& p, const aff<F>& p2, uint32_t a, uint32_t b) {
    jac<F> t; pt_from_aff(t, p); pt_add_mixed(t, t, p2);
    jac<F> acc; pt_set_inf(acc);
    for (int i = 31; i >= 0; i--) {
        HB_USYNC();
        pt_dbl(acc, acc);
        const int sel = ((a >> i) & 1) | (((b >> i) & 1) << 1);
        if (sel == 3) pt_add(acc, acc, t);
        else if (sel) pt_add_mixed(acc, acc, sel == 1 ? p : p2);
    }
    r = acc;
}

// ---- the same two-base ladders over the JOINT SPARSE FORM of (a, b) (Solinas): signed digits u0_i, u1_i in {-1, 0, 1}, <= 33 digit
// pairs of which on average 16.8 are non-zero (24 of 32 for the plain binary pairs above) -- 6 additions fewer per ladder after the
// one extra table entry P - P2.  The digits depend on the coefficient only, which a warp's 32 rounds share: control flow stays uniform.
// Bit i of nz0 / ng0 (nz1 / ng1): digit i of a (of b) is non-zero / negative.  Returns the number of digits.
HB_DEV int jsf_pack(uint32_t a, uint32_t b, uint64_t& nz0, uint64_t& ng0, uint64_t& nz1, uint64_t& ng1) {
    uint64_t k0 = a, k1 = b; uint32_t d0 = 0, d1 = 0; int n = 0;
    nz0 = ng0 = nz1 = ng1 = 0;
    while (k0 + d0 != 0 || k1 + d1 != 0) {
        const uint32_t l0 = (uint32_t)((k0 + d0) & 7u), l1 = (uint32_t)((k1 + d1) & 7u);
        int u0 = 0, u1 = 0;
        if (l0 & 1u) { u0 = (l0 & 3u) == 1u ? 1 : -1; if ((l0 == 3u || l0 == 5u) && (l1 & 3u) == 2u) u0 = -u0; }
        if (l1 & 1u) { u1 = (l1 & 3u) == 1u ? 1 : -1; if ((l1 == 3u || l1 == 5u) && (l0 & 3u) == 2u) u1 = -u1; }
        if (2 * (int)d0 == 1 + u0) d0 = 1u - d0;
        if (2 * (int)d1 == 1 + u1) d1 = 1u - d1;
        k0 >>= 1; k1 >>= 1;
        if (u0) { nz0 |= 1ull << n; if (u0 < 0) ng0 |= 1ull << n; }
        if (u1) { nz1 |= 1ull << n; if (u1 < 0) ng1 |= 1ull << n; }
        n++;
    }
    return n;
}
template <class F> HB_NOINLINE void pt_mul_2d_jsf(jac<F>& r, const jac<F>& p, const jac<F>& p2, uint32_t a, uint32_t b) {
    uint64_t nz0, ng0, nz1, ng1; const int n = jsf_pack(a, b, nz0, ng0, nz1, ng1);
    jac<F> t, m, q; pt_add(t, p, p2); pt_neg(q, p2); pt_add(m, p, q);          // P + P2, P - P2
    jac<F> acc; pt_set_inf(acc);
    for (int i = n - 1; i >= 0; i--) {
        HB_USYNC();
        pt_dbl(acc, acc);
        const bool z0 = (nz0 >> i) & 1, z1 = (nz1 >> i) & 1, n0 = (ng0 >> i) & 1, n1 = (ng1 >> i) & 1;
        if (!z0 && !z1) continue;
        // +-P, +-P2, +-(P + P2) when the signs agree, +-(P - P2) when they differ; the overall sign is that of the a-digit (or of
        // the b-digit when a's is zero)
        const bool neg = z0 ? n0 : n1;
        q = (z0 && z1) ? (n0 == n1 ? t : m) : (z0 ? p : p2);
        if (neg) pt_neg(q, q);
        pt_add(acc, acc, q);
    }
    r = acc;
}
template <class F> HB_NOINLINE void pt_mul_2d_aff_jsf(jac<F>& r, const aff<F>& p, const aff<F>& p2, uint32_t a, uint32_t b) {
    uint64_t nz0, ng0, nz1, ng1; const int n = jsf_pack(a, b, nz0, ng0, nz1, ng1);
    jac<F> t, m, q; aff<F> w;
    pt_from_aff(t, p); pt_add_mixed(t, t, p2);
    w = p2; f_neg(w.y, w.y); pt_from_aff(m, p); pt_add_mixed(m, m, w);
    jac<F> acc; pt_set_inf(acc);
    for (int i = n - 1; i >= 0; i--) {
        HB_USYNC();
        pt_dbl(acc, acc);
        const bool z0 = (nz0 >> i) & 1, z1 = (nz1 >> i) & 1, n0 = (ng0 >> i) & 1, n1 = (ng1 >> i) & 1;
        if (!z0 && !z1) continue;
        const bool neg = z0 ? n0 : n1;
        if (z0 && z1) { q = n0 == n1 ? t : m; if (neg) pt_neg(q, q); pt_add(acc, acc, q); }
        else { w = z0 ? p : p2; if (neg) f_neg(w.y, w.y); pt_add_mixed(acc, acc, w); }
    }
    r = acc;
}

// ---- r = sum_t [k_t] P_t over N (affine point, 32-bit scalar) pairs with ONE shared accumulator (Straus): every k_t in non-adjacent
// form (<= 33 signed digits, 11.4 of them non-zero on average), so the N ladders share their 33 doublings and a non-zero digit costs
// one mixed addition of +-P_t.  load(t, q) yields P_t and is called once per non-zero digit: no table, no Jacobian temporaries.  The
// digits depend on the scalars alone, so callers whose warps share them stay divergence-free.  Exceptional sums (an identity P_t,
// acc == +-P_t) take pt_add_mixed's branches.
// NAF by bit operations: np - nm == k with np & nm == 0 and no two adjacent non-zero digits (bit i of np / nm: digit i is +1 / -1)
HB_DEV void naf_masks(uint32_t k, uint64_t& np, uint64_t& nm) {
    const uint64_t x = k, xh = x >> 1, x3 = x + xh, c = xh ^ x3;
    np = x3 & c; nm = xh & c;
}
template <class E, int N, class Load> HB_NOINLINE void pt_mul_joint_naf(jac<E>& r, const uint32_t* k, Load load) {
    jac<E> acc; pt_set_inf(acc);
    for (int i = 32; i >= 0; i--) {
        HB_USYNC();
        pt_dbl(acc, acc);
#pragma unroll 1
        for (int t = 0; t < N; t++) {
            uint64_t np, nm; naf_masks(k[t], np, nm);
            if ((((np | nm) >> i) & 1) == 0) continue;
            aff<E> q; load(t, q);
            if ((nm >> i) & 1) f_neg(q.y, q.y);
            pt_add_mixed(acc, acc, q);
        }
    }
    r = acc;
}

HB_DEV void g1_generator(g1& r) { fp_set(r.x, K_G1_X); fp_set(r.y, K_G1_Y); fp_one(r.z); }

// ------------------------------------------------------------------ endomorphisms and subgroup membership
// psi(x, y) = (conj(x) * cx, conj(y) * cy): acts as [p] (== [z] on G2); maps the all-zero identity to itself.  E = fp2 or fp2h.
template <class E> HB_DEV void g2_psi_aff(aff<E>& r, const aff<E>& a) {
    E t; fp2_conj(t, a.x); fp2_mul(r.x, t, fp2_k<E>(K_PSI_CX));
    fp2_conj(t, a.y); fp2_mul(r.y, t, fp2_k<E>(K_PSI_CY));
}
// Jacobian form: psi(X, Y, Z) = (conj(X) cx, conj(Y) cy, conj(Z)) -- no inversion.  E = fp2 or the lane-pair carrier fp2h.
template <class E> HB_DEV void g2_psi(jac<E>& r, const jac<E>& p) {
    E t; fp2_conj(t, p.x); fp2_mul(r.x, t, fp2_k<E>(K_PSI_CX));
    fp2_conj(t, p.y); fp2_mul(r.y, t, fp2_k<E>(K_PSI_CY));
    fp2_conj(r.z, p.z);
}
// psi^2(X, Y, Z) = (X * N(cx), -Y, Z)
template <class E> HB_DEV void g2_psi2(jac<E>& r, const jac<E>& p) {
    fp2_mul_fp(r.x, p.x, fp_k(K_PSI2_CX)); fp2_neg(r.y, p.y); r.z = p.z;
}

// ------------------------------------------------------------------ secret-scalar ladders (sign, GetPublicKey): constant time
// The sequence of field operations, every branch and every address depend only on public data (the point, the item count), never on
// the scalar: complete projective formulas (no identity / equal-point cases), a regular recoding whose digits are all non-zero, and
// table reads that load every entry and keep one by select.
// HB_CT_PROBE(tag) marks the formulas, the table reads and the ladder steps.  It compiles to nothing in the library; the constant-time
// tests build with HB_CT_PROBE_HOST (host emulation: a trace of tags) or HB_CT_PROBE_DEVICE (active mask and count per thread) and
// define hb_ct_probe themselves.
#if defined(HB_CT_PROBE_HOST) || defined(HB_CT_PROBE_DEVICE)
__device__ void hb_ct_probe(uint32_t tag);
#define HB_CT_PROBE(tag) hb_ct_probe(tag)
#else
#define HB_CT_PROBE(tag) ((void)0)
#endif
enum { CT_ADD = 1, CT_DBL, CT_READ, CT_STEP, CT_GLS_STEP };

template <class F> struct prj { F x, y, z; };     // homogeneous projective: (X/Z, Y/Z); identity (0 : 1 : 0)

// 3b x by additions: b = 4 on G1 (12 x); b' = 4 (1 + i) on G2 (12 (1 + i) x, the helper of the Miller doubling step)
HB_DEV void f_mul3b(fp& r, const fp& a) { fp t; fp_dbl(t, a); fp_add(t, t, a); fp_dbl(t, t); fp_dbl(r, t); }
HB_DEV void f_mul3b(fp2& r, const fp2& a) { fp2_mul_twist3b(r, a); }
HB_DEV void f_mul3b(fp2h& r, const fp2h& a) { fp2_mul_twist3b(r, a); }

// complete addition for y^2 = x^3 + b (Renes-Costello-Batina 2016, Algorithm 7): 12 M + 2 (x 3b), valid for every pair of points
// (the identity, P == Q, P == -Q included).  r may alias p or q.
template <class F> HB_NOINLINE void prj_add(prj<F>& r, const prj<F>& p, const prj<F>& q) {
    HB_CT_PROBE(CT_ADD);
    F t0, t1, t2, t3, t4, x3, y3, z3;
    f_mul(t0, p.x, q.x); f_mul(t1, p.y, q.y); f_mul(t2, p.z, q.z);
    f_add(t3, p.x, p.y); f_add(t4, q.x, q.y); f_mul(t3, t3, t4);
    f_add(t4, t0, t1); f_sub(t3, t3, t4);                                   // X1 Y2 + X2 Y1
    f_add(t4, p.y, p.z); f_add(x3, q.y, q.z); f_mul(t4, t4, x3);
    f_add(x3, t1, t2); f_sub(t4, t4, x3);                                   // Y1 Z2 + Y2 Z1
    f_add(x3, p.x, p.z); f_add(y3, q.x, q.z); f_mul(x3, x3, y3);
    f_add(y3, t0, t2); f_sub(y3, x3, y3);                                   // X1 Z2 + X2 Z1
    f_dbl(x3, t0); f_add(t0, x3, t0);                                       // 3 X1 X2
    f_mul3b(t2, t2);
    f_add(z3, t1, t2); f_sub(t1, t1, t2);
    f_mul3b(y3, y3);
    f_mul(x3, t4, y3); f_mul(t2, t3, t1); f_sub(x3, t2, x3);
    f_mul(y3, y3, t0); f_mul(t1, t1, z3); f_add(y3, t1, y3);
    f_mul(t0, t0, t3); f_mul(z3, z3, t4); f_add(z3, z3, t0);
    r.x = x3; r.y = y3; r.z = z3;
}
// complete doubling (Algorithm 9): 6 M + 2 S + 1 (x 3b)
template <class F> HB_NOINLINE void prj_dbl(prj<F>& r, const prj<F>& p) {
    HB_CT_PROBE(CT_DBL);
    F t0, t1, t2, x3, y3, z3;
    f_sqr(t0, p.y); f_dbl(z3, t0); f_dbl(z3, z3); f_dbl(z3, z3);           // 8 Y^2
    f_mul(t1, p.y, p.z); f_sqr(t2, p.z);
    f_mul3b(t2, t2);
    f_mul(x3, t2, z3); f_add(y3, t0, t2);
    f_mul(z3, t1, z3);
    f_dbl(t1, t2); f_add(t2, t1, t2);
    f_sub(t0, t0, t2); f_mul(y3, t0, y3); f_add(y3, x3, y3);
    f_mul(t1, p.x, p.y); f_mul(x3, t0, t1); f_dbl(x3, x3);
    r.x = x3; r.y = y3; r.z = z3;
}
template <class F> HB_DEV void prj_set_inf(prj<F>& r) { f_zero(r.x); f_one(r.y); f_zero(r.z); }
// Jacobian (X/Z^2, Y/Z^3) -> (X Z : Y : Z^3); the all-zero identity -> (0 : 1 : 0).  Only for public points (the base of a ladder).
template <class F> HB_DEV void prj_from_jac(prj<F>& r, const jac<F>& p) {
    F z2, one; f_sqr(z2, p.z); f_mul(r.x, p.x, p.z); f_mul(r.z, z2, p.z); r.y = p.y;
    f_one(one); f_cmov(r.y, one, pt_is_inf(p));
}
// (X : Y : Z) -> Jacobian (X Z, Y Z^2, Z) by products only; the identity (0 : Y : 0) lands on the all-zero struct
template <class F> HB_DEV void prj_to_jac(jac<F>& r, const prj<F>& p) {
    F z2; f_sqr(z2, p.z); f_mul(r.x, p.x, p.z); f_mul(r.y, p.y, z2); r.z = p.z;
}
template <class F> HB_DEV void pt_cmov(prj<F>& r, const prj<F>& a, bool c) { f_cmov(r.x, a.x, c); f_cmov(r.y, a.y, c); f_cmov(r.z, a.z, c); }
// r = -r when c, by select
template <class F> HB_DEV void pt_cneg_ct(prj<F>& r, bool c) { F n; f_neg(n, r.y); f_cmov(r.y, n, c); }
// r = t[i]: every entry is read, the one wanted is kept by select (the index never forms an address)
template <class F, int N> HB_DEV void pt_select_ct(prj<F>& r, const prj<F>* t, uint32_t i) {
    HB_CT_PROBE(CT_READ);
    r = t[0];
#pragma unroll 1
    for (int j = 1; j < N; j++) pt_cmov(r, t[j], (uint32_t)j == i);
}

// r = [k]p for any 256-bit k (8 little-endian 32-bit words), in constant time.  k is made odd (k' = k | 1) and recoded into 64 odd
// signed digits of 4 bits, k' = sum_i d_i 16^i: d_i = ((bits 4i .. 4i+4 of k') | 1) - 16 for i < 63, d_63 = (k' >> 252) | 1 (the
// recurrence k_{i+1} = (k_i - d_i) / 16 = (k_i >> 4) | 1).  Table of the odd multiples P, 3P, .., 15P; per window 4 doublings and one
// addition of the selected, conditionally negated entry; the closing addition adds -P when k was even and the identity otherwise, so
// k = 0 and k = r - 1 need no special case.  252 doublings + 64 additions + the table, whatever k.
template <class F> HB_NOINLINE void pt_mul_ct(jac<F>& r, const jac<F>& p, const uint32_t* k) {
    prj<F> P, T[8], acc, q;
    prj_from_jac(P, p);
    T[0] = P; prj_dbl(q, P);
#pragma unroll 1
    for (int j = 1; j < 8; j++) prj_add(T[j], T[j - 1], q);
    const bool even = (k[0] & 1u) == 0;
    uint32_t kk[9];
    for (int j = 0; j < 8; j++) kk[j] = k[j];
    kk[0] |= 1u; kk[8] = 0;
    pt_select_ct<F, 8>(acc, T, ((kk[7] >> 28) | 1u) >> 1);                  // d_63 > 0: entry (d_63 - 1) / 2
#pragma unroll 1
    for (int i = 62; i >= 0; i--) {
        HB_CT_PROBE(CT_STEP);
        prj_dbl(acc, acc); prj_dbl(acc, acc); prj_dbl(acc, acc); prj_dbl(acc, acc);
        const int b = 4 * i;
        const uint32_t w = ((uint32_t)((((uint64_t)kk[(b >> 5) + 1] << 32) | kk[b >> 5]) >> (b & 31)) & 31u) | 1u;     // d_i + 16
        const uint32_t neg = ((w >> 4) & 1u) ^ 1u;                           // d_i < 0
        pt_select_ct<F, 8>(q, T, ((w ^ (15u * neg)) & 15u) >> 1);             // |d_i| = 2 entry + 1
        pt_cneg_ct(q, neg != 0);
        prj_add(acc, acc, q);
    }
    prj_set_inf(q);
    prj<F> m = T[0]; pt_cneg_ct(m, true); pt_cmov(q, m, even);
    prj_add(acc, acc, q);
    prj_to_jac(r, acc);
}

// r = sk H on G2 from the base-Z digits of sk = d0 + d1 Z + d2 Z^2 + d3 Z^3 (d_j < Z = |z| < 2^64), in constant time.  psi acts as
// [z] = [-Z], so sk H = d0 P0 + d1 P1 + d2 P2 + d3 P3 with P0 = H, P1 = -psi(H), P2 = psi^2(H), P3 = -psi^3(H).  Sign-aligned column
// recoding (GLV-SAC, Faz-Hernandez, Longa, Sanchez 2014): with d0 odd, column i has the sign s_i = 2 bit_{i+1}(d0) - 1 (s_64 = +1) and
// adds s_i (P0 + sum_j c_ij P_j), c_ij = the low bit of d_j after the earlier columns took theirs (d_j <- (d_j - s_i c_ij) / 2).  The
// eight sums P0 + {0,1} P1 + {0,1} P2 + {0,1} P3 form the table; 65 columns of one doubling and one addition each.  d0 is made odd
// (d0 | 1) and the closing addition adds -H when it was even, the identity otherwise.  h is the affine H (public); E = fp2 or fp2h.
template <class E> HB_NOINLINE void g2_mul_gls_ct(jac<E>& r, const aff<E>& h, const uint64_t* d) {
    jac<E> B[4];                                                              // P0..P3; every one has Z = 1, so it is its own
    B[0].x = h.x; B[0].y = h.y; f_one(B[0].z);                                // projective form too
    g2_psi(B[1], B[0]); pt_neg(B[1], B[1]);
    g2_psi2(B[2], B[0]);
    g2_psi(B[3], B[2]); pt_neg(B[3], B[3]);
    prj<E> Pj[4], T[8], acc, q;
    for (int j = 0; j < 4; j++) { Pj[j].x = B[j].x; Pj[j].y = B[j].y; Pj[j].z = B[j].z; }
    T[0] = Pj[0];
#pragma unroll 1
    for (int u = 1; u < 8; u++) { const int top = u >= 4 ? 4 : u >= 2 ? 2 : 1; prj_add(T[u], T[u - top], Pj[top == 4 ? 3 : top]); }
    const bool even = (d[0] & 1u) == 0;
    uint64_t s = (d[0] | 1u) >> 1, k1 = d[1], k2 = d[2], k3 = d[3];
    uint8_t col[65];                                                          // bits 0-2: table entry, bit 3: negative column
#pragma unroll 1
    for (int i = 0; i < 65; i++) {
        const uint32_t pos = (uint32_t)(s & 1u) | (i == 64 ? 1u : 0u); s >>= 1;
        const uint32_t c1 = (uint32_t)(k1 & 1u), c2 = (uint32_t)(k2 & 1u), c3 = (uint32_t)(k3 & 1u), ng = pos ^ 1u;
        k1 = (k1 >> 1) + (c1 & ng); k2 = (k2 >> 1) + (c2 & ng); k3 = (k3 >> 1) + (c3 & ng);
        col[i] = (uint8_t)(c1 | c2 << 1 | c3 << 2 | ng << 3);
    }
    prj_set_inf(acc);
#pragma unroll 1
    for (int i = 64; i >= 0; i--) {
        HB_CT_PROBE(CT_GLS_STEP);
        prj_dbl(acc, acc);
        pt_select_ct<E, 8>(q, T, col[i] & 7u);
        pt_cneg_ct(q, (col[i] >> 3) != 0);
        prj_add(acc, acc, q);
    }
    prj_set_inf(q);
    prj<E> m = Pj[0]; pt_cneg_ct(m, true); pt_cmov(q, m, even);
    prj_add(acc, acc, q);
    prj_to_jac(r, acc);
}
// Q in G2  <=>  psi(Q) == [z]Q   (same boolean as [r]Q == O; SURVEY A.5)
template <class E> HB_NOINLINE bool g2_in_subgroup(const jac<E>& p) {
    if (pt_is_inf(p)) return true;
    jac<E> a, b; g2_psi(a, p); pt_mul_zabs(b, p); pt_neg(b, b);
    return pt_eq(a, b);
}
// the same test of an affine point (the all-zero identity passes): the ladder adds its affine base with mixed additions
template <class E> HB_NOINLINE bool g2_in_subgroup_aff(const aff<E>& p) {
    if (aff_is_inf(p)) return true;
    aff<E> q; g2_psi_aff(q, p);
    jac<E> a, b; pt_from_aff(a, q); pt_mul_zabs_aff(b, p); pt_neg(b, b);
    return pt_eq(a, b);
}
// P in G1  <=>  phi(P) == -[z^2]P, phi(x, y) = (beta x, y)
HB_NOINLINE bool g1_in_subgroup(const g1& p) {
    if (pt_is_inf(p)) return true;
    g1 a = p, b;
    pt_mul_zabs(b, p); pt_mul_zabs(b, b); pt_neg(b, b);
    fp_mul(a.x, a.x, fp_k(K_BETA));
    return pt_eq(a, b);
}

// Batch-verification coefficient applied to one round: the 64-bit draw c = (b << 32 | a) stands for the scalar
// s = a + b z^2 (mod r) -- 2^63 distinct values (a is forced odd), and [z^2] is an endomorphism on both groups:
//   G1: [z^2](x, y) = -phi(x, y) = (beta x, -y)      (g1_in_subgroup above: phi = -[z^2])
//   G2: [z^2] = psi^2,  psi^2(x, y) = (N(cx) x, -y)   (psi = [p] = [z] on G2)
// so both scalings are 32-step two-base ladders instead of 64-step ones.  Inputs must lie in G1 / G2 (the callers'
// points are sums of subgroup-checked keys and subgroup-checked signatures).
#ifndef HB_JSF
#define HB_JSF 1
#endif
HB_DEV void rlc_scale_g1(g1& ra, const g1& apk, uint64_t c) {
    const uint32_t a = (uint32_t)c | 1u, b = (uint32_t)(c >> 32);
    g1 p2;
    fp_mul(p2.x, apk.x, fp_k(K_BETA)); fp_neg(p2.y, apk.y); p2.z = apk.z;
#if HB_JSF
    pt_mul_2d_jsf(ra, apk, p2, a, b);
#else
    pt_mul_2d(ra, apk, p2, a, b);
#endif
}
template <class E> HB_DEV void rlc_scale_g2(jac<E>& rs, const aff<E>& sig, uint64_t c) {
    const uint32_t a = (uint32_t)c | 1u, b = (uint32_t)(c >> 32);
    aff<E> q2;
    fp2_mul_fp(q2.x, sig.x, fp_k(K_PSI2_CX)); fp2_neg(q2.y, sig.y);
#if HB_JSF
    pt_mul_2d_aff_jsf(rs, sig, q2, a, b);
#else
    pt_mul_2d_aff(rs, sig, q2, a, b);
#endif
}
HB_DEV void rlc_scale_pair(g1& ra, g2& rs, const g1& apk, const g2a& sig, uint64_t c) { rlc_scale_g1(ra, apk, c); rlc_scale_g2(rs, sig, c); }

// ------------------------------------------------------------------ codecs (SURVEY A.5; reference crypto/bls/bls.go:67-71,109-118)
// bytes are little-endian; the 12 u32 words of a canonical coordinate ARE its 48 bytes on this little-endian target
// serialized inputs sit in the library's own device buffers (256-byte aligned, item strides 32 / 48 / 96 bytes): word loads
// (LDG.E, vectorised by the compiler when n is a constant); unaligned caller pointers (device-pointer entry) fall back to bytes
HB_DEV void load_words(uint32_t* w, const uint8_t* b, int n) {
    if ((reinterpret_cast<uintptr_t>(b) & 3u) == 0) {
        const uint32_t* p = reinterpret_cast<const uint32_t*>(b);
        for (int i = 0; i < n; i++) w[i] = p[i];
        return;
    }
    for (int i = 0; i < n; i++) w[i] = (uint32_t)b[4 * i] | ((uint32_t)b[4 * i + 1] << 8) | ((uint32_t)b[4 * i + 2] << 16) | ((uint32_t)b[4 * i + 3] << 24);
}
HB_DEV void store_words(uint8_t* b, const uint32_t* w, int n) {
    for (int i = 0; i < n; i++) { b[4 * i] = (uint8_t)w[i]; b[4 * i + 1] = (uint8_t)(w[i] >> 8); b[4 * i + 2] = (uint8_t)(w[i] >> 16); b[4 * i + 3] = (uint8_t)(w[i] >> 24); }
}
HB_DEV bool fp_is_odd(const fp& a) { fp v; fp_to_int(v, a); return v.l[0] & 1u; }

HB_NOINLINE void g1_serialize(uint8_t* out, const g1& p) {
    if (pt_is_inf(p)) { for (int i = 0; i < 48; i++) out[i] = 0; return; }
    g1a a; pt_to_aff(a, p);
    fp v; fp_to_int(v, a.x); store_words(out, v.l, 12);
    if (fp_is_odd(a.y)) out[47] |= 0x80;
}
// returns false on: coordinate >= p, x not on curve, (check_order) not in the r-torsion
HB_NOINLINE bool g1_deserialize(g1& r, const uint8_t* in, bool check_order) {
    fp v; load_words(v.l, in, 12);
    if (fp_is_zero(v)) { pt_set_inf(r); return true; }
    bool odd = (v.l[11] >> 31) != 0; v.l[11] &= 0x7fffffffu;
    if (fp_int_geq_p(v)) return false;
    fp x, y, t;
    fp_from_int(x, v);
    fp_sqr(t, x); fp_mul(t, t, x); fp_add(t, t, fp_k(K_B1));
    if (!fp_sqrt(y, t)) return false;
    if (fp_is_odd(y) != odd) fp_neg(y, y);
    g1 q; q.x = x; q.y = y; fp_one(q.z);
    if (check_order && !g1_in_subgroup(q)) return false;
    r = q;
    return true;
}
HB_NOINLINE void g2_serialize(uint8_t* out, const g2& p) {
    if (pt_is_inf(p)) { for (int i = 0; i < 96; i++) out[i] = 0; return; }
    g2a a; pt_to_aff(a, p);
    fp v; fp_to_int(v, a.x.a); store_words(out, v.l, 12);
    fp_to_int(v, a.x.b); store_words(out + 48, v.l, 12);
    if (fp_is_odd(a.y.a)) out[95] |= 0x80;
}
HB_NOINLINE bool g2_deserialize(g2& r, const uint8_t* in, bool check_order) {
    fp va, vb; load_words(va.l, in, 12); load_words(vb.l, in + 48, 12);
    if (fp_is_zero(va) && fp_is_zero(vb)) { pt_set_inf(r); return true; }
    bool odd = (vb.l[11] >> 31) != 0; vb.l[11] &= 0x7fffffffu;
    if (fp_int_geq_p(va) || fp_int_geq_p(vb)) return false;
    fp2 x, y, t;
    fp_from_int(x.a, va); fp_from_int(x.b, vb);
    fp2_sqr(t, x); fp2_mul(t, t, x); fp2_add(t, t, fp2_k(K_B2));
    if (!fp2_sqrt_anysign(y, t)) return false;                    // the parity bit picks the sign below
    if (fp_is_odd(y.a) != odd) fp2_neg(y, y);
    g2 q; q.x = x; q.y = y; fp2_one(q.z);
    if (check_order && !g2_in_subgroup(q)) return false;
    r = q;
    return true;
}

// ------------------------------------------------------------------ message -> G2 (SURVEY A.3; SignHash/VerifyHash of the reference)
// mcl Fp::setArrayMask: first min(len, 48) bytes little-endian, masked to 381 bits, to 380 if still >= p
HB_DEV void hash_to_fp(fp& t, const uint8_t* msg, uint32_t len) {
    uint8_t b[48];
    uint32_t n = len > 48 ? 48 : len;
    for (uint32_t i = 0; i < 48; i++) b[i] = i < n ? msg[i] : 0;
    fp v; load_words(v.l, b, 12);
    v.l[11] &= 0x1fffffffu;
    if (fp_int_geq_p(v)) v.l[11] &= 0x0fffffffu;
    fp_from_int(t, v);
}
// mcl MapTo::calcBN over Fp2 (Shallue-van de Woestijne / Fouque-Tibouchi); false when the map is undefined (t = 0)
// GCD = true: the one inversion of the map by binary GCD (latency path)
template <bool GCD = false> HB_NOINLINE bool sw_map_g2(g2& r, const fp2& t) {
    if (fp2_is_zero(t)) return false;
    fp n; fp2 w, x, y, g;
    const fp &c1 = fp_k(K_SW_C1), &c2 = fp_k(K_SW_C2), &one = fp_k(K_ONE); const fp2& bb = fp2_k(K_B2);
    // negative = Legendre(N(t)) < 0.  SignHash / VerifyHash always map t = (t0, 0): N(t) = t0^2 is a square, so the
    // exponentiation is skipped for them (uniform branch); the general case keeps mcl's rule.
    bool negative = false;
    if (!fp_is_zero(t.b)) { fp2_norm(n, t); negative = fp_legendre(n) < 0; }
    // Same candidates and same "first x_i with x_i^3 + b square" rule as mcl, but with warp-uniform control flow:
    // one shared inversion (u * c1 t)^-1 yields both w and 1/w, squareness of g(x_1), g(x_2) is decided by the
    // Legendre symbol of the Fp2 norm, and only ONE Fp2 square root (of the selected candidate) is taken.
    fp2 u, ct, d, x2, x3, g2v;
    fp2_sqr(u, t); fp2_add(u, u, bb); fp_add(u.a, u.a, one);        // u = t^2 + b + 1
    if (fp2_is_zero(u)) return false;
    fp2_mul_fp(ct, t, c1);                                          // c1 t
    fp2_mul(d, u, ct);
    if (GCD) fp2_inv_gcd(d, d); else fp2_inv(d, d);                 // (u c1 t)^-1
    fp2_sqr(w, ct); fp2_mul(w, w, d);                               // w = c1 t / u
    fp2_sqr(x3, u); fp2_mul(x3, x3, d); fp2_sqr(x3, x3); fp_add(x3.a, x3.a, one);   // x3 = 1 + 1/w^2
    fp2_mul(x, t, w); fp2_neg(x, x); fp_add(x.a, x.a, c2);          // x1 = c2 - t w
    fp2_neg(x2, x); fp_sub(x2.a, x2.a, one);                        // x2 = -x1 - 1
    fp2_sqr(g, x); fp2_mul(g, g, x); fp2_add(g, g, bb);
    fp2_sqr(g2v, x2); fp2_mul(g2v, g2v, x2); fp2_add(g2v, g2v, bb);
    fp n1, n2; fp2_norm(n1, g); fp2_norm(n2, g2v);
    const bool sq1 = fp_legendre(n1) >= 0, sq2 = fp_legendre(n2) >= 0;
    if (!sq1) {
        if (sq2) { x = x2; g = g2v; }
        else { x = x3; fp2_sqr(g, x); fp2_mul(g, g, x); fp2_add(g, g, bb); }
    }
    if (!fp2_sqrt(y, g)) return false;                              // cannot happen: one of the three is a square
    if (negative) fp2_neg(y, y);
    r.x = x; r.y = y; fp2_one(r.z);
    return true;
}
// The same map in two halves around its single Fp2 inversion, so that a thread which maps several messages in turn can share
// that inversion (f_batch_inv): pre() yields d = u * c1 t, post() continues from dinv = 1/d exactly as sw_map_g2 does.
HB_NOINLINE bool sw_map_g2_pre(fp2& u, fp2& ct, fp2& d, const fp2& t) {
    if (fp2_is_zero(t)) return false;
    const fp &c1 = fp_k(K_SW_C1), &one = fp_k(K_ONE); const fp2& bb = fp2_k(K_B2);
    fp2_sqr(u, t); fp2_add(u, u, bb); fp_add(u.a, u.a, one);
    if (fp2_is_zero(u)) return false;
    fp2_mul_fp(ct, t, c1);
    fp2_mul(d, u, ct);
    return true;
}
HB_NOINLINE bool sw_map_g2_post(g2& r, const fp2& t, const fp2& u, const fp2& ct, const fp2& dinv) {
    fp n; fp2 w, x, y, g;
    const fp &c2 = fp_k(K_SW_C2), &one = fp_k(K_ONE); const fp2& bb = fp2_k(K_B2);
    bool negative = false;
    if (!fp_is_zero(t.b)) { fp2_norm(n, t); negative = fp_legendre(n) < 0; }
    fp2 x2, x3, g2v;
    fp2_sqr(w, ct); fp2_mul(w, w, dinv);
    fp2_sqr(x3, u); fp2_mul(x3, x3, dinv); fp2_sqr(x3, x3); fp_add(x3.a, x3.a, one);
    fp2_mul(x, t, w); fp2_neg(x, x); fp_add(x.a, x.a, c2);
    fp2_neg(x2, x); fp_sub(x2.a, x2.a, one);
    fp2_sqr(g, x); fp2_mul(g, g, x); fp2_add(g, g, bb);
    fp2_sqr(g2v, x2); fp2_mul(g2v, g2v, x2); fp2_add(g2v, g2v, bb);
    fp n1, n2; fp2_norm(n1, g); fp2_norm(n2, g2v);
    const bool sq1 = fp_legendre(n1) >= 0, sq2 = fp_legendre(n2) >= 0;
    if (!sq1) {
        if (sq2) { x = x2; g = g2v; }
        else { x = x3; fp2_sqr(g, x); fp2_mul(g, g, x); fp2_add(g, g, bb); }
    }
    if (!fp2_sqrt(y, g)) return false;
    if (negative) fp2_neg(y, y);
    r.x = x; r.y = y; fp2_one(r.z);
    return true;
}
// Budroni-Pintore cofactor clearing: [z^2 - z - 1]P + psi([z - 1]P) + psi^2([2]P)   (plain h2 gives other bytes)
template <class E> HB_NOINLINE void g2_clear_cofactor(jac<E>& r, const jac<E>& p) {
    jac<E> zp, z2p, t1, t2, t3, np;
    pt_mul_zabs(zp, p); pt_neg(zp, zp);
    pt_mul_zabs(z2p, zp); pt_neg(z2p, z2p);
    pt_neg(np, p);
    pt_add(t1, z2p, np); pt_neg(t2, zp); pt_add(t1, t1, t2);
    pt_add(t2, zp, np); g2_psi(t2, t2);
    pt_dbl(t3, p); g2_psi2(t3, t3);
    pt_add(t1, t1, t2); pt_add(r, t1, t3);
}
// The same h(P) for an affine P, in the order of RFC 9380's clear_cofactor_bls12381_g2 (z < 0, so [z] = -[|z|]):
//   t1 = [z]P,  t2 = [z](t1 + psi(P)),  h(P) = t2 - t1 - psi(P) - P + psi^2(2P)
// (t2 = [z^2]P + psi([z]P), so this is the combination above), in two halves of one |z| ladder each so that each can run as a kernel
// of its own.  Three Jacobian points live at most, and every addend that is affine (P in the first ladder, psi(P), P) goes in by a
// mixed addition.  Same group element as g2_clear_cofactor for every point of E', torsion included (the group law's exceptional cases
// take their branches); the Jacobian representative may differ.
template <class E> HB_NOINLINE void g2_clear_cofactor_aff_z1(jac<E>& t1, const aff<E>& p) {
    pt_mul_zabs_aff(t1, p); pt_neg(t1, t1);
}
// h(P) from t1 = [z]P (g2_clear_cofactor_aff_z1) and P
template <class E> HB_NOINLINE void g2_clear_cofactor_aff_z2(jac<E>& r, const jac<E>& t1, const aff<E>& p) {
    jac<E> t2, t; aff<E> q;
    g2_psi_aff(q, p); pt_add_mixed(t2, t1, q);
    pt_mul_zabs(t2, t2); pt_neg(t2, t2);
    pt_neg(t, t1); pt_add(t2, t2, t);
    f_neg(q.y, q.y); pt_add_mixed(t2, t2, q);
    q = p; f_neg(q.y, q.y); pt_add_mixed(t2, t2, q);
    pt_from_aff(t, p); pt_dbl(t, t); g2_psi2(t, t);
    pt_add(r, t2, t);
}
HB_NOINLINE bool map_to_g2(g2& r, const uint8_t* msg, uint32_t len) {
    fp2 t; hash_to_fp(t.a, msg, len); fp_zero(t.b);
    g2 a; if (!sw_map_g2(a, t)) return false;
    g2_clear_cofactor(r, a); return true;
}

}  // namespace hb
