"""The field, tower and group-law primitives of csrc/, one at a time, against big-integer arithmetic (oracle/pyref.py).

Every op of tests/arith/arith_ops.cuh gets seeded random operands plus the edges where its carry chains, branches and lane-pair
exchanges go wrong: stored 0, 1, R mod p, p - 1, p - 2, (p +- 1) / 2, powers of two, all-ones limbs under a top limb below p_11,
alternating limbs, pairs summing to p - 1, p and p + 1, zero halves of Fp2 values, sparse and all-(p - 1) Fp12 values, identities,
P + P with different Z, P + (-P), and for the lane-pair verdicts a difference confined to one limb of one half of one coefficient.
Inputs and outputs are the STORED limbs (Montgomery form): an expected Fp result is f(values) R mod p, the 768-bit layer is
compared as raw integers.  Each op runs in each of its aliasing forms (distinct, r = x, r = y, x = y, r = x = y for binary ops;
distinct, r = x for unary ones), and the test asserts that the items reach both sides of every branch it restates (the
conditional subtraction of the Montgomery reduction, the carry / borrow of add / sub / half, the six outcomes of fp2_sqrt, the
five cases of pt_add, the trial subtractions of vm_lin).

CPU: the op table under the host emulation (tests/emu/emu_arith.cpp), the default build and the code switches that change the host
build.  GPU: the same table compiled for sm_90a with the library's own nvcc flags (tests/arith/arith_driver.cu), launched twice --
edge items scattered among the random ones so that both share warps, then sorted by class -- and once more under every
off-by-default code switch.  The host build keeps its carries in a variable and never sees NVVM's stack-slot assignment; this
is the per-primitive check of the device build (DESIGN.md section 6, "Toolchain notes")."""
import concurrent.futures, ctypes, os, random, subprocess, sys, tempfile
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "oracle"))
import pyref as o                                   # noqa: E402
from harmony_b200.build import NVCC_FLAGS           # noqa: E402

_BUILD = tempfile.mkdtemp(prefix="hbls_arith_")
P = o.P
R = 1 << 384
RINV = pow(R, -1, P)
ONE = R % P
NPRIME = (-pow(P, -1, R)) % R
P11 = P >> 352
MIN_HITS = 32                                       # items required on each side of every restated branch


def mont(v): return v % P * R % P
def val(s): return s * RINV % P


# ------------------------------------------------------------------ layouts: stored units (one Fp = 12 words) <-> values
SLOT_K = (0, 2, 4, 1, 3, 5)                         # fp12_slot: struct position j holds the coefficient of w^SLOT_K[j]

def F2(u, k): return (val(u[k]), val(u[k + 1]))
def F6(u, k): return tuple(F2(u, k + 2 * j) for j in range(3))
def F12(u, k):
    w = [None] * 6
    for j in range(6): w[SLOT_K[j]] = F2(u, k + 2 * j)
    return tuple(w)
def mF2(x): return [mont(x[0]), mont(x[1])]
def mF6(x): return [s for c in x for s in mF2(c)]
def mF12(w): return [s for j in range(6) for s in mF2(w[SLOT_K[j]])]
def w12_from_f6(a0, a1): return (a0[0], a1[0], a0[1], a1[1], a0[2], a1[2])      # (c0, c1) of Fp6 -> w powers


# ------------------------------------------------------------------ operand classes (stored values)
def _alt(lo):
    v = sum((0xffffffff if (j & 1) == lo else 0) << (32 * j) for j in range(12))
    return v % P
EDGE_S = sorted({0, 1, 2, ONE, P - 1, P - 2, (P - 1) // 2, (P + 1) // 2, P - ONE, _alt(0), _alt(1),
                 (P11 - 1) << 352 | ((1 << 352) - 1), (1 << 352) - 1, 1 << 352 | ((1 << 352) - 1)}
                | {1 << k for k in (31, 32, 63, 64, 191, 192, 255, 351, 352, 380)})


def rs(rng): return rng.randrange(P)


def gen_fp1(rng, n):
    return [([e], [], "edge") for e in EDGE_S] + [([rs(rng)], [], "rand") for _ in range(n)]


def gen_fp2op(rng, n):
    items = [([a, b], [], "edge") for a in EDGE_S[::2] for b in EDGE_S[1::2]]
    for s in (P - 1, P, P + 1):                     # pairs summing to p - 1, p, p + 1
        for _ in range(16):
            a = rng.randrange(1, P - 1); items.append(([a, (s - a) % P if s - a >= P else s - a], [], "sum"))
    return items + [([rs(rng), rs(rng)], [], "rand") for _ in range(n)]


def rand_f2(rng, cls=None):
    c = rng.randrange(8) if cls is None else cls
    if c == 0: return [0, rs(rng)]
    if c == 1: return [rs(rng), 0]
    if c == 2: return [rng.choice(EDGE_S), rng.choice(EDGE_S)]
    return [rs(rng), rs(rng)]


def gen_f2_1(rng, n):
    items = [([a, b], [], "edge") for a in EDGE_S[::3] for b in EDGE_S[1::3]] + [([0, 0], [], "zero")] * 4
    items += [([rs(rng), 0], [], "im0") for _ in range(8)] + [([0, rs(rng)], [], "re0") for _ in range(8)]
    return items + [(rand_f2(rng, 3), [], "rand") for _ in range(n)]


def gen_f2_2(rng, n):
    items = [(rand_f2(rng, c % 3) + rand_f2(rng, (c // 3) % 3), [], "edge") for c in range(36)]
    items += [([a, b, a, b], [], "equal") for a, b in ((0, 0), (P - 1, P - 1), (ONE, 0))]
    return items + [(rand_f2(rng, 3) + rand_f2(rng, 3), [], "rand") for _ in range(n)]


def rand_f12(rng, sparse=False):
    u = []
    for j in range(6):
        u += [0, 0] if sparse and rng.randrange(2) else rand_f2(rng, rng.randrange(8))
    return u


F12_ONE_S = [ONE] + [0] * 11
def gen_f12(rng, n, units_after=0, nonzero=False):
    extra = lambda: [s for _ in range(units_after // 2) for s in rand_f2(rng, rng.randrange(8))]
    items = [([P - 1] * 12 + extra(), [], "all_p-1"), (F12_ONE_S + extra(), [], "one")]
    if not nonzero: items.append(([0] * 12 + extra(), [], "zero"))
    items += [(rand_f12(rng, True) + extra(), [], "sparse") for _ in range(16)]
    items = [it for it in items if not (nonzero and not any(it[0][:12]))]
    return items + [(rand_f12(rng) + extra(), [], "rand") for _ in range(n)]


def cyclotomic(w):
    f = o.f12_mul(o.f12_conj(w), o.f12_inv(w))
    return o.f12_mul(o.f12_frob2(f), f)


def gen_cyc(rng, n):
    items = [(F12_ONE_S, [], "one")]
    for k in range(n):
        u = rand_f12(rng, sparse=k < 8)
        if not any(u): u = F12_ONE_S
        items.append((mF12(cyclotomic(F12(u, 0))), [], "sparse" if k < 8 else "rand"))
    return items


# ---- points: consecutive multiples of a base point, each in Jacobian form with a random Z
class G1F:
    F = o.FP; W = 1
    @staticmethod
    def dec(u, k): return val(u[k])
    @staticmethod
    def enc(x): return [mont(x)]
    @staticmethod
    def rnd(rng): return rng.randrange(1, P)
    base = o.G1_GEN

class G2F:
    F = o.FP2; W = 2
    @staticmethod
    def dec(u, k): return F2(u, k)
    @staticmethod
    def enc(x): return mF2(x)
    @staticmethod
    def rnd(rng): return (rng.randrange(P), rng.randrange(1, P))
    base = o.pt_from_affine(o.FP2, *o.sw_map_fp2((5, 7)))


def rescale(G, p, lam):
    F = G.F; l2 = F.sqr(lam)
    return (F.mul(p[0], l2), F.mul(p[1], F.mul(l2, lam)), F.mul(p[2], lam))


def enc_pt(G, p):
    if G.F.is_zero(p[2]): return [0] * (3 * G.W)
    return G.enc(p[0]) + G.enc(p[1]) + G.enc(p[2])


def dec_pt(G, u, k):
    W = G.W
    return (G.dec(u, k), G.dec(u, k + W), G.dec(u, k + 2 * W))


def points(G, rng, n):
    out, q = [], G.base
    for _ in range(n):
        out.append(rescale(G, q, G.rnd(rng)))
        q = o.pt_add(G.F, q, G.base)
    return out


def gen_pt2(G, rng, n, mixed=False):
    """(p, q) pairs by pt_add class; q affine (x, y, 1) or the affine identity (0, 0) for pt_add_mixed"""
    F, pts = G.F, points(G, rng, n + 64)
    inf = (F.zero, F.zero, F.zero)
    def aff(p):
        a = o.pt_affine(F, p)
        return (a[0], a[1], F.one)
    items = []
    def add(p, q, cls):
        items.append((enc_pt(G, p) + (G.enc(q[0]) + G.enc(q[1]) if mixed else enc_pt(G, q)), [], cls))
    for k in range(40):
        a, b = pts[k], pts[k + 1]
        add(inf, aff(b) if mixed else b, "p_inf")
        add(a, inf if not mixed else (F.zero, F.zero, F.zero), "q_inf")
        add(a, aff(a) if mixed else rescale(G, a, G.rnd(rng)), "double")
        add(a, aff(o.pt_neg(F, a)) if mixed else rescale(G, o.pt_neg(F, a), G.rnd(rng)), "opposite")
    for k in range(n):
        a, b = pts[64 + k], pts[rng.randrange(n + 64)]
        add(a, aff(b) if mixed else b, "rand")
    return items


def pt_norm(G, p):
    return [0] * (3 * G.W) if G.F.is_zero(p[2]) else enc_pt(G, p)


def pt_add_ref(G, p, q):
    F = G.F
    if F.is_zero(p[2]): return q
    if F.is_zero(q[2]): return p
    return o.pt_add(F, p, q)


def pt_add_branch(G, p, q):
    F = G.F
    if F.is_zero(p[2]): return "p_inf"
    if F.is_zero(q[2]): return "q_inf"
    Z1Z1, Z2Z2 = F.sqr(p[2]), F.sqr(q[2])
    H = F.sub(F.mul(q[0], Z1Z1), F.mul(p[0], Z2Z2))
    Rr = F.sub(F.mul(F.mul(q[1], p[2]), Z1Z1), F.mul(F.mul(p[1], q[2]), Z2Z2))
    if F.is_zero(H): return "H0_R0" if F.is_zero(Rr) else "H0_Rne0"
    return "general"


# ------------------------------------------------------------------ the op table: generator, expectation, restated branches
class Op:
    def __init__(self, gen, exp, tier=0, same=None, branch=None, branches=()):
        self.gen, self.exp, self.tier, self.same, self.branch, self.branches = gen, exp, tier, same, branch, branches


def same_first(k):
    """x == y forms: the second operand (k units from unit k) is the first one"""
    return lambda u, w: (u[:k] + u[:k] + u[2 * k:], w)


def redc_branch(T):
    m = (T % R) * NPRIME % R
    return "t>=p" if (T + m * P) >> 384 >= P else "t<p"


def bin_fp(f, br=None, brs=()):
    return Op(gen_fp2op, lambda u, w: ([mont(f(val(u[0]), val(u[1])))], None), same=same_first(1), branch=br, branches=brs)


def un_fp(f, tier=0, br=None, brs=()):
    return Op(gen_fp1, lambda u, w: ([mont(f(val(u[0])))], None), tier=tier, branch=br, branches=brs)


def legendre_flag(v):
    return [o.fp_legendre(v) & 0xffffffff] * 2


def sqrt_exp(u, w):
    r = o.fp_sqrt(val(u[0]))
    return ([None if r is None else mont(r)], [int(r is not None)] * 2)


def sqrt_inv_exp(u, w):
    r = o.fp_sqrt(val(u[0]))
    if r is None: return ([None, None], [0, 0])
    return ([mont(r), mont(pow(r, P - 2, P))], [1, 1])


def wide_gen(rng, n, k):
    top = R - 1
    items = [([top] * k, [], "max"), ([top, 1][:k], [], "max"), ([1 << 383] * k, [], "top_bit"), ([0] * k, [], "zero"),
             ([P - 1] * k, [], "p-1")]
    items += [([rng.getrandbits(384) for _ in range(k)], [], "rand") for _ in range(n)]
    return items


def w24(x): return [x % R, x >> 384]


def mul_wide2_gen(rng, n):
    top = R - 1
    items = [([top, top, 2, top], [], "sum=2^768-1"), ([top, top, 1, 1], [], "max"), ([P - 1] * 4, [], "p-1")]
    for _ in range(n):
        a1, b1 = rng.getrandbits(384), rng.getrandbits(384)
        room = R * R - 1 - a1 * b1
        a2 = rng.randrange(1, R); b2 = min(room // a2, R - 1)
        items.append(([a1, b1, a2, rng.randrange(b2 + 1)], [], "rand"))
    # the x == y forms square both pairs: keep a1^2 + a2^2 < 2^768 as well
    return [it for it in items if it[0][0] ** 2 + it[0][2] ** 2 < R * R]


def redc_gen(rng, n):
    items = [(w24(P * R - 1), [], "max"), (w24(0), [], "zero"), (w24(P * R - P), [], "edge"), (w24((P - 1) ** 2), [], "edge"),
             (w24(4 * P * P - 1), [], "4p^2")]
    return items + [(w24(rng.randrange(P * R)), [], "rand") for _ in range(n)]


def regs_gen(rng, n, k):
    """operands of the fused Fp2 products: canonical, with the squaring paths' s, d up to their < 2p bounds"""
    items = [([P - 1] * k, [], "p-1"), ([P - 1, 0] * (k // 2), [], "edge"), ([0, P - 1] * (k // 2), [], "edge")]
    return items + [([rs(rng) for _ in range(k)], [], "rand") for _ in range(n)]


# ---- Fp2 sqrt: the six outcomes of fp2_sqrt, restated
INV2 = (P + 1) // 2
def f2_sqrt_branch(a, b):
    if b == 0:
        if a == 0: return "x=0"
        return "b=0,a_res" if o.fp_sqrt(a) is not None else "b=0,a_nonres"
    n = o.fp_sqrt((a * a + b * b) % P)
    if n is None: return "norm_nonres"
    t2 = (a + n) * INV2 % P
    u = pow(t2, (P - 3) // 4, P); c = t2 * u % P
    if c * c % P == t2: return "first"
    h = (-(b * u % P) * INV2) % P
    return "second,leg(h)=%d" % o.fp_legendre(h)


def gen_sqrt2(rng, n):
    items = [([0, 0], [], "zero")] * 40
    items += [([mont(rng.randrange(P) ** 2 % P), 0], [], "b=0") for _ in range(40)]
    nr = [x for x in (rng.randrange(1, P) for _ in range(200)) if o.fp_legendre(x) < 0][:40]
    items += [([mont(x), 0], [], "b=0") for x in nr]
    for k in range(n):
        if k & 1:
            y = (rng.randrange(P), rng.randrange(P)); items.append((mF2(o.f2_sqr(y)), [], "square"))
        else:
            items.append((rand_f2(rng, 3), [], "rand"))
    return items


def f2_sqrt_exp(u, w):
    r = o.f2_sqrt(F2(u, 0))
    return ([None, None] if r is None else mF2(r), [int(r is not None)] * 2)


def f2_sqrt_any_exp(u, w):
    """a root of x (checked by squaring back, from the output), the same verdict as fp2_sqrt, and the documented choice for b = 0"""
    x = F2(u, 0); r = o.f2_sqrt(x)
    if r is None: return ([None, None], [0, 0])
    if x[1] == 0: return (mF2(r), [1, 1])
    return (lambda out: o.f2_sqr((val(out[0]), val(out[1]))) == x, [1, 1])


# ---- tower ops (both carriers)
FROB_G = [o.f2_pow(o.XI, k * (P - 1) // 6) for k in range(6)]
def f12_frob(w): return tuple(o.f2_mul(o.f2_conj(w[k]), FROB_G[k]) for k in range(6))
def line(o0, o1, o4): return (o0, o.F2_ZERO, o1, o4, o.F2_ZERO, o.F2_ZERO)
def f6_of(u, k): return F6(u, k)
def f12_of(u, k): return F12(u, k)
def verdict(b): return [int(b)] * 2


def lane_verdict_f2(rng):
    """zero / equal values and differences confined to one limb of one half"""
    items = [([0, 0], [], "zero")] * 40
    for h in range(2):
        for j in range(12):
            u = [0, 0]; u[h] = 1 << (32 * j); items.append((u, [], "one_limb"))
    return items


def gen_is_zero(rng, n):
    return lane_verdict_f2(rng) + [(rand_f2(rng), [], "rand") for _ in range(n)]


def gen_eq(rng, n):
    items = []
    for _ in range(40):
        a = rand_f2(rng, 3); items.append((a + a, [], "equal"))
    for h in range(2):
        for j in range(12):
            a = rand_f2(rng, 3); b = list(a); b[h] ^= 1 << (32 * j)
            if b[h] >= P: b[h] = a[h] ^ 1
            items.append((a + b, [], "one_limb"))
    return items + [(rand_f2(rng) + rand_f2(rng), [], "rand") for _ in range(n)]


def gen_is_one(rng, n):
    items = [(F12_ONE_S, [], "one")] * 40
    for c in range(6):
        for h in range(2):
            for j in range(12):
                u = list(F12_ONE_S); u[2 * c + h] ^= 1 << (32 * j); items.append((u, [], "one_limb"))
    items += [([0] * 12, [], "zero"), ([P - 1] * 12, [], "all_p-1")]
    return items + [(rand_f12(rng, sparse=True), [], "rand") for _ in range(n)]


def tower_ops(pre):
    T = {}
    g1 = lambda f, tier=0: Op(gen_f2_1, lambda u, w: (mF2(f(F2(u, 0))), None), tier=tier)
    g2 = lambda f, tier=0: Op(gen_f2_2, lambda u, w: (mF2(f(F2(u, 0), F2(u, 2))), None), tier=tier, same=same_first(2))
    T["mul"] = g2(o.f2_mul); T["add"] = g2(o.f2_add); T["sub"] = g2(o.f2_sub)
    T["sqr"] = g1(o.f2_sqr); T["neg"] = g1(o.f2_neg); T["dbl"] = g1(lambda x: o.f2_add(x, x))
    T["inv"] = g1(o.f2_inv, 1); T["inv_gcd"] = g1(o.f2_inv, 1); T["mul_xi"] = g1(o.f2_mul_xi); T["conj"] = g1(o.f2_conj)
    T["half"] = g1(lambda x: o.f2_mulfp(x, INV2)); T["mul_twist3b"] = g1(lambda x: o.f2_mulfp(o.f2_mul_xi(x), 12))
    T["mul_fp"] = Op(lambda rng, n: [(u + [k], [], c) for (u, _, c), k in
                                     zip(gen_f2_1(rng, n), [rng.choice(EDGE_S) if i % 5 == 0 else rs(rng) for i in range(10 ** 5)])],
                     lambda u, w: (mF2(o.f2_mulfp(F2(u, 0), val(u[2]))), None))
    T["is_zero"] = Op(gen_is_zero, lambda u, w: ([], verdict(u[0] == 0 and u[1] == 0)))
    T["eq"] = Op(gen_eq, lambda u, w: ([], verdict(u[0:2] == u[2:4])), same=same_first(2))
    T["one"] = Op(lambda rng, n: [([], [], "const")] * 64, lambda u, w: ([ONE, 0], None))
    T["const"] = Op(lambda rng, n: [([], [], "const")] * 64, lambda u, w: (mF2(FROB_G[1]), None))
    f6g = lambda k: (lambda rng, n: [(rand_f12(rng, i < 16)[:6] + [s for _ in range(k) for s in rand_f2(rng)], [], "sparse" if i < 16 else "rand")
                                    for i in range(n + 16)] + [([P - 1] * (6 + 2 * k), [], "all_p-1")])
    T["fp6_mul"] = Op(lambda rng, n: [(a[:6] + b[:6], [], c) for (a, _, c), (b, _, _) in zip(gen_f12(rng, n), gen_f12(rng, n))],
                      lambda u, w: (mF6(o._f6_mul(F6(u, 0), F6(u, 6))), None), tier=2, same=same_first(6))
    T["fp6_inv"] = Op(lambda rng, n: [it for it in f6g(0)(rng, n) if any(it[0])], lambda u, w: (mF6(o._f6_inv(F6(u, 0))), None), tier=2)
    T["fp6_mul_by_01"] = Op(f6g(2), lambda u, w: (mF6(o._f6_mul(F6(u, 0), (F2(u, 6), F2(u, 8), o.F2_ZERO))), None), tier=2)
    T["fp6_mul_by_1"] = Op(f6g(1), lambda u, w: (mF6(o._f6_mul(F6(u, 0), (o.F2_ZERO, F2(u, 6), o.F2_ZERO))), None), tier=2)
    T["fp6_mul_by_12"] = Op(f6g(2), lambda u, w: (mF6(o._f6_mul(F6(u, 0), (o.F2_ZERO, F2(u, 6), F2(u, 8)))), None), tier=2)
    T["fp12_mul"] = Op(lambda rng, n: [(a + b, [], c) for (a, _, c), (b, _, _) in zip(gen_f12(rng, n), gen_f12(rng, n))],
                       lambda u, w: (mF12(o.f12_mul(F12(u, 0), F12(u, 12))), None), tier=2, same=same_first(12))
    T["fp12_sqr"] = Op(gen_f12, lambda u, w: (mF12(o.f12_sqr(F12(u, 0))), None), tier=2)
    T["fp12_inv"] = Op(lambda rng, n: gen_f12(rng, n, nonzero=True), lambda u, w: (mF12(o.f12_inv(F12(u, 0))), None), tier=2)
    T["fp12_conj"] = Op(gen_f12, lambda u, w: (mF12(o.f12_conj(F12(u, 0))), None), tier=2)
    T["fp12_mul_by_014"] = Op(lambda rng, n: gen_f12(rng, n, 6),
                              lambda u, w: (mF12(o.f12_mul(F12(u, 0), line(F2(u, 12), F2(u, 14), F2(u, 16)))), None), tier=2)
    T["fp12_mul_by_two_lines"] = Op(lambda rng, n: gen_f12(rng, n, 12),
                                    lambda u, w: (mF12(o.f12_mul(o.f12_mul(F12(u, 0), line(F2(u, 12), F2(u, 14), F2(u, 16))),
                                                                 line(F2(u, 18), F2(u, 20), F2(u, 22)))), None), tier=2)
    T["fp12_frob"] = Op(gen_f12, lambda u, w: (mF12(f12_frob(F12(u, 0))), None), tier=2)
    T["fp12_frob2"] = Op(gen_f12, lambda u, w: (mF12(o.f12_frob2(F12(u, 0))), None), tier=2)
    T["fp12_is_one"] = Op(gen_is_one, lambda u, w: ([], verdict(u[:12] == F12_ONE_S)), tier=2)
    T["fp12_cyc_sqr"] = Op(gen_cyc, lambda u, w: (mF12(o.f12_sqr(F12(u, 0))), None), tier=2)
    T["fp12_cyc_exp_z"] = Op(gen_cyc, lambda u, w: (mF12(o.f12_conj(o.f12_pow(F12(u, 0), o.Z_ABS))), None), tier=3)
    T["final_exp"] = Op(lambda rng, n: gen_f12(rng, n, nonzero=True)[:n + 2],
                        lambda u, w: (mF12(o.f12_pow(o.final_exp(F12(u, 0)), 3)), None), tier=4)
    if pre == "fp2h":                                                   # the split carrier's add / sub / ... are single-lane ops: cheap
        for k in ("mul", "sqr", "inv", "inv_gcd", "mul_xi", "conj", "mul_fp", "is_zero", "eq"):
            T[k].tier = max(T[k].tier, 1)
        for k in ("fp6_mul", "fp6_inv", "fp6_mul_by_01", "fp6_mul_by_1", "fp6_mul_by_12"):
            T[k].tier = 2
    return {pre + "_" + k: v for k, v in T.items()}


def group_ops(pre, G, pair):
    F, W = G.F, G.W
    tier = 2 if pair else 1
    def jac2(u): return dec_pt(G, u, 0), dec_pt(G, u, 3 * W)
    def add_exp(u, w):
        p, q = jac2(u)
        return (pt_norm(G, pt_add_ref(G, p, q)), None)
    def mixed_exp(u, w):
        p = dec_pt(G, u, 0); qx, qy = G.dec(u, 3 * W), G.dec(u, 4 * W)
        if F.is_zero(qx) and F.is_zero(qy): return (pt_norm(G, p), None)
        return (pt_norm(G, pt_add_ref(G, p, (qx, qy, F.one))), None)
    def dbl_exp(u, w):
        p = dec_pt(G, u, 0)
        return (pt_norm(G, p if F.is_zero(p[2]) else o.pt_dbl(F, p)), None)
    def eq_exp(u, w):
        p, q = jac2(u)
        pi, qi = F.is_zero(p[2]), F.is_zero(q[2])
        return ([], verdict(pi and qi if pi or qi else o.pt_eq(F, p, q)))
    def aff_enc(p):
        a = o.pt_affine(F, p)
        return [0] * (2 * W) if a is None else G.enc(a[0]) + G.enc(a[1])
    def gen_dbl(rng, n):
        return [([0] * (3 * W), [], "inf")] * 40 + [(enc_pt(G, p), [], "rand") for p in points(G, rng, n)]
    def gen_eq(rng, n):
        items = gen_pt2(G, rng, n)
        pts = points(G, rng, 40)
        items += [(enc_pt(G, p) + enc_pt(G, rescale(G, p, G.rnd(rng))), [], "equal") for p in pts]
        return items
    def gen_aff(rng, n):
        # identity lanes among ordinary points: the scattered launch mixes them into the same warps
        return [([0] * (3 * W), [], "inf")] * 40 + [(enc_pt(G, p), [], "rand") for p in points(G, rng, n)]
    def gen_zinv(rng, n):
        return [(it + G.enc(G.rnd(rng)) if not any(it) else it + G.enc(F.inv(dec_pt(G, it, 0)[2])), w, c)
                for it, w, c in gen_aff(rng, n)]
    def zinv_exp(u, w):
        return (aff_enc(dec_pt(G, u, 0)), None)
    def gen_binv(rng, n):
        items = []
        for k in range(n + 64):
            zs = [G.rnd(rng) for _ in range(4)]
            skip = [1, 1, 1, 1] if k % 16 == 0 else ([0, 0, 0, 0] if k % 16 == 1 else [rng.randrange(2) for _ in range(4)])
            items.append(([s for z in zs for s in G.enc(z)], skip, "rand" if k >= 64 else "skip"))
        return items
    def binv_exp(u, w):
        out = []
        for k in range(4):
            z = G.dec(u, k * W)
            out += G.enc(z) if w[k] else G.enc(F.inv(z))
        return (out, None)
    ops = {
        "pt_dbl": Op(gen_dbl, dbl_exp, tier),
        "pt_add": Op(lambda rng, n: gen_pt2(G, rng, n), add_exp, tier, same=same_first(3 * W),
                     branch=lambda u, w: pt_add_branch(G, *jac2(u)), branches=("p_inf", "q_inf", "H0_R0", "H0_Rne0", "general")),
        "pt_add_mixed": Op(lambda rng, n: gen_pt2(G, rng, n, mixed=True), mixed_exp, tier),
        "pt_eq": Op(gen_eq, eq_exp, tier, same=same_first(3 * W)),
        "pt_to_aff": Op(gen_aff, lambda u, w: (aff_enc(dec_pt(G, u, 0)), None), tier),
        "pt_to_aff_zinv": Op(gen_zinv, zinv_exp, tier),
        "batch_inv": Op(gen_binv, binv_exp, tier),
    }
    return {pre + "_" + k: v for k, v in ops.items()}


# ---- step machine
def atom(s, half, neg, m): return s | half << 8 | neg << 9 | (m - 1) << 10
def row_words(atoms):
    atoms = atoms + [atom(8, 0, 0, 1)] * (8 - len(atoms))
    return [atoms[2 * k] | atoms[2 * k + 1] << 16 for k in range(4)]


def vm_lin_gen(rng, n):
    items = []
    def add(slots, ra, ia, cls):
        items.append(([s for v in slots for s in v], row_words(ra) + row_words(ia) + [max(len(ra), len(ia))], cls))
    pm1 = [[P - 1, P - 1]] * 8
    for _ in range(8):
        add(pm1, [atom(k, k & 1, 0, 4) for k in range(8)], [atom(k, 1, 0, 4) for k in range(8)], "+4(p-1)x8")
        add(pm1, [atom(k, 0, 1, 4) for k in range(8)], [atom(k, k & 1, 1, 4) for k in range(8)], "-4(p-1)x8")
    for _ in range(16):
        a = rs(rng); b = (P - a) % P                 # a + b = p, then k p with multipliers
        s = [[a, b], [b, a]] + [[rs(rng), rs(rng)] for _ in range(6)]
        add(s, [atom(0, 0, 0, 1), atom(0, 0, 1, 1)], [atom(0, 0, 0, 1), atom(0, 1, 0, 1)], "sum=0,p")
        add(s, [atom(0, 0, 0, 3), atom(0, 1, 0, 3)], [atom(1, 0, 0, 4), atom(1, 1, 0, 4), atom(0, 0, 0, 2), atom(0, 1, 0, 2)], "sum=kp")
        add(s, [atom(8, 0, 0, 4), atom(8, 1, 1, 3)], [atom(2, 1, 0, 2), atom(8, 0, 1, 4)], "zero_slot")
    for _ in range(n):
        s = [[rs(rng), rs(rng)] for _ in range(8)]
        na = rng.randrange(1, 9)
        rnd = lambda: [atom(rng.choice((rng.randrange(8), 8)) if rng.randrange(6) == 0 else rng.randrange(8), rng.randrange(2),
                            rng.randrange(2), rng.randrange(1, 5)) for _ in range(na)]
        add(s, rnd(), rnd(), "rand")
    return items


def vm_lin_sums(u, w):
    def lane(words):
        atoms = [(words[k >> 1] >> (16 * (k & 1))) & 0xffff for k in range(8)][:w[8]]
        tot = 0
        for a in atoms:
            s, h, neg, m = a & 0xff, (a >> 8) & 1, (a >> 9) & 1, ((a >> 10) & 3) + 1
            v = 0 if s == 8 else u[2 * s + h]
            tot += -m * v if neg else m * v
        return tot
    return lane(w[0:4]), lane(w[4:8])


def vm_lin_exp(u, w):
    re, im = vm_lin_sums(u, w)
    return ([re % P, im % P], None)


def vm_lin_branch(u, w):
    """the latency form: value = sum + 631 p, less floor(top 42 bits / (p_11 + 1)) p; [p, 2p) needs a trial subtraction"""
    hit = False
    for s in vm_lin_sums(u, w):
        v = s + 631 * P
        rem = v - ((v >> 352) // (P11 + 1)) * P
        hit |= rem >= P
    return "[p,2p)" if hit else "[0,p)"


VM_OPS = {
    "vm_mul": Op(gen_f2_2, lambda u, w: ([s % P for s in mF2(o.f2_mul(F2(u, 0), F2(u, 2)))], None), same=same_first(2)),
    "vm_sqr": Op(gen_f2_1, lambda u, w: (mF2(o.f2_sqr(F2(u, 0))), None)),
    "vm_lin": Op(vm_lin_gen, vm_lin_exp, branch=vm_lin_branch, branches=("[p,2p)", "[0,p)")),
}

SPECS = {
    "fp_mul": bin_fp(lambda a, b: a * b, lambda u, w: redc_branch(u[0] * u[1]), ("t>=p", "t<p")),
    "fp_sqr": un_fp(lambda a: a * a, br=lambda u, w: redc_branch(u[0] * u[0]), brs=("t>=p", "t<p")),
    "fp_add": bin_fp(lambda a, b: a + b, lambda u, w: "carry" if u[0] + u[1] >= P else "no_carry", ("carry", "no_carry")),
    "fp_sub": bin_fp(lambda a, b: a - b, lambda u, w: "borrow" if u[0] < u[1] else "no_borrow", ("borrow", "no_borrow")),
    "fp_dbl": un_fp(lambda a: 2 * a),
    "fp_neg": un_fp(lambda a: -a),
    "fp_half": un_fp(lambda a: a * INV2, br=lambda u, w: "odd" if u[0] & 1 else "even", brs=("odd", "even")),
    "fp_inv": un_fp(lambda a: pow(a, P - 2, P), tier=1),
    "fp_inv_gcd": un_fp(lambda a: pow(a, P - 2, P), tier=1),
    "fp_sqrt": Op(gen_fp1, sqrt_exp, tier=1),
    "fp_sqrt_inv": Op(gen_fp1, sqrt_inv_exp, tier=1),
    "fp_legendre": Op(gen_fp1, lambda u, w: ([], legendre_flag(u[0]))),
    "fp_legendre_pow": Op(gen_fp1, lambda u, w: ([], legendre_flag(u[0])), tier=1),
    "fp_from_int": Op(gen_fp1, lambda u, w: ([u[0] * R % P], None)),
    "fp_to_int": Op(gen_fp1, lambda u, w: ([val(u[0])], None)),
    "fp_int_geq_p": Op(lambda rng, n: [([v], [], "edge") for v in (P - 1, P, P + 1, R - 1, 0, P - ONE, P11 << 352)]
                       + [([rng.getrandbits(384) >> rng.randrange(4)], [], "rand") for _ in range(n)],
                       lambda u, w: ([], verdict(u[0] >= P))),
    "mul_wide": Op(lambda rng, n: wide_gen(rng, n, 2), lambda u, w: (w24(u[0] * u[1]), None), same=same_first(1)),
    "mul_wide_k": Op(lambda rng, n: wide_gen(rng, n, 2), lambda u, w: (w24(u[0] * u[1]), None), same=same_first(1)),
    "mul_wide2": Op(mul_wide2_gen, lambda u, w: (w24(u[0] * u[1] + u[2] * u[3]), None),
                    same=lambda u, w: ([u[0], u[0], u[2], u[2]], w)),
    "sqr_wide": Op(lambda rng, n: wide_gen(rng, n, 1), lambda u, w: (w24(u[0] * u[0]), None)),
    "redc_wide": Op(redc_gen, lambda u, w: ([(u[0] + (u[1] << 384)) * RINV % P], None),
                    branch=lambda u, w: redc_branch(u[0] + (u[1] << 384)), branches=("t>=p", "t<p")),
    "fp2_mul_regs": Op(lambda rng, n: regs_gen(rng, n, 4), lambda u, w: (mF2(o.f2_mul(F2(u, 0), F2(u, 2))), None), same=same_first(2)),
    "fp2_mul_regs_cios": Op(lambda rng, n: regs_gen(rng, n, 4), lambda u, w: (mF2(o.f2_mul(F2(u, 0), F2(u, 2))), None), same=same_first(2)),
    "fp2_sqr_regs": Op(lambda rng, n: regs_gen(rng, n, 2), lambda u, w: (mF2(o.f2_sqr(F2(u, 0))), None)),
    "fp2_sqr_regs_cios": Op(lambda rng, n: regs_gen(rng, n, 2), lambda u, w: (mF2(o.f2_sqr(F2(u, 0))), None)),
    "fp2_sqrt": Op(gen_sqrt2, f2_sqrt_exp, tier=1, branch=lambda u, w: f2_sqrt_branch(*F2(u, 0)),
                   branches=("x=0", "b=0,a_res", "b=0,a_nonres", "norm_nonres", "first", "second,leg(h)=1", "second,leg(h)=-1")),
    "fp2_sqrt_anysign": Op(gen_sqrt2, f2_sqrt_any_exp, tier=1),
    "fp2_norm": Op(gen_f2_1, lambda u, w: ([mont(o.f2_norm(F2(u, 0)))], None)),
}
SPECS.update(tower_ops("fp2")); SPECS.update(tower_ops("fp2h"))
SPECS.update(group_ops("g1", G1F, False)); SPECS.update(group_ops("g2", G2F, False)); SPECS.update(group_ops("g2h", G2F, True))
SPECS.update(VM_OPS)

# random items per op by cost tier (the host emulation runs a lane pair on two threads and is slow for the Fp12 layer)
N_GPU = {0: 4096, 1: 4096, 2: 4096, 3: 256, 4: 8}
N_CPU = {0: 4096, 1: 512, 2: 48, 3: 4, 4: 2}
N_VARIANT = 512
# code switches of csrc/ that are off by default; the host build ignores the ones that only change inlining or CTA barriers
VARIANTS = ["-DHB_FUSED_FP2=1", "-DHB_FUSED_FP2=2", "-DHB_KARATSUBA=1", "-DHB_OUTLINE_FP=1", "-DHB_SPLIT_INLINE=0",
            "-DHB_VM_LIN_V1=1", "-DHB_LOCKSTEP=3"]
HOST_VARIANTS = ["-DHB_FUSED_FP2=1", "-DHB_FUSED_FP2=2", "-DHB_KARATSUBA=1", "-DHB_VM_LIN_V1=1"]


# ------------------------------------------------------------------ items, runs, checks
_ITEMS = {}
def items_for(name, n):
    """edges + n seeded random items with their expected outputs (cached: the CPU, GPU and variant runs share them)"""
    key = (name, n)
    if key not in _ITEMS:
        spec = SPECS[name]
        rng = random.Random(sum(map(ord, name)) * 7919 + n)
        its = spec.gen(rng, n)
        exp = {}
        for same in (False, True):
            if same and spec.same is None: continue
            exp[same] = [spec.exp(*(spec.same(u, w) if same else (u, w))) for u, w, c in its]
        _ITEMS[key] = (its, exp)
    return _ITEMS[key]


def pack(its, in_w):
    out = bytearray()
    for u, w, c in its:
        b = b"".join(x.to_bytes(48, "little") for x in u) + b"".join(x.to_bytes(4, "little") for x in w)
        assert len(b) == 4 * in_w, (len(b), in_w)
        out += b
    return bytes(out)


class Lib:
    def __init__(self, path):
        L = ctypes.CDLL(path)
        L.ar_run.argtypes = [ctypes.c_int, ctypes.c_int, ctypes.c_size_t, ctypes.c_char_p, ctypes.c_char_p]
        L.ar_op_name.restype = ctypes.c_char_p
        L.ar_op_info.argtypes = [ctypes.c_int, ctypes.POINTER(ctypes.c_int)]
        self.L = L
        self.ops = {}
        for i in range(L.ar_op_count()):
            v = (ctypes.c_int * 4)(); L.ar_op_info(i, v)
            self.ops[L.ar_op_name(i).decode()] = (i, v[0], v[1], v[2], v[3])

    def forms(self, name):
        return [a for a in range(5) if (self.ops[name][2] >> a) & 1]

    def run(self, name, alias, its):
        i, carrier, forms, in_w, out_w = self.ops[name]
        n = len(its)
        out = ctypes.create_string_buffer(4 * out_w * n)
        rc = self.L.ar_run(i, alias, n, pack(its, in_w), out)
        assert rc == 0, (name, alias, rc)
        raw = out.raw
        res = []
        for k in range(n):
            b = raw[4 * out_w * k:4 * out_w * (k + 1)]
            nu = out_w // 12
            units = [int.from_bytes(b[48 * j:48 * j + 48], "little") for j in range(nu)]
            flags = [int.from_bytes(b[48 * nu + 4 * j:48 * nu + 4 * j + 4], "little") for j in range(out_w % 12)]
            res.append((units, flags))
        return res


def mismatches(name, alias, its, exp, got):
    bad = []
    for k, ((u, w, c), (eu, ef), (gu, gf)) in enumerate(zip(its, exp, got)):
        if callable(eu): ok = ef is None or ef == gf[:len(ef)] and eu(gu)
        else:
            ok = all(e is None or e == g for e, g in zip(eu, gu)) and (ef is None or ef == gf)
        if not ok:
            bad.append((k, c, [hex(x) for x in u][:4], w[:4]))
    return ["%s form %d: %d of %d items differ, first %s" % (name, alias, len(bad), len(its), bad[:3])] if bad else []


def check_op(lib, name, n, scatter_sort=False):
    spec = SPECS[name]
    its, exp = items_for(name, n)
    errs = []
    orders = [None]
    if scatter_sort:
        rng = random.Random(len(its))
        scattered = list(range(len(its))); rng.shuffle(scattered)
        orders = [scattered, sorted(range(len(its)), key=lambda k: its[k][2])]
    for alias in lib.forms(name):
        e = exp[alias >= 3]
        for order in orders:
            oi = its if order is None else [its[k] for k in order]
            oe = e if order is None else [e[k] for k in order]
            errs += mismatches(name, alias, oi, oe, lib.run(name, alias, oi))
    return errs


def coverage(name, n):
    spec = SPECS[name]
    if spec.branch is None: return []
    its, _ = items_for(name, n)
    cnt = {}
    for u, w, c in its:
        b = spec.branch(u, w); cnt[b] = cnt.get(b, 0) + 1
    return ["%s: branch %s reached by %d items" % (name, b, cnt.get(b, 0)) for b in spec.branches if cnt.get(b, 0) < MIN_HITS]


# ------------------------------------------------------------------ builds
def build_emu(defs=()):
    tag = "_".join(d.strip("-D").replace("=", "") for d in defs) or "default"
    out = os.path.join(_BUILD, "libemu_arith_%s.so" % tag)
    if not os.path.exists(out):
        subprocess.check_call(["g++", "-O1", "-std=c++17", "-fPIC", "-shared", "-pthread", *defs, "-o", out,
                               os.path.join(ROOT, "tests", "emu", "emu_arith.cpp")])
    return out


def build_driver(defs=()):
    tag = "_".join(d.strip("-D").replace("=", "") for d in defs) or "default"
    out = os.path.join(_BUILD, "libarith_driver_%s.so" % tag)
    if not os.path.exists(out):
        nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
        subprocess.check_call([nvcc, *NVCC_FLAGS, *defs, "-o", out, os.path.join(ROOT, "tests", "arith", "arith_driver.cu")])
    return out


def build_all(builder, variants):
    with concurrent.futures.ThreadPoolExecutor(max_workers=min(9, os.cpu_count() or 1)) as ex:
        futs = {v: ex.submit(builder, (v,) if v else ()) for v in variants}
        return {v: f.result() for v, f in futs.items()}


# ------------------------------------------------------------------ CPU: host emulation
@pytest.fixture(scope="module")
def emu_libs():
    return {v: Lib(p) for v, p in build_all(build_emu, [None] + HOST_VARIANTS).items()}


def test_every_op_has_a_spec_and_runs_each_form(emu_libs):
    lib = emu_libs[None]
    assert sorted(lib.ops) == sorted(SPECS)
    for name, (i, carrier, forms, in_w, out_w) in lib.ops.items():
        want = {0x1f: 5, 0x3: 2, 0x9: 2, 0x1: 1}[forms]
        assert len(lib.forms(name)) == want
        if want == 5 or forms == 0x9: assert SPECS[name].same is not None, name


@pytest.mark.parametrize("name", sorted(SPECS))
def test_emu_op(emu_libs, name):
    n = N_CPU[SPECS[name].tier]
    assert not coverage(name, max(n, 4096) if SPECS[name].tier == 0 else n)
    assert not check_op(emu_libs[None], name, n)


def test_emu_op_coverage():
    errs = [e for name in SPECS for e in coverage(name, N_CPU[SPECS[name].tier])]
    assert not errs, errs


@pytest.mark.parametrize("flag", HOST_VARIANTS)
def test_emu_variant(emu_libs, flag):
    errs = []
    for name in sorted(SPECS):
        errs += check_op(emu_libs[flag], name, min(N_VARIANT, N_CPU[SPECS[name].tier]))
    assert not errs, errs


# ------------------------------------------------------------------ GPU: the same table compiled for sm_90a
@pytest.fixture(scope="module")
def gpu_libs():
    return {v: Lib(p) for v, p in build_all(build_driver, [None] + VARIANTS).items()}


@pytest.mark.gpu
def test_gpu_every_op_exercised(gpu_libs):
    assert sorted(gpu_libs[None].ops) == sorted(SPECS)


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(SPECS))
def test_gpu_op(gpu_libs, name):
    n = N_GPU[SPECS[name].tier]
    assert not coverage(name, n)
    errs = check_op(gpu_libs[None], name, n, scatter_sort=True)
    assert not errs, errs


@pytest.mark.gpu
@pytest.mark.parametrize("flag", VARIANTS)
def test_gpu_variant(gpu_libs, flag):
    errs = []
    for name in sorted(SPECS):
        errs += check_op(gpu_libs[flag], name, min(N_VARIANT, N_GPU[SPECS[name].tier]))
    assert not errs, errs
