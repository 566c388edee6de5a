"""Subgroup membership on every decode path, with valid points plus small-order torsion.

A point on the curve but outside the prime-order subgroup must be rejected where it is decoded; nothing behind the decoder checks
again.  For T of small order q in E(Fp) (q a prime of the G1 cofactor h1), pk + T satisfies the bare pairing equation
e(B, sigma) == e(pk + T, H(m)) for every signature sigma that pk made: without the membership test it is a second encoding of pk.  On
G2 the batched form applies each coefficient as a + b psi^2, which equals [a + b z^2] only on G2, and its 2^-63 bound assumes prime
order.

The library has four membership tests: g1_in_subgroup (k_g1_decode, k_g1_decode_jac, k_single), g2_in_subgroup over Fp2 in a thread
(k_g2_decode, k_single) and in the split kernel k_g2_subgroup, and g2_in_subgroup over the lane-pair carrier (k_g2_decode_pair,
k_g2_subgroup_pair; the warm H(m)-cache path decodes without it and runs k_g2_subgroup_pair beside the first Miller loop).  The C
oracle uses the same endomorphism tests as the device, so the expected verdicts come from oracle/pyref.py with check_order=True,
which tests [r]P == O.  The reference pins none of these rejections byte for byte (SURVEY A.7); a sign bit on an all-zero x is
listed in UNPINNED, and follows pyref and the C oracle like the rest.

Crafted inputs (module scope, seeded): a point T of exact order q for every prime q^e || h1 and q^e || h2, and one point of G2 whose
order is the 448-bit prime part of h2; each T alone, P + T and -P + T for a real key or signature P; the encoding edges (x = p, x >= p
only through bit 381 or 382, one Fp2 coordinate >= p, the sign bit flipped, the identity).

CPU: pyref against the C oracle; the device decoders run on the host (tests/emu) against pyref.
GPU: every entry point that decodes a key or a signature, in each form of the pipeline, on batches of honest rounds with the crafted
ones at seeded positions.  Every knob and the batch mode are restored whatever happens."""
import contextlib, ctypes, os, random, subprocess, sys
import pytest
from harmony_b200 import workload as wl

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "oracle"))
import pyref as o                                   # noqa: E402

Z, R, P = o.Z, o.R, o.P

# ------------------------------------------------------------------ cofactors
H1 = (Z - 1) ** 2 // 3
H1_FACTORS = {3: 1, 11: 2, 10177: 2, 859267: 2, 52437899: 2}
H2_NUM = Z ** 8 - 4 * Z ** 7 + 5 * Z ** 6 - 4 * Z ** 4 + 6 * Z ** 3 - 4 * Z ** 2 - 4 * Z + 13
H2 = H2_NUM // 9


def trial_division(n, bound):
    small = {}
    for d in range(2, bound):
        while n % d == 0:
            small[d] = small.get(d, 0) + 1
            n //= d
    return small, n


H2_SMALL, H2_LARGE = trial_division(H2, 1 << 19)


def is_probable_prime(n):
    d, s = n - 1, 0
    while d % 2 == 0: d //= 2; s += 1
    for a in (2, 3, 5, 7, 11, 13, 17, 19, 23, 29, 31, 37):
        x = pow(a, d, n)
        if x in (1, n - 1): continue
        for _ in range(s - 1):
            x = x * x % n
            if x == n - 1: break
        else:
            return False
    return True


# ------------------------------------------------------------------ torsion points
_rng = random.Random(0x5b9)


def _rand_g1():
    while True:
        x = _rng.randrange(P); y = o.fp_sqrt((x ** 3 + o.B1) % P)
        if y is not None: return o.pt_from_affine(o.FP, x, y)


def _rand_g2():
    while True:
        x = (_rng.randrange(P), _rng.randrange(P)); y = o.f2_sqrt(o.f2_add(o.f2_mul(o.f2_sqr(x), x), o.B2))
        if y is not None: return o.pt_from_affine(o.FP2, x, y)


def _torsion(F, rand, order, q, e):
    """[order / q^e] Q for a random curve point Q (again while that is O), then multiplied down by q to exact order q."""
    while True:
        T = o.pt_mul(F, rand(), order // q ** e)
        if not o.pt_is_inf(F, T): break
    while not o.pt_is_inf(F, o.pt_mul(F, T, q)): T = o.pt_mul(F, T, q)
    return T


T1 = {q: _torsion(o.FP, _rand_g1, H1 * R, q, e) for q, e in H1_FACTORS.items()}
if o.pt_affine(o.FP, T1[3])[1] % 2 == 0:             # order 3: (0, +-2); the even one would encode as the identity
    T1[3] = o.pt_neg(o.FP, T1[3])
T2 = {q: _torsion(o.FP2, _rand_g2, H2 * R, q, e) for q, e in H2_SMALL.items()}
while True:                                          # order H2_LARGE: the torsion part of h2 that is not small
    T2["L"] = o.pt_mul(o.FP2, _rand_g2(), R * (H2 // H2_LARGE))
    if not o.pt_is_inf(o.FP2, T2["L"]): break
T2_ORDER = {**{q: q for q in H2_SMALL}, "L": H2_LARGE}

X0_ODD_G1 = bytes(47) + b"\x80"                      # x = 0 with the sign bit: the order-3 point (0, -2) of E(Fp)
X0_ODD_G2 = bytes(95) + b"\x80"                      # x = 0 with the sign bit: 4 (1 + i) is no square, not on E'
UNPINNED = {"x=0 odd"}                               # a sign bit on an all-zero x: the reference does not pin it (SURVEY A.7)


# ------------------------------------------------------------------ point classes and encoding edges
def _set(b, byte, mask):
    x = bytearray(b); x[byte] |= mask; return bytes(x)


def _flip(b, byte):
    x = bytearray(b); x[byte] ^= 0x80; return bytes(x)


def key_classes(pk48):
    """T alone, pk + T, -pk + T for every G1 torsion point, and x = 0 with the sign bit."""
    pk = o.g1_deserialize(pk48, check_order=False)
    out = [("x=0 odd", X0_ODD_G1)]
    for q, T in T1.items():
        out += [(f"T{q}", o.g1_serialize(T)), (f"P+T{q}", o.g1_serialize(o.pt_add(o.FP, pk, T))),
                (f"-P+T{q}", o.g1_serialize(o.pt_add(o.FP, o.pt_neg(o.FP, pk), T)))]
    return out


def sig_classes(sig96):
    sg = o.g2_deserialize(sig96, check_order=False)
    out = [("x=0 odd", X0_ODD_G2)]
    for q, T in T2.items():
        out += [(f"T{q}", o.g2_serialize(T)), (f"P+T{q}", o.g2_serialize(o.pt_add(o.FP2, sg, T))),
                (f"-P+T{q}", o.g2_serialize(o.pt_add(o.FP2, o.pt_neg(o.FP2, sg), T)))]
    return out


def key_edges(pk48):
    pb = P.to_bytes(48, "little")
    return [("x=p", pb), ("x=p odd", _set(pb, 47, 0x80)), ("bit 381", _set(pk48, 47, 0x20)), ("bit 382", _set(pk48, 47, 0x40)),
            ("sign flipped", _flip(pk48, 47)), ("identity", bytes(48))]


def sig_edges(sig96):
    c0, c1 = int.from_bytes(sig96[:48], "little"), int.from_bytes(sig96[48:], "little")
    sign, c1 = c1 >> 383, c1 & ((1 << 383) - 1)
    return [("c0=p", P.to_bytes(48, "little") + sig96[48:]), ("c0+p", (c0 + P).to_bytes(48, "little") + sig96[48:]),
            ("c0 bit 383", _set(sig96, 47, 0x80)), ("c1+p", sig96[:48] + ((c1 + P) | sign << 383).to_bytes(48, "little")),
            ("c1 bit 381", _set(sig96, 95, 0x20)), ("c1 bit 382", _set(sig96, 95, 0x40)),
            ("sign flipped", _flip(sig96, 95)), ("identity", bytes(96))]


def all_keys(pk48): return key_classes(pk48) + key_edges(pk48)
def all_sigs(sig96): return sig_classes(sig96) + sig_edges(sig96)


# a real key and its signature; the crafted encodings built from them, with pyref's verdicts (decoded, decoded without the order test)
SK = wl.seeded_sk("sgm", 0)
MSG = wl.commit_payload("sgm", 0)
PK_PT = o.get_public_key(SK)
SIG_PT = o.sign_hash(SK, MSG)
PK48, SIG96 = o.g1_serialize(PK_PT), o.g2_serialize(SIG_PT)
G1_CASES = [(n, b, o.g1_deserialize(b) is not None, o.g1_deserialize(b, check_order=False) is not None) for n, b in all_keys(PK48)]
G2_CASES = [(n, b, o.g2_deserialize(b) is not None, o.g2_deserialize(b, check_order=False) is not None) for n, b in all_sigs(SIG96)]
VALID_EDGES = {"sign flipped", "identity"}


# ------------------------------------------------------------------ CPU: the inputs themselves
def test_cofactor_factorizations():
    assert (Z - 1) ** 2 % 3 == 0 and H2_NUM % 9 == 0
    prod = 1
    for q, e in H1_FACTORS.items(): prod *= q ** e
    assert prod == H1
    assert H2_SMALL == {13: 2, 23: 2, 2713: 1, 11953: 1, 262069: 1}
    assert H2_LARGE.bit_length() == 448 and is_probable_prime(H2_LARGE)
    prod = H2_LARGE
    for q, e in H2_SMALL.items(): prod *= q ** e
    assert prod == H2
    # #E(Fp) = h1 r and #E'(Fp2) = h2 r: both kill a random point
    assert o.pt_is_inf(o.FP, o.pt_mul(o.FP, _rand_g1(), H1 * R)) and o.pt_is_inf(o.FP2, o.pt_mul(o.FP2, _rand_g2(), H2 * R))


def test_torsion_points_have_exact_order():
    for q, T in T1.items():
        assert o.pt_on_curve(o.FP, T) and not o.pt_is_inf(o.FP, T) and o.pt_is_inf(o.FP, o.pt_mul(o.FP, T, q)), q
        assert not o.pt_in_subgroup(o.FP, T)
    for q, T in T2.items():
        assert o.pt_on_curve(o.FP2, T) and not o.pt_is_inf(o.FP2, T) and o.pt_is_inf(o.FP2, o.pt_mul(o.FP2, T, T2_ORDER[q])), q
        assert not o.pt_in_subgroup(o.FP2, T)
    assert o.g1_serialize(T1[3]) == X0_ODD_G1


def test_bare_pairing_accepts_key_plus_torsion():
    """Why the G1 membership test matters: e(B, sigma) == e(pk + T, H(m)) holds for a signature of pk, for every small order q.  Only
    the decoder's subgroup test tells pk + T from pk."""
    assert o.verify_hash(SIG_PT, PK_PT, MSG)
    for q, T in T1.items():
        pkT = o.pt_add(o.FP, PK_PT, T)
        assert o.verify_hash(SIG_PT, pkT, MSG), q
        assert o.g1_deserialize(o.g1_serialize(pkT)) is None and o.g1_deserialize(o.g1_serialize(pkT), check_order=False) is not None


def test_crafted_verdicts():
    """Every torsion class decodes without the order test and is rejected with it; x >= p never decodes; the sign bit picks -P; the
    identity decodes."""
    for cases, neg, dec, F in ((G1_CASES, o.pt_neg(o.FP, PK_PT), o.g1_deserialize, o.FP), (G2_CASES, o.pt_neg(o.FP2, SIG_PT), o.g2_deserialize, o.FP2)):
        got = {n: (want, plain) for n, _, want, plain in cases}
        for n, (want, plain) in got.items():
            if n.startswith(("T", "P+T", "-P+T")): assert (want, plain) == (False, True), n
            elif n in VALID_EDGES: assert (want, plain) == (True, True), n
            elif n not in UNPINNED: assert (want, plain) == (False, False), n
        flipped = dict((n, b) for n, b, _, _ in cases)["sign flipped"]
        assert o.pt_eq(F, dec(flipped), neg)
    assert dict((n, w) for n, _, w, _ in G1_CASES)["x=0 odd"] is False and dict((n, p) for n, _, _, p in G1_CASES)["x=0 odd"] is True
    assert dict((n, p) for n, _, _, p in G2_CASES)["x=0 odd"] is False


def test_pyref_against_c_oracle(oracle):
    for n, b, want, _ in G1_CASES: assert oracle.pk_check(b) == want, n
    for n, b, want, _ in G2_CASES: assert oracle.sig_check(b) == want, n


# ------------------------------------------------------------------ CPU: the device decoders on the host
def _compile(src, out, flags=()):
    csrc = os.path.join(ROOT, "harmony_b200", "csrc")
    deps = [src] + [os.path.join(csrc, f) for f in os.listdir(csrc) if f.endswith(".cuh")]
    if not os.path.exists(out) or any(os.path.getmtime(d) > os.path.getmtime(out) for d in deps):
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-pthread", *flags, "-o", out, src])
    return ctypes.CDLL(out)


@pytest.fixture(scope="module")
def emu():
    return _compile(os.path.join(ROOT, "tests", "emu", "emu_main.cpp"), os.path.join(ROOT, "tests", "emu", "libhbls_emu.so"))


@pytest.fixture(scope="module")
def emuk():
    L = _compile(os.path.join(ROOT, "tests", "emu", "emu_kernels.cpp"), os.path.join(ROOT, "tests", "emu", "libhbls_emu_kernels.so"))
    L.emu_decode_flags.argtypes = [ctypes.c_int, ctypes.c_int, ctypes.c_size_t, ctypes.c_char_p, ctypes.c_char_p]
    return L


def test_thread_deserializers_on_host(emu):
    """g1_deserialize / g2_deserialize with the order test (the code of k_single's OP_G1_DES / OP_G2_DES and of the thread decoders)."""
    assert {n: emu.emu_g1_check(b) == 1 for n, b, _, _ in G1_CASES} == {n: w for n, _, w, _ in G1_CASES}
    assert {n: emu.emu_g2_check(b) == 1 for n, b, _, _ in G2_CASES} == {n: w for n, _, w, _ in G2_CASES}


DECODE_FORMS = {0: "k_g1_decode", 1: "k_g1_decode_jac", 2: "k_single G1_DES", 3: "k_g2_decode", 4: "k_g2_decode+k_g2_subgroup",
                5: "k_g2_decode_pair", 6: "k_g2_decode_pair+k_g2_subgroup_pair", 7: "k_single G2_DES", 8: "k_single G2_DES_ADD"}


@pytest.mark.parametrize("form", sorted(DECODE_FORMS), ids=lambda f: DECODE_FORMS[f])
def test_decode_kernels_on_host(emuk, form):
    """Each decode kernel (tests/emu/emu_kernels.cpp emu_decode_flags) gives pyref's verdict on every crafted encoding; the kernels that
    can skip the order test accept exactly what decodes without it, so the rejections above are the membership test's."""
    cases = G1_CASES if form < 3 else G2_CASES
    blob = b"".join(b for _, b, _, _ in cases)
    ok = ctypes.create_string_buffer(len(cases))
    assert emuk.emu_decode_flags(form, 1, len(cases), blob, ok) == 0
    assert {n: ok.raw[i] for i, (n, _, _, _) in enumerate(cases)} == {n: int(w) for n, _, w, _ in cases}
    if form in (0, 1, 3, 5):
        assert emuk.emu_decode_flags(form, 0, len(cases), blob, ok) == 0
        assert {n: ok.raw[i] for i, (n, _, _, _) in enumerate(cases)} == {n: int(p) for n, _, _, p in cases}


def test_lane_pair_decoder_matches_thread_decoder(emuk):
    """emu_pair_decode_hash: k_g2_decode_pair == k_g2_decode (point and flag) on every crafted signature."""
    sigs = [b for _, b, _, _ in G2_CASES]
    msgs = [wl.commit_payload("sgm/lp", i) for i in range(len(sigs))]
    assert emuk.emu_pair_decode_hash(len(sigs), b"".join(sigs), b"".join(msgs), 48) & 1 == 1


# ------------------------------------------------------------------ GPU
KNOBS = ("rlc_min", "rlc_g", "tpsm", "tpsm_split", "tpsm_light", "coop_max", "overlap", "coop_wpsm", "hm_cache", "hash_coop_max",
         "mask_sort", "hash_split", "hash_fallback", "rlc_two_phase", "tpsm_cof", "tpsm_dec", "tpsm_scale", "tpsm_scale_g1",
         "scale_split", "decode_split", "exact_two_phase", "tpsm_lines", "tpsm_accum", "tpsm_sw", "rlc_block")
N = 64                                               # committee slots


@contextlib.contextmanager
def knobs(gbls, mode=1, **kv):
    saved = {k: gbls.GetParam(k) for k in KNOBS}
    saved_mode = gbls.GetBatchMode()
    try:
        gbls.SetBatchMode(mode)
        for k, v in kv.items(): gbls.SetParam(k, v)
        yield
    finally:
        for k, v in saved.items(): gbls.SetParam(k, v)
        gbls.SetBatchMode(saved_mode)
    assert {k: gbls.GetParam(k) for k in KNOBS} == saved and gbls.GetBatchMode() == saved_mode


@pytest.fixture(scope="module")
def net(oracle):
    """A committee of N keys and B rounds against it (random signer sets, distinct messages); independent triples (own key, message,
    signature)."""
    rng = random.Random(0x5b91)
    sks = [wl.seeded_sk("sgm/c", i) for i in range(N)]
    pks = [oracle.get_public_key(wl.sk_bytes(k)) for k in sks]
    B = 200
    bitmaps, msgs, sigs = [], [], []
    for j in range(B):
        members = rng.sample(range(N), rng.choice((1, 5, 40, N)))
        bm = bytearray(N // 8)
        for i in members: bm[i >> 3] |= 1 << (i & 7)
        m = wl.commit_payload("sgm/r", j)
        bitmaps.append(bytes(bm)); msgs.append(m)
        sigs.append(oracle.sign_hash(wl.sk_bytes(sum(sks[i] for i in members) % R), m))
    K = 258
    tsk = [wl.sk_bytes(wl.seeded_sk("sgm/t", j)) for j in range(K)]
    tmsg = [wl.commit_payload("sgm/t", j) for j in range(K)]
    return {"sks": sks, "pks": pks, "bitmaps": bitmaps, "msgs": msgs, "sigs": sigs, "och": oracle.committee(pks),
            "tpk": [oracle.get_public_key(s) for s in tsk], "tsig": [oracle.sign_hash(s, m) for s, m in zip(tsk, tmsg)], "tmsg": tmsg}


_verdicts = {}


def decodes(b):
    """pyref's verdict with the order test ([r]P == O), by encoding length."""
    if b not in _verdicts:
        _verdicts[b] = (o.g1_deserialize(b) if len(b) == 48 else o.g2_deserialize(b)) is not None
    return _verdicts[b]


def inject(n_rounds, crafted, seed):
    """crafted = [(name, fn(j) -> replacement)]: one seeded round each."""
    pos = random.Random(seed).sample(range(n_rounds), len(crafted))
    return dict(zip(pos, crafted))


def agg_rounds(net, seed):
    """The aggregate rounds with every crafted signature class (built from the replaced round's own signature) at seeded rounds."""
    sigs = list(net["sigs"])
    names = [n for n, _ in all_sigs(sigs[0])]
    at = inject(len(sigs), names, seed)
    for j, n in at.items(): sigs[j] = dict(all_sigs(sigs[j]))[n]
    return sigs, at


def agg_want(oracle, net, sigs, at):
    want = bytearray(b"\x01" * len(sigs))
    for j in at:
        want[j] = 1 if decodes(sigs[j]) and oracle.committee_aggregate_verify(net["och"], net["bitmaps"][j], sigs[j], net["msgs"][j]) == 1 else 0
    assert not any(want[j] for j in at)              # every crafted round fails, valid encodings (-sigma, identity) too
    return bytes(want)


@pytest.mark.gpu
def test_part1_deserialize(gbls):
    """blsPublicKeyDeserialize / blsSignatureDeserialize (k_single): ValueError exactly where pyref rejects; -P for the sign bit."""
    for cases, cls in ((G1_CASES, gbls.PublicKey), (G2_CASES, gbls.Sign)):
        for n, b, want, _ in cases:
            x = cls()
            if want:
                x.Deserialize(b); assert x.Serialize() == b, n
            else:
                with pytest.raises(ValueError): x.Deserialize(b)


@pytest.mark.gpu
def test_committee_names_first_bad_key(gbls, net):
    rng = random.Random(7)
    for k, (n, _) in enumerate(all_keys(net["pks"][0])):
        if n in VALID_EDGES: continue
        pks = list(net["pks"])
        first, second = sorted(rng.sample(range(N), 2))
        pks[first] = dict(all_keys(pks[first]))[n]; pks[second] = dict(all_keys(pks[second]))[n]
        with pytest.raises(ValueError, match=rf"index {first}$"): gbls.Committee(pks)
    assert len(gbls.Committee(net["pks"])) == N


_VB_FORMS = {"latency": {}, "thread": {"coop_max": 0}, "groups": {"rlc_min": 16}}


@pytest.mark.gpu
@pytest.mark.parametrize("form", sorted(_VB_FORMS))
def test_verify_batch_status(gbls, oracle, net, form):
    """Triples with every crafted key class (pk + T: VB_BAD_KEY_ENCODING) and every crafted signature class (VB_BAD_SIG_ENCODING),
    each built from the replaced triple's own key or signature; every honest triple VB_OK."""
    pks, sigs, msgs = list(net["tpk"]), list(net["tsig"]), net["tmsg"]
    K = len(pks)
    crafted = [("key", n) for n, _ in all_keys(pks[0])] + [("sig", n) for n, _ in all_sigs(sigs[0])]
    at = inject(K, crafted, 11)
    for j, (kind, n) in at.items():
        if kind == "key": pks[j] = dict(all_keys(pks[j]))[n]
        else: sigs[j] = dict(all_sigs(sigs[j]))[n]
    want = bytearray([gbls.VB_OK] * K)
    for j in at:
        want[j] = (gbls.VB_BAD_KEY_ENCODING if not decodes(pks[j]) else gbls.VB_BAD_SIG_ENCODING if not decodes(sigs[j])
                   else gbls.VB_OK if oracle.verify_hash(sigs[j], pks[j], msgs[j]) else gbls.VB_BAD_SIG)
        assert want[j] != gbls.VB_OK, at[j]
        assert want[j] == (gbls.VB_BAD_SIG if at[j][1] in VALID_EDGES else gbls.VB_BAD_KEY_ENCODING if at[j][0] == "key" else gbls.VB_BAD_SIG_ENCODING)
    with knobs(gbls, **_VB_FORMS[form]):
        st = gbls.VerifyBatchStatus(b"".join(pks), b"".join(sigs), b"".join(msgs), 48)
        info = gbls.LastBatchInfo()
        res = gbls.VerifyBatch(b"".join(pks), b"".join(sigs), b"".join(msgs), 48)
    assert {j: (at.get(j), st[j]) for j in range(K) if st[j] != want[j]} == {}
    assert res == bytes(1 if w == gbls.VB_OK else 0 for w in want)
    assert info["mode"] == (1 if form == "groups" else 0)


_AV_FORMS = {"latency": {}, "thread_decode_split0": {"coop_max": 0, "decode_split": 0}, "thread_decode_split1": {"coop_max": 0, "decode_split": 1},
             "groups_of_4": {"rlc_min": 16, "rlc_g": 4}, "groups_of_8": {"rlc_min": 16, "rlc_g": 8}, "blocks": {"rlc_min": 16, "rlc_g": 4, "rlc_block": 1}}


@pytest.mark.gpu
@pytest.mark.parametrize("form", sorted(_AV_FORMS))
def test_aggregate_verify_batch(gbls, oracle, net, form):
    """sigma + T (and the signature edges) at seeded rounds of a batch: exactly those rounds fail, and in the batched forms exactly the
    groups that hold one."""
    sigs, at = agg_rounds(net, 21)
    want = agg_want(oracle, net, sigs, at)
    com = gbls.Committee(net["pks"])
    B = len(sigs)
    with knobs(gbls, **_AV_FORMS[form]):
        res = com.AggregateVerifyBatch(b"".join(net["bitmaps"]), b"".join(sigs), b"".join(net["msgs"]), 48)
        info = gbls.LastBatchInfo()
    assert {j: (at.get(j), res[j]) for j in range(B) if res[j] != want[j]} == {}
    if form.startswith(("groups", "blocks")):
        G = _AV_FORMS[form]["rlc_g"]; ng = B // G
        failed = {j % ng for j in at if j < G * ng}
        assert (info["mode"], info["group_size"], info["groups"]) == (1, G, ng)
        assert info["groups_failed"] == len(failed) and info["rounds_rechecked"] == G * len(failed)
    else:
        assert info["mode"] == 0


@pytest.mark.gpu
def test_warm_hash_cache_path(gbls, oracle, net):
    """H(m) cached (SignHash on the message first): k_g2_decode_pair skips the order test, k_miller_pq_coop consumes the point and
    k_g2_subgroup_pair decides afterwards.  AggregateVerify, a same-message AggregateVerifyBatch and DeviceMask.VerifyHash reject every
    crafted signature, warm and cold, and pass the honest ones; VerifyHeaders (one header, and a same-message range) reports the
    encoding error."""
    import torch
    from torch.profiler import profile, ProfilerActivity
    sks, bm = net["sks"], net["bitmaps"][3]
    signers = [i for i in range(N) if bm[i >> 3] >> (i & 7) & 1]
    msg = wl.commit_payload("sgm/warm", 0)
    agg = wl.sk_bytes(sum(sks[i] for i in signers) % R)
    sig = oracle.sign_hash(agg, msg)
    crafted = all_sigs(sig)
    com = gbls.Committee(net["pks"]); dm = gbls.DeviceMask(com); dm.SetMask(bm)
    # a same-message batch: round j signed by member j alone, crafted signatures of those rounds at seeded positions
    Bm = 40
    bms = [bytes(1 << (i & 7) if k == i >> 3 else 0 for k in range(N // 8)) for i in range(Bm)]
    bsig = [oracle.sign_hash(wl.sk_bytes(sks[i]), msg) for i in range(Bm)]
    bat = inject(Bm, [n for n, _ in crafted], 31)
    for j, n in bat.items(): bsig[j] = dict(all_sigs(bsig[j]))[n]
    bwant = bytes(0 if j in bat else 1 for j in range(Bm))
    for hm in (1, 0):
        with knobs(gbls, hm_cache=hm, overlap=1):
            sk = gbls.SecretKey(); sk.Deserialize(agg)
            assert sk.SignHash(msg).Serialize() == sig                  # puts H(msg) in the cache (hm_cache = 1)
            h0 = gbls.HashCacheStats()["hits"]
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                assert com.AggregateVerify(bm, sig, msg) is True
                torch.cuda.synchronize()
            kern = [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
            assert (gbls.HashCacheStats()["hits"] > h0) == bool(hm)
            assert any("k_g2_subgroup_pair" in k for k in kern) == bool(hm) and any("k_miller_pq_coop" in k for k in kern) == bool(hm), kern
            for n, b in crafted:
                assert com.AggregateVerify(bm, b, msg) is False, (hm, n)
                assert dm.VerifyHash(b, msg) is False, (hm, n)
                # the pairing rejects sigma + T by itself: only the status tells that the membership test did
                want = gbls.HDR_BAD_SIG if decodes(b) else gbls.HDR_BAD_ENCODING
                assert com.VerifyHeaders(b, bm, msg, 48, 0) == bytes([want]), (hm, n)
            assert dm.VerifyHash(sig, msg) is True
            res = com.AggregateVerifyBatch(b"".join(bms), b"".join(bsig), msg * Bm, 48)
            assert {j: (bat.get(j), res[j]) for j in range(Bm) if res[j] != bwant[j]} == {}, hm
            st = com.VerifyHeaders(b"".join(bsig), b"".join(bms), msg * Bm, 48, 0)
            swant = bytes(gbls.HDR_OK if j not in bat else gbls.HDR_BAD_SIG if decodes(bsig[j]) else gbls.HDR_BAD_ENCODING for j in range(Bm))
            assert {j: (bat.get(j), st[j]) for j in range(Bm) if st[j] != swant[j]} == {}, hm
            assert (gbls.HashCacheStats()["hits"] > h0) == bool(hm)


@pytest.mark.gpu
def test_aggregate_sigs_and_add_vote(gbls, oracle, net):
    """AggregateSigBytes raises on any crafted signature among honest ones; BallotBox.AddVote raises and leaves the box as it was."""
    honest = net["sigs"][:5]
    com = gbls.Committee(net["pks"]); box = gbls.BallotBox(com)
    one = bytearray(N // 8); one[0] = 1
    assert box.AddVote(bytes(one), honest[0]) is True
    for k, (n, b) in enumerate(all_sigs(honest[1])):
        if n in VALID_EDGES: continue
        with pytest.raises(ValueError): gbls.AggregateSigBytes(honest[:2] + [b] + honest[2:])
        bm = bytearray(N // 8); bm[1] = 1 << (k % 8)             # a slot not yet collected: the decode decides
        with pytest.raises(ValueError): box.AddVote(bytes(bm), b)
    assert gbls.AggregateSigBytes(honest) == oracle.aggregate_sigs(honest)
    assert box.Aggregate() == (honest[0], bytes(one))


_SV_FORMS = {"lane_pair_warm": {}, "lane_pair_cold": {"hm_cache": 0}, "thread_split": {"coop_max": 32}, "thread": {"coop_max": 32, "decode_split": 0}}


@pytest.mark.gpu
@pytest.mark.parametrize("form", sorted(_SV_FORMS))
def test_submit_votes(gbls, oracle, net, form):
    """A queue of N votes, one distinct member each, with every crafted signature class at seeded votes: BALLOT_BAD_SIG_ENCODING (the
    valid edges BALLOT_BAD_SIG), the honest votes accepted and folded.  64 votes: within coop_max (lane-pair decode; warm when H(m) is
    cached) and past it (coop_max = 32: k_g2_decode with or without k_g2_subgroup)."""
    ACC, BENC, BSIG = gbls.BALLOT_ACCEPTED, gbls.BALLOT_BAD_SIG_ENCODING, gbls.BALLOT_BAD_SIG
    msg = wl.commit_payload("sgm/vq", 0)
    bms = [bytes(1 << (i & 7) if k == i >> 3 else 0 for k in range(N // 8)) for i in range(N)]
    sigs = [oracle.sign_hash(wl.sk_bytes(net["sks"][i]), msg) for i in range(N)]
    at = inject(N, [n for n, _ in all_sigs(sigs[0])], 41)
    for j, n in at.items(): sigs[j] = dict(all_sigs(sigs[j]))[n]
    want = bytes((BSIG if at[j] in VALID_EDGES else BENC) if j in at else ACC for j in range(N))
    assert all(decodes(sigs[j]) == (at[j] in VALID_EDGES) for j in at)
    with knobs(gbls, **_SV_FORMS[form]):
        gbls.HashPrefetch(msg)
        box = gbls.BallotBox(gbls.Committee(net["pks"]))
        st = box.SubmitVotes(bms, sigs, msg)
    assert {j: (at.get(j), st[j]) for j in range(N) if st[j] != want[j]} == {}
    honest = [j for j in range(N) if j not in at]
    collected = sum(1 << j for j in honest).to_bytes(N // 8, "little")
    assert box.Aggregate() == (oracle.aggregate_sigs([sigs[j] for j in honest]), collected)


@pytest.mark.gpu
def test_verify_headers_and_items(gbls, oracle, net):
    sigs, at = agg_rounds(net, 51)
    want = agg_want(oracle, net, sigs, at)
    com = gbls.Committee(net["pks"])
    B = len(sigs)
    with knobs(gbls):
        st = com.VerifyHeaders(b"".join(sigs), b"".join(net["bitmaps"]), b"".join(net["msgs"]), 48, 0)
        items = gbls.AggregateVerifyItems([com] * B, net["bitmaps"], b"".join(sigs), b"".join(net["msgs"]), 48)
    hwant = bytes(gbls.HDR_OK if j not in at else gbls.HDR_BAD_SIG if decodes(sigs[j]) else gbls.HDR_BAD_ENCODING for j in range(B))
    assert {j: (at.get(j), st[j]) for j in range(B) if st[j] != hwant[j]} == {}
    assert items == want


@pytest.mark.gpu
def test_rlc_partial_fold_and_split(gbls, net):
    """A slice holding one crafted key or signature is never proved by RlcPartial / RlcFold; verify_triples_split then gives the exact
    booleans."""
    from harmony_b200 import shard
    S = 8
    pks, sigs, msgs = net["tpk"][:S], net["tsig"][:S], net["tmsg"][:S]
    blob = lambda x: b"".join(x)
    clean = gbls.RlcPartial(blob(pks), blob(sigs), blob(msgs), 48)
    with knobs(gbls):
        assert gbls.RlcFold([clean]) is True
        for kind, cases in (("key", all_keys), ("sig", all_sigs)):
            for k, (n, _) in enumerate(cases(pks[0] if kind == "key" else sigs[0])):
                p2, s2 = list(pks), list(sigs); j = k % S
                if kind == "key": p2[j] = dict(cases(p2[j]))[n]
                else: s2[j] = dict(cases(s2[j]))[n]
                rec = gbls.RlcPartial(blob(p2), blob(s2), blob(msgs), 48)
                assert gbls.RlcFold([rec]) is False and gbls.RlcFold([clean, rec]) is False, (kind, n)
        K = len(net["tpk"])
        p2, s2 = list(net["tpk"]), list(net["tsig"])
        at = inject(K, [("key", n) for n, _ in all_keys(p2[0])] + [("sig", n) for n, _ in all_sigs(s2[0])], 61)
        for j, (kind, n) in at.items():
            if kind == "key": p2[j] = dict(all_keys(p2[j]))[n]
            else: s2[j] = dict(all_sigs(s2[j]))[n]
        res, settled = shard.verify_triples_split(blob(p2), blob(s2), blob(net["tmsg"]), 48)
    assert settled is False
    assert res == bytes(0 if j in at else 1 for j in range(K))
