"""The joint per-group ladder of the coefficient stage gives the group sums and bad flags of the per-round form it replaces.

For batches whose groups fill the chip, hbls.cu scales the signatures with k_rlc_group_scale_g2_pair: one lane pair per group runs ONE
ladder over the group's 2G half-scalars (pt_mul_joint_naf) into the Jacobian sum Sg, and k_g2_normalize_batch turns it affine.
Smaller batches keep a ladder per round (k_rlc_scale_g2_pair; its reference k_rlc_scale_g2) and k_rlc_group_sum<G>.  The group law
is exact, so both give the same group element, whose affine form is unique: every byte of Sg and every bad flag must agree.

CPU: the kernels on the host (tests/emu/emu_group_scale.cpp, a lane pair on two host threads): G = 4 and 8, group and block
coefficients with the unit one, gates, undecodable and identity signatures, identity keys and H(m), and degenerate sums (equal
signatures, sigma and -sigma, a signature equal to the running sum); the executed Fp products of both forms.
GPU: the same comparison on the device (tests/lane_pair/group_scale_driver.cu, compiled with nvcc for sm_90a) on 4 096 rounds with
bad ones, each kernel launched with the geometry hbls.cu gives it."""
import ctypes, os, random, subprocess, sys, tempfile
import pytest
from harmony_b200 import workload as wl

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "oracle"))
import pyref as o                                   # noqa: E402

_BUILD = tempfile.mkdtemp(prefix="hbls_group_scale_")
_NCO = 8 + 8 * 16


def _neg(sig):
    return o.g2_serialize(o.pt_neg(o.FP2, o.g2_deserialize(sig, False)))


def _add(s1, s2):
    return o.g2_serialize(o.pt_add(o.FP2, o.g2_deserialize(s1, False), o.g2_deserialize(s2, False)))


def make_items(oracle, n, seed, bad=True):
    """n rounds (key, signature, 48-byte message); with bad: undecodable (x >= p) and identity signatures, identity keys and messages
    whose map is undefined (H(m) = identity) at seeded positions"""
    rng = random.Random(seed)
    sks = [wl.seeded_sk("gsc", i) for i in range(16)]
    pks = [oracle.get_public_key(wl.sk_bytes(k)) for k in sks]
    keys, sigs, msgs = [], [], []
    for j in range(n):
        k = rng.randrange(16); m = wl.commit_payload("gsc%d" % seed, j)
        c = rng.randrange(12) if bad else -1
        if c == 3: m = bytes(48)                     # t = 0: the map is undefined
        s = oracle.sign_hash(wl.sk_bytes(sks[k]), m) if c != 3 else oracle.sign_hash(wl.sk_bytes(sks[k]), b"x" * 48)
        if c == 0: s = o.P.to_bytes(48, "little") + s[48:]
        elif c == 1: s = bytes(96)
        keys.append(bytes(48) if c == 2 else pks[k]); sigs.append(s); msgs.append(m)
    return keys, sigs, msgs


def coeffs(seed, unit=False):
    rng = random.Random(seed)
    return (ctypes.c_uint64 * _NCO)(*([1] * _NCO if unit else [rng.getrandbits(64) for _ in range(_NCO)]))


# ------------------------------------------------------------------ CPU: host emulation
@pytest.fixture(scope="module")
def emul():
    src = os.path.join(ROOT, "tests", "emu", "emu_group_scale.cpp")
    out = os.path.join(_BUILD, "libemu_group_scale.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-pthread", "-o", out, src])
    L = ctypes.CDLL(out)
    L.emu_group_scale.argtypes = [ctypes.c_int, ctypes.c_size_t, ctypes.c_char_p, ctypes.c_char_p, ctypes.c_char_p, ctypes.c_uint32,
                                  ctypes.c_size_t, ctypes.POINTER(ctypes.c_uint64), ctypes.c_int, ctypes.c_int, ctypes.c_char_p, ctypes.c_char_p]
    L.emu_group_scale_counts.argtypes = [ctypes.c_int, ctypes.c_size_t, ctypes.c_char_p, ctypes.POINTER(ctypes.c_uint64),
                                         ctypes.POINTER(ctypes.c_uint64)]
    return L


def run_emu(L, G, keys, sigs, msgs, co, blocks=0, gate=-1):
    n = len(msgs); ng = n // G
    bad = ctypes.create_string_buffer(n); sg = ctypes.create_string_buffer(192 * ng)
    diff = L.emu_group_scale(G, n, b"".join(keys), b"".join(sigs), b"".join(msgs), 48, ng, co, blocks, gate, bad, sg)
    return diff, bad.raw[:n], [sg.raw[192 * g:192 * g + 192] for g in range(ng)]


def want_bad(keys, sigs, msgs, oracle):
    return bytes(1 if (k == bytes(48) or s == bytes(96) or oracle.map_to_g2(m) is None or not oracle.sig_check(s)) else 0
                 for k, s, m in zip(keys, sigs, msgs))


@pytest.mark.parametrize("G", [4, 8])
@pytest.mark.parametrize("blocks,gate", [(0, -1), (1, -1), (1, 1), (1, 0)])
def test_emu_joint_matches_per_round(emul, oracle, G, blocks, gate):
    keys, sigs, msgs = make_items(oracle, 8 * G, 0x65 + G)
    diff, bad, _ = run_emu(emul, G, keys, sigs, msgs, coeffs(G + 3 * blocks + gate), blocks, gate)
    assert diff == 0
    assert bad == want_bad(keys, sigs, msgs, oracle) and 0 < sum(bad) < len(msgs)


@pytest.mark.parametrize("G", [4, 8])
def test_emu_joint_degenerate_sums(emul, oracle, G):
    """group 0: two equal signatures; group 1: sigma and -sigma; group 2: all signatures equal (the running sum meets +-sigma);
    group 3: the third signature is the sum of the first two; group 4: identity signatures only"""
    ng = 6
    keys, sigs, msgs = make_items(oracle, ng * G, 0x77 + G, bad=False)
    at = lambda g, k: k * ng + g                     # round of position k in group g
    sigs[at(0, 2)] = sigs[at(0, 1)]
    sigs[at(1, 3)] = _neg(sigs[at(1, 0)])
    for k in range(1, G): sigs[at(2, k)] = sigs[at(2, 0)]
    sigs[at(3, 2)] = _add(sigs[at(3, 0)], sigs[at(3, 1)])
    for k in range(G): sigs[at(4, k)] = bytes(96)
    for co in (coeffs(0x99 + G), coeffs(0, unit=True)):
        diff, bad, sg = run_emu(emul, G, keys, sigs, msgs, co)
        assert diff == 0
        assert bad == want_bad(keys, sigs, msgs, oracle)
    # unit coefficients everywhere: Sg is the plain sum of the group's signatures, checked against the big-integer oracle
    for g in range(ng):
        acc = o.pt_inf(o.FP2)
        for k in range(G): acc = o.pt_add(o.FP2, acc, o.g2_deserialize(sigs[at(g, k)], False))
        a = o.pt_affine(o.FP2, acc)
        want = bytes(192) if a is None else b"".join(v.to_bytes(48, "little") for v in (a[0][0], a[0][1], a[1][0], a[1][1]))
        assert sg[g] == want, g
    assert sg[4] == bytes(192)


def test_emu_joint_counts(emul, oracle):
    """executed Fp products of the stage's G2 side on valid signatures in groups of 8 (the benchmark's G) with random coefficients:
    the joint ladder needs at least 30 % fewer than a ladder per round plus the group sums"""
    G = 8
    _, sigs, _ = make_items(oracle, 4 * G, 0x5ca1e, bad=False)
    per_round = joint = 0
    for seed in range(6):
        out = (ctypes.c_uint64 * 4)()
        assert emul.emu_group_scale_counts(G, len(sigs), b"".join(sigs), coeffs(0xc0 + seed), out) == 0
        per_round += out[0] + out[1]; joint += out[2] + out[3]
    assert joint <= 0.7 * per_round, (joint, per_round)


# ------------------------------------------------------------------ GPU: the kernels on the device
@pytest.fixture(scope="module")
def driver():
    src = os.path.join(ROOT, "tests", "lane_pair", "group_scale_driver.cu")
    out = os.path.join(_BUILD, "libgroup_scale_driver.so")
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    subprocess.check_call([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-Xcompiler", "-fPIC", "-shared", "-o", out, src])
    L = ctypes.CDLL(out)
    L.gs_compare.argtypes = [ctypes.c_size_t, ctypes.c_char_p, ctypes.c_char_p, ctypes.c_char_p, ctypes.c_uint32, ctypes.c_size_t,
                             ctypes.POINTER(ctypes.c_uint64), ctypes.c_int]
    return L


@pytest.mark.gpu
def test_gpu_joint_matches_per_round(driver, oracle):
    keys, sigs, msgs = make_items(oracle, 4096, 0x3d1)
    at = lambda g, k, ng: k * ng + g
    for G in (4, 8):
        ng = 4096 // G
        s = list(sigs)
        g1, g2 = [g for g in range(ng) if all(o.g2_deserialize(s[at(g, k, ng)], False) for k in range(G))][:2]
        s[at(g1, 2, ng)] = s[at(g1, 1, ng)]; s[at(g2, 3, ng)] = _neg(s[at(g2, 0, ng)])          # equal signatures; sigma and -sigma
        for blocks in (0, 1):
            for co in (coeffs(0x10 + G + blocks), coeffs(0, unit=True)):
                assert driver.gs_compare(4096, b"".join(keys), b"".join(s), b"".join(msgs), 48, ng, co, blocks) == 0, (G, blocks)
