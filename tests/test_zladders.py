"""The |z| ladders with an affine base give the outputs of the ladders they replace.

hbls.cu runs the subgroup test of the split signature decode (k_g2_subgroup_pair: g2_in_subgroup_aff, whose |z| ladder adds its affine
base with mixed additions) and the cofactor clearing of hash-to-G2 (k_hash_cofactor_z1_pair + k_hash_cofactor_z2_pair: RFC 9380's order
of the Budroni-Pintore combination, one |z| ladder per kernel, three live points).  The subgroup kernel keeps its outputs, so its flags
and zeroed points must equal those of the thread kernel k_g2_subgroup byte for byte.  The new cofactor clearing gives the same group
element as k_hash_cofactor_pair but may give another Jacobian representative, so the two are compared after k_g2_normalize_batch: the
affine H(m) bytes must agree.

Inputs: valid signatures, points of small order of E'(Fp2) (one per prime of the G2 cofactor, and the large prime part of it), P + T and
-P + T for a signature P, random curve points outside G2, the identity, undecodable encodings, SW-map outputs of messages, dropped ok
flags, and batch sizes that are not a multiple of a warp.  The expected subgroup flags come from the input classes.

CPU: the kernels on the host (tests/emu/emu_zladders.cpp, a lane pair on two host threads).
GPU: the same comparison on the device (tests/zladders/zladders_driver.cu, compiled here with nvcc for sm_90a) on 4 109 points and
4 109 messages, with the CTA sizes the resident-thread settings tpsm_sub / tpsm_cof can give."""
import ctypes, os, random, subprocess, sys, tempfile
import pytest
from harmony_b200 import workload as wl

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "oracle"))
import pyref as o                                   # noqa: E402

_BUILD = tempfile.mkdtemp(prefix="hbls_zladders_")
Z, R = o.Z, o.R
H2 = (Z ** 8 - 4 * Z ** 7 + 5 * Z ** 6 - 4 * Z ** 4 + 6 * Z ** 3 - 4 * Z ** 2 - 4 * Z + 13) // 9


def _small_factors(n, bound):
    small = {}
    for d in range(2, bound):
        while n % d == 0:
            small[d] = small.get(d, 0) + 1
            n //= d
    return small, n


def _rand_curve_g2(rng):
    while True:
        x = (rng.randrange(o.P), rng.randrange(o.P)); y = o.f2_sqrt(o.f2_add(o.f2_mul(o.f2_sqr(x), x), o.B2))
        if y is not None: return o.pt_from_affine(o.FP2, x, y)


def _torsion(rng):
    """a point of exact order q for every prime q^e || h2, and one of order the large prime part of h2"""
    small, large = _small_factors(H2, 1 << 19)
    out = []
    for q, e in small.items():
        while True:
            T = o.pt_mul(o.FP2, _rand_curve_g2(rng), H2 * R // q ** e)
            if not o.pt_is_inf(o.FP2, T): break
        while not o.pt_is_inf(o.FP2, o.pt_mul(o.FP2, T, q)): T = o.pt_mul(o.FP2, T, q)
        out.append(T)
    while True:
        T = o.pt_mul(o.FP2, _rand_curve_g2(rng), R * (H2 // large))
        if not o.pt_is_inf(o.FP2, T): return out + [T]


@pytest.fixture(scope="module")
def classes(oracle):
    """(serialized point, in G2) pools: valid signatures, torsion points alone and added to +-signature, random curve points outside
    G2, the identity, x = p"""
    rng = random.Random(0x2a1)
    sks = [wl.seeded_sk("zl", i) for i in range(8)]
    sigs = [oracle.sign_hash(wl.sk_bytes(k), wl.commit_payload("zl", i)) for i, k in enumerate(sks)]
    good = [(s, True) for s in sigs] + [(bytes(96), True)]
    bad = [(o.P.to_bytes(48, "little") + sigs[0][48:], False)]
    for j, T in enumerate(_torsion(rng)):
        P = o.g2_deserialize(sigs[j % len(sigs)])
        bad += [(o.g2_serialize(T), False), (o.g2_serialize(o.pt_add(o.FP2, P, T)), False),
                (o.g2_serialize(o.pt_add(o.FP2, o.pt_neg(o.FP2, P), T)), False)]
    bad += [(o.g2_serialize(_rand_curve_g2(rng)), False) for _ in range(3)]
    return good, bad


def make_items(classes, n, seed):
    """n serialized points (every class outside G2 once, then a seeded mix), the expected subgroup flags, n messages, and
    drop flags for 2n items (points then messages)"""
    good, bad = classes
    rng = random.Random(seed)
    pick = list(bad)
    while len(pick) < n: pick.append(rng.choice(good) if rng.random() < 0.6 else rng.choice(bad))
    rng.shuffle(pick)
    drop = bytes(1 if rng.random() < 0.1 else 0 for _ in range(2 * n))
    want = bytes(1 if ing and not drop[i] else 0 for i, (_, ing) in enumerate(pick))
    msgs = b"".join(wl.commit_payload("zl%d" % seed, j) for j in range(n))
    return b"".join(p for p, _ in pick), want, msgs, drop


# ------------------------------------------------------------------ CPU: host emulation
@pytest.fixture(scope="module")
def emul():
    src = os.path.join(ROOT, "tests", "emu", "emu_zladders.cpp")
    out = os.path.join(_BUILD, "libemu_zladders.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-pthread", "-o", out, src])
    L = ctypes.CDLL(out)
    L.emu_zl_subgroup.argtypes = [ctypes.c_size_t, ctypes.c_char_p, ctypes.c_char_p, ctypes.c_char_p]
    L.emu_zl_cofactor.argtypes = [ctypes.c_size_t, ctypes.c_char_p, ctypes.c_size_t, ctypes.c_char_p, ctypes.c_uint32, ctypes.c_char_p,
                                  ctypes.c_char_p]
    return L


def test_emu_subgroup_pair_matches_thread_kernel(emul, classes):
    pts, want, msgs, drop = make_items(classes, 37, 0x31)
    n = len(want)
    ok = ctypes.create_string_buffer(n)
    assert emul.emu_zl_subgroup(n, pts, drop, ok) == 0
    assert ok.raw[:n] == want and 0 < sum(want) < n


def test_emu_cofactor_z_pairs_match_pair_kernel(emul, classes):
    pts, want, msgs, drop = make_items(classes, 29, 0x32)
    n = len(want)
    ok = ctypes.create_string_buffer(2 * n)
    assert emul.emu_zl_cofactor(n, pts, n, msgs, 48, drop, ok) == 0
    assert 0 < sum(ok.raw[:2 * n]) < 2 * n and sum(drop) > 0


# ------------------------------------------------------------------ GPU: the kernels on the device
@pytest.fixture(scope="module")
def driver():
    src = os.path.join(ROOT, "tests", "zladders", "zladders_driver.cu")
    out = os.path.join(_BUILD, "libzladders_driver.so")
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    subprocess.check_call([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-Xcompiler", "-fPIC", "-shared", "-o", out, src])
    L = ctypes.CDLL(out)
    L.zl_subgroup.argtypes = [ctypes.c_size_t, ctypes.c_char_p, ctypes.c_char_p, ctypes.c_uint, ctypes.c_char_p]
    L.zl_cofactor.argtypes = [ctypes.c_size_t, ctypes.c_char_p, ctypes.c_size_t, ctypes.c_char_p, ctypes.c_uint32, ctypes.c_char_p,
                              ctypes.c_uint, ctypes.c_char_p]
    return L


@pytest.fixture(scope="module")
def big(classes):
    return make_items(classes, 4109, 0x33)


@pytest.mark.gpu
@pytest.mark.parametrize("cta", [256, 384, 512])
def test_gpu_zladders_match_current_kernels(driver, big, cta):
    pts, want, msgs, drop = big
    n = len(want)
    ok = ctypes.create_string_buffer(2 * n)
    assert driver.zl_subgroup(n, pts, drop, cta, ok) == 0
    assert ok.raw[:n] == want
    assert driver.zl_cofactor(n, pts, n, msgs, 48, drop, cta, ok) == 0
    assert 0 < sum(ok.raw[:2 * n]) < 2 * n
