"""The large-batch G2 ladders on the lane-pair carrier give bit-for-bit the outputs of the thread-per-item kernels they replace.

hbls.cu runs the subgroup test of the split signature decode (k_g2_subgroup_pair, zeroing rejected points), the cofactor clearing of
hash-to-G2 (k_hash_cofactor_pair) and the signature side of the coefficient scaling (k_rlc_scale_g2_pair) one item per lane pair.
The thread kernels (k_g2_subgroup, k_hash_cofactor_jac, k_rlc_scale_g2) stay in kernels.cuh as the reference.  Both forms run the
same formulas over canonical field elements, so every Jacobian coordinate, flag and zeroed point must agree byte for byte.

CPU: the kernels on the host (tests/emu/emu_ladders.cpp, a lane pair on two host threads): random inputs, the identity, undecodable
and out-of-subgroup items, the unit coefficient of position 0, group and block coefficients.
GPU: the same comparison on the device (tests/lane_pair/ladders_driver.cu, compiled here with nvcc for sm_90a) on 4 096 items with
mixed invalid ones, each kernel launched with the geometry hbls.cu gives it."""
import ctypes, os, random, subprocess, sys, tempfile
import pytest
from harmony_b200 import workload as wl

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "harmony_b200", "csrc")
sys.path.insert(0, os.path.join(ROOT, "oracle"))
import pyref as o                                   # noqa: E402

_BUILD = tempfile.mkdtemp(prefix="hbls_lane_pair_")


def _rand_curve_g2(rng):
    """a point of E'(Fp2) with a random x: outside G2 with overwhelming probability (checked)"""
    while True:
        x = (rng.randrange(o.P), rng.randrange(o.P)); y = o.f2_sqrt(o.f2_add(o.f2_mul(o.f2_sqr(x), x), o.B2))
        if y is not None:
            p = o.pt_from_affine(o.FP2, x, y)
            if not o.pt_in_subgroup(o.FP2, p): return o.g2_serialize(p)


def make_items(oracle, n, seed):
    """n rounds (key, signature, 48-byte message) with invalid items at seeded positions: signatures outside the subgroup, not
    decodable (x >= p) or the identity, identity keys, and messages whose map output is dropped (drop flags)."""
    rng = random.Random(seed)
    sks = [wl.seeded_sk("lpl", i) for i in range(16)]
    pks = [oracle.get_public_key(wl.sk_bytes(k)) for k in sks]
    off_curve = [_rand_curve_g2(rng) for _ in range(3)]
    keys, sigs, msgs, drop = [], [], [], []
    for j in range(n):
        k = rng.randrange(16); m = wl.commit_payload("lpl%d" % seed, j)
        s = oracle.sign_hash(wl.sk_bytes(sks[k]), m)
        c = rng.randrange(16)
        if c == 0: s = off_curve[j % 3]
        elif c == 1: s = o.P.to_bytes(48, "little") + s[48:]
        elif c == 2: s = bytes(96)
        keys.append(bytes(48) if c == 3 else pks[k]); sigs.append(s); msgs.append(m); drop.append(1 if c == 4 else 0)
    return b"".join(keys), b"".join(sigs), b"".join(msgs), bytes(drop)


def coeffs(seed):
    rng = random.Random(seed)
    return (ctypes.c_uint64 * (8 + 8 * 16))(*[rng.getrandbits(64) for _ in range(8 + 8 * 16)])


# ------------------------------------------------------------------ CPU: host emulation
@pytest.fixture(scope="module")
def emul():
    src = os.path.join(ROOT, "tests", "emu", "emu_ladders.cpp")
    out = os.path.join(_BUILD, "libemu_ladders.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-pthread", "-o", out, src])
    L = ctypes.CDLL(out)
    L.emu_ladder_subgroup.argtypes = [ctypes.c_size_t, ctypes.c_char_p, ctypes.c_char_p]
    L.emu_ladder_cofactor.argtypes = [ctypes.c_size_t, ctypes.c_char_p, ctypes.c_uint32, ctypes.c_char_p]
    L.emu_ladder_scale.argtypes = [ctypes.c_size_t, ctypes.c_char_p, ctypes.c_char_p, ctypes.c_char_p, ctypes.c_uint32, ctypes.c_size_t,
                                   ctypes.c_uint64, ctypes.c_int]
    return L


@pytest.fixture(scope="module")
def items(oracle):
    return make_items(oracle, 64, 0x1a9)


def test_emu_subgroup_pair_matches_thread_kernel(emul, items):
    keys, sigs, msgs, drop = items
    n = len(msgs) // 48
    ok = ctypes.create_string_buffer(n)
    assert emul.emu_ladder_subgroup(n, sigs, ok) == 0
    want = bytes(1 if o.g2_deserialize(sigs[96 * i:96 * i + 96]) is not None else 0 for i in range(n))
    assert ok.raw[:n] == want and 0 < sum(want) < n


def test_emu_cofactor_pair_matches_thread_kernel(emul, items):
    keys, sigs, msgs, drop = items
    n = len(msgs) // 48
    assert 0 < sum(drop) < n
    assert emul.emu_ladder_cofactor(n, msgs, 48, drop) == 0


@pytest.mark.parametrize("blocks", [0, 1])
def test_emu_scale_pair_matches_thread_kernel(emul, items, blocks):
    keys, sigs, msgs, drop = items
    n = len(msgs) // 48
    for G in (4, 8):                          # groups of G: rounds j < n / G sit at position 0 (unit coefficient in group 0 / member 0)
        assert emul.emu_ladder_scale(n, keys, sigs, msgs, 48, n // G, 0x5eed + G, blocks) == 0


# ------------------------------------------------------------------ GPU: the kernels on the device
@pytest.fixture(scope="module")
def driver():
    src = os.path.join(ROOT, "tests", "lane_pair", "ladders_driver.cu")
    out = os.path.join(_BUILD, "libladders_driver.so")
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    subprocess.check_call([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-Xcompiler", "-fPIC", "-shared", "-o", out, src])
    L = ctypes.CDLL(out)
    L.lp_subgroup.argtypes = [ctypes.c_size_t, ctypes.c_char_p, ctypes.c_char_p]
    L.lp_cofactor.argtypes = [ctypes.c_size_t, ctypes.c_char_p, ctypes.c_uint32, ctypes.c_char_p]
    L.lp_scale.argtypes = [ctypes.c_size_t, ctypes.c_char_p, ctypes.c_char_p, ctypes.c_char_p, ctypes.c_uint32, ctypes.c_size_t,
                           ctypes.POINTER(ctypes.c_uint64), ctypes.c_int]
    return L


@pytest.fixture(scope="module")
def big(oracle):
    return make_items(oracle, 4096, 0x2b7)


@pytest.mark.gpu
def test_gpu_lane_pair_ladders_match_thread_kernels(driver, big):
    keys, sigs, msgs, drop = big
    n = len(msgs) // 48
    ok = ctypes.create_string_buffer(n)
    assert driver.lp_subgroup(n, sigs, ok) == 0
    assert 0 < sum(ok.raw[:n]) < n
    assert driver.lp_cofactor(n, msgs, 48, drop) == 0
    for G in (4, 8):
        for blocks in (0, 1):
            assert driver.lp_scale(n, keys, sigs, msgs, 48, n // G, coeffs(G + 2 * blocks), blocks) == 0, (G, blocks)
