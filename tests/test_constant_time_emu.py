"""CPU-only: the secret-scalar kernels (k_g1_mul_gen, k_sign_hash, k_sign_hm_pair, k_sign_hm_gls_pair) run on the host
(tests/emu/emu_ct.cpp, lane pairs on two host threads) give the oracle's bytes for edge and random keys, and execute the same trace of
complete formulas, table reads and ladder steps, and the same number of Fp products and squarings, whatever the key.  The messages
stay fixed while the keys vary.  Also the host key helpers of harmony_b200/csrc/secret_key.hpp against Python integers."""
import ctypes, os, random, subprocess, tempfile
import pytest
import oracle_lib
from harmony_b200 import workload as wl

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
R = wl.R_ORDER
Z = 0xd201000000010000


def from_digits(d):
    return d[0] + d[1] * Z + d[2] * Z ** 2 + d[3] * Z ** 3


def edge_keys():
    """every key below r the constant-time ladders must treat alike"""
    keys = [0, 1, 2, 3, 15, 16, 17,                                          # small keys
            R - 1, R - 2, (R - 1) // 2,                                      # near the group order
            Z - 1, Z, Z + 1, Z ** 2, Z ** 3, Z ** 3 + Z - 1, 2 ** 64 - 1]    # near powers of Z
    keys += [from_digits([Z - 1] * 3 + [3]), from_digits([Z - 1] * 3 + [0]), from_digits([Z - 1, 0, Z - 1, 1]),   # digit patterns
             from_digits([Z - 2, Z - 1, 0, Z - 1]), from_digits([1, Z - 1, Z - 1, 2]), from_digits([2, 0, 0, 3])]
    keys += [int("f" * 63, 16) % R, int("1" * 63, 16), int("10" * 31 + "1", 16), int("0f" * 31 + "0", 16)]  # all-one / all-zero windows
    rng = random.Random(0xc7)
    keys += [rng.randrange(R) for _ in range(20)]
    assert all(0 <= k < R for k in keys) and len(set(keys)) == len(keys)
    return keys


# hand-filled structs >= Z^4 (not valid keys, but signable).  Below Z^3 2^64 the four digits still fit 64 bits and the psi ladder takes
# them; above, the 256-bit ladder of k_sign_hm_pair does.
BIG_KEYS = [Z ** 4, 2 ** 256 - 1, 2 ** 256 - 2, 2 ** 255, Z ** 4 + R, Z ** 3 * 2 ** 64 - 1, Z ** 3 * 2 ** 64]
LIM = Z ** 3 * 2 ** 64


@pytest.fixture(scope="module")
def emuct():
    src = os.path.join(ROOT, "tests", "emu", "emu_ct.cpp")
    out = os.path.join(tempfile.mkdtemp(prefix="hbls_emu_ct_"), "libemu_ct.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-pthread", "-o", out, src])
    L = ctypes.CDLL(out)
    L.emu_ct_run.argtypes = [ctypes.c_int, ctypes.c_char_p, ctypes.c_char_p, ctypes.c_uint32, ctypes.c_char_p, ctypes.POINTER(ctypes.c_uint64)]
    L.emu_ct_digits.argtypes = [ctypes.POINTER(ctypes.c_uint64), ctypes.POINTER(ctypes.c_uint64)]
    L.emu_ct_lt_r.argtypes = [ctypes.POINTER(ctypes.c_uint64)]
    L.emu_ct_eq32.argtypes = [ctypes.c_char_p, ctypes.c_char_p]
    return L


@pytest.fixture(scope="module")
def oracle():
    return oracle_lib.load()


def k32(k):
    return k.to_bytes(32, "little")


def run(emuct, kernel, k, msg):
    out = ctypes.create_string_buffer(96); rec = (ctypes.c_uint64 * 8)()
    rc = emuct.emu_ct_run(kernel, k32(k), msg, len(msg), out, rec)
    return rc, out.raw[:48 if kernel == 0 else 96], tuple(rec)


MSG = wl.commit_payload("ct", 0)


def want(oracle, kernel, k):
    return oracle.get_public_key(k32(k % R)) if kernel == 0 else oracle.sign_hash(k32(k % R), MSG)


@pytest.mark.parametrize("kernel", [0, 1, 2, 3], ids=["g1_mul_gen", "sign_hash", "sign_hm_pair", "sign_hm_gls_pair"])
def test_ct_kernel_parity_and_trace(emuct, oracle, kernel):
    """Every edge key: the oracle's bytes; every key: one and the same trace and Fp operation counts, on each lane."""
    keys = edge_keys() + (BIG_KEYS if kernel == 2 else [k for k in BIG_KEYS if k < LIM] if kernel == 3 else [])
    recs = set()
    for k in keys:
        rc, got, rec = run(emuct, kernel, k, MSG)
        assert rc == 1 and got == want(oracle, kernel, k), hex(k)
        recs.add(rec)
    assert len(recs) == 1, recs
    (rec,) = recs
    assert rec[0] > 0 and (kernel >= 2 or rec[2] > 0)        # lane-pair products do not pass the thread counters
    if kernel >= 2:
        assert rec[4] == rec[0] and rec[5] == rec[1]          # both lanes of the pair walk the same trace


def test_ct_gls_rejects_keys_beyond_64_bit_digits(emuct):
    big = [k for k in BIG_KEYS if k >= LIM]
    assert big
    for k in big:
        assert run(emuct, 3, k, MSG)[0] == -2


def test_ct_unmappable_message(emuct):
    """A message that maps to no point (t = 0): not ok, identity output -- the ladder kernels decide that on public data."""
    for kernel in (1, 2, 3):
        rc, got, _ = run(emuct, kernel, 12345, bytes(48))
        assert rc == 0 and got == bytes(96)


def test_host_key_helpers(emuct):
    """Base-|z| digits by restoring division, k < r by the borrow, equality without early exit: against Python integers."""
    rng = random.Random(0x5ec)
    vals = edge_keys() + BIG_KEYS + [R, R + 1, 2 ** 256 - 1, Z ** 4 - 1] + [rng.getrandbits(256) for _ in range(50)]
    for k in vals:
        w = (ctypes.c_uint64 * 4)(*[(k >> (64 * i)) & (2 ** 64 - 1) for i in range(4)]); d = (ctypes.c_uint64 * 4)()
        fits = emuct.emu_ct_digits(w, d)
        assert fits == (1 if k < LIM else 0), hex(k)
        if fits:
            assert all(x < Z for x in d[:3]) and from_digits(list(d)) == k, hex(k)
        else:
            assert from_digits(list(d)) % Z ** 3 == k % Z ** 3
        assert emuct.emu_ct_lt_r(w) == (1 if k < R else 0), hex(k)
    a = k32(R - 1)
    for i in range(32):
        b = bytearray(a); b[i] ^= 0x80
        assert emuct.emu_ct_eq32(a, bytes(b)) == 0
    assert emuct.emu_ct_eq32(a, a) == 1 and emuct.emu_ct_eq32(bytes(32), bytes(32)) == 1
