"""GPU: the constant-time secret-scalar ladders on the device.

No divergence: tests/ct/ct_driver.cu, built with the library's nvcc flags plus -DHB_CT_PROBE_DEVICE, runs each of k_g1_mul_gen,
k_sign_hash, k_sign_hm_pair and k_sign_hm_gls_pair on warps where every lane (or lane pair) holds a different edge key.  Every probe
(complete formulas, table reads, ladder steps) records __activemask() and a per-thread count and tag hash: on the code nvcc emitted,
every mask must be the full warp and every thread must pass the same probes.  The outputs are the oracle's bytes.

Parity through the C ABI: blsSignHash (H(m) cold and cached), blsGetPublicKey, hbls_sign_hash_batch, hbls_get_public_key_batch and a
Part-1 turn of sign and GetPublicKey requests from several threads give the oracle's bytes for the edge keys; the secret-key verdicts
of blsSecretKeyIsEqual / blsSecretKeyDeserialize are unchanged."""
import ctypes, os, random, subprocess, tempfile, threading
import pytest
from harmony_b200 import build, workload as wl
from test_constant_time_emu import edge_keys, BIG_KEYS, LIM, R, Z, k32

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MSG = wl.commit_payload("ct-gpu", 0)


class CtRec(ctypes.Structure):
    _fields_ = [("count", ctypes.c_uint32), ("partial", ctypes.c_uint32), ("hash", ctypes.c_uint64)]


@pytest.fixture(scope="module")
def driver():
    out = os.path.join(tempfile.mkdtemp(prefix="hbls_ct_"), "libct_probe.so")
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    subprocess.check_call([nvcc] + build.NVCC_FLAGS + ["-DHB_CT_PROBE_DEVICE", "-o", out, os.path.join(ROOT, "tests", "ct", "ct_driver.cu")])
    L = ctypes.CDLL(out)
    L.ct_run.argtypes = [ctypes.c_int, ctypes.c_size_t, ctypes.c_char_p, ctypes.POINTER(ctypes.c_uint64), ctypes.c_char_p, ctypes.c_uint32,
                         ctypes.c_char_p, ctypes.c_char_p, ctypes.POINTER(CtRec)]
    return L


def digits(k):
    d = []
    for _ in range(3):
        d.append(k % Z); k //= Z
    return d + [k]


def warp_keys(kernel):
    """64 items with pairwise different keys (2 warps of threads, or 4 warps of lane pairs): the edge keys (kernels 2 and 3: also the
    hand-filled ones they take), seeded random keys after them"""
    keys = edge_keys() + (BIG_KEYS if kernel == 2 else [k for k in BIG_KEYS if k < LIM] if kernel == 3 else [])
    rng = random.Random(0x7a + kernel)
    while len(keys) < 64: keys.append(rng.randrange(R))
    return keys[:64]


@pytest.mark.parametrize("kernel", [0, 1, 2, 3], ids=["g1_mul_gen", "sign_hash", "sign_hm_pair", "sign_hm_gls_pair"])
def test_gpu_ct_no_divergence_and_parity(driver, oracle, kernel):
    keys = warp_keys(kernel)
    n = len(keys)
    sk = b"".join(k32(k) for k in keys)
    dig = (ctypes.c_uint64 * (4 * n))(*[x for k in keys for x in digits(k)]) if kernel == 3 else None
    w = 48 if kernel == 0 else 96
    out = ctypes.create_string_buffer(96 * n); ok = ctypes.create_string_buffer(n)
    threads = 2 * n if kernel >= 2 else n
    rec = (CtRec * threads)()
    assert driver.ct_run(kernel, n, sk, dig, MSG, len(MSG), out, ok, rec) == 0
    assert ok.raw[:n] == b"\x01" * n
    for i, k in enumerate(keys):
        want = oracle.get_public_key(k32(k % R)) if kernel == 0 else oracle.sign_hash(k32(k % R), MSG)
        assert out.raw[w * i:w * i + w] == want, (i, hex(k))
    assert all(r.partial == 0 for r in rec), [i for i, r in enumerate(rec) if r.partial]
    assert len({(r.count, r.hash) for r in rec}) == 1 and rec[0].count > 0


@pytest.fixture(scope="module")
def keyset():
    rng = random.Random(0x5151)
    return edge_keys() + [rng.randrange(R) for _ in range(4)]


def test_gpu_ct_capi_sign_and_public_key(gbls, oracle, keyset):
    """blsSignHash with H(m) cold, then cached; blsGetPublicKey: the oracle's bytes for every edge key"""
    for j, k in enumerate(keyset):
        s = gbls.SecretKey(); s.Deserialize(k32(k))
        assert s.GetPublicKey().Serialize() == oracle.get_public_key(k32(k)), hex(k)
        msg = wl.commit_payload("ct-capi", j)                         # a message not signed before: H(m) cold, then cached
        want = oracle.sign_hash(k32(k), msg)
        assert s.SignHash(msg).Serialize() == want, hex(k)
        assert s.SignHash(msg).Serialize() == want, hex(k)


def test_gpu_ct_capi_hand_filled_keys(gbls, oracle):
    """structs >= Z^4 filled by hand (Deserialize rejects them): the psi ladder below Z^3 2^64, the 256-bit ladder above"""
    for k in BIG_KEYS:
        s = gbls.SecretKey()
        for i in range(4): s.v.d[i] = (k >> (64 * i)) & (2 ** 64 - 1)
        assert s.SignHash(MSG).Serialize() == oracle.sign_hash(k32(k % R), MSG), hex(k)
        assert s.GetPublicKey().Serialize() == oracle.get_public_key(k32(k % R)), hex(k)


def test_gpu_ct_batch_entries(gbls, oracle, keyset):
    sks = b"".join(k32(k) for k in keyset)
    msgs = b"".join(wl.commit_payload("ct-batch", j) for j in range(len(keyset)))
    sigs, ok = gbls.SignHashBatch(sks, msgs, 48)
    assert ok == b"\x01" * len(keyset)
    pks = gbls.GetPublicKeyBatch(sks)
    for j, k in enumerate(keyset):
        assert sigs[96 * j:96 * j + 96] == oracle.sign_hash(k32(k), msgs[48 * j:48 * j + 48]), hex(k)
        assert pks[48 * j:48 * j + 48] == oracle.get_public_key(k32(k)), hex(k)


def test_gpu_ct_part1_turn_from_threads(gbls, oracle, keyset):
    """sign and GetPublicKey requests from 8 threads at once (combined into shared turns): every caller gets its own oracle bytes"""
    T = 8
    got, errors = {}, []
    def body(t):
        try:
            for j in range(t, len(keyset), T):
                s = gbls.SecretKey(); s.Deserialize(k32(keyset[j]))
                msg = MSG if j % 2 else wl.commit_payload("ct-turn", j)
                got[j] = (s.SignHash(msg).Serialize(), s.GetPublicKey().Serialize(), msg)
        except BaseException as e:
            errors.append(repr(e))
    th = [threading.Thread(target=body, args=(t,)) for t in range(T)]
    for x in th: x.start()
    for x in th: x.join(timeout=600)
    assert not errors and len(got) == len(keyset), errors[:3]
    for j, k in enumerate(keyset):
        sig, pk, msg = got[j]
        assert sig == oracle.sign_hash(k32(k), msg) and pk == oracle.get_public_key(k32(k)), hex(k)


def test_gpu_ct_secret_key_verdicts(gbls):
    """Deserialize accepts 0 and r - 1, rejects r and 2^256 - 1; IsEqual on equal keys and on keys that differ"""
    for k, accepted in ((0, True), (R - 1, True), (R, False), (2 ** 256 - 1, False)):
        s = gbls.SecretKey()
        if accepted:
            s.Deserialize(k32(k)); assert s.Serialize() == k32(k)
        else:
            with pytest.raises(ValueError): s.Deserialize(k32(k))
    a, b, c = gbls.SecretKey(), gbls.SecretKey(), gbls.SecretKey()
    a.Deserialize(k32(R - 1)); b.Deserialize(k32(R - 1)); c.Deserialize(k32(R - 1 - 2 ** 200))
    z0, z1 = gbls.SecretKey(), gbls.SecretKey(); z0.Deserialize(k32(0))
    assert a.IsEqual(b) and not a.IsEqual(c) and z0.IsEqual(z1) and not z0.IsEqual(a)
