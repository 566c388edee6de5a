"""Multi-key signing: hbls_sign_hash_keys, where k keys sign each of m messages in one call (a node running several BLS keys:
consensus/construct.go:97-114, leader.go:57-75, threshold.go:53-69, view_change_construct.go:402-483).

CPU: the key sum of harmony_b200/csrc/secret_key.hpp (sk_sum_mod_r, whose base-|z| digits are the aggregate's ladder scalar) against
Python integers.

GPU (marked): per-key signatures and aggregates against the CPU oracle, AggregateSigBytes and SignHashBatch; unmappable, long and
repeated messages; degenerate key sums and hand-filled keys; a launch count that does not grow with k; the H(m) cache; argument
errors; threads signing while others verify; the C++ multibls mirror against the SignHash + Add loop it replaces."""
import ctypes, os, random, subprocess, tempfile, threading
import pytest
from harmony_b200 import workload as wl

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
R = wl.R_ORDER
Z = 0xd201000000010000
LIM = Z ** 3 * 2 ** 64
# hand-filled structs (not valid keys, but signable): below LIM the psi ladder takes their digits, from LIM on the 256-bit ladder
BIG_KEYS = [Z ** 4, 2 ** 256 - 1, 2 ** 256 - 2, 2 ** 255, Z ** 4 + R, LIM - 1, LIM]


def k32(k):
    return k.to_bytes(32, "little")


def from_digits(d):
    return d[0] + d[1] * Z + d[2] * Z ** 2 + d[3] * Z ** 3


# ------------------------------------------------------------------ CPU: the key sum
@pytest.fixture(scope="module")
def emusum():
    out = os.path.join(tempfile.mkdtemp(prefix="hbls_key_sum_"), "libemu_key_sum.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-o", out, os.path.join(ROOT, "tests", "emu", "emu_key_sum.cpp")])
    L = ctypes.CDLL(out)
    L.emu_key_sum.argtypes = [ctypes.c_char_p, ctypes.c_size_t, ctypes.POINTER(ctypes.c_uint64), ctypes.POINTER(ctypes.c_uint64)]
    return L


def key_sum(emusum, keys):
    s = (ctypes.c_uint64 * 4)(); d = (ctypes.c_uint64 * 4)()
    fits = emusum.emu_key_sum(b"".join(k32(k) for k in keys), len(keys), s, d)
    got = sum(int(x) << (64 * i) for i, x in enumerate(s))
    assert fits == 1 and all(x < Z for x in d[:3]) and from_digits(list(d)) == got, [hex(k) for k in keys]   # digits recompose
    return got


EDGE = [0, 1, R - 1, R, R + 1, 2 ** 256 - 1] + BIG_KEYS


@pytest.mark.parametrize("k", EDGE, ids=lambda k: hex(k)[:12])
def test_key_sum_single_edge_keys(emusum, k):
    """k = 1: the key reduced mod r (two conditional subtractions cover every 256-bit value)"""
    assert key_sum(emusum, [k]) == k % R


def test_key_sum_edge_pairs_and_all(emusum):
    for a in EDGE:
        for b in EDGE:
            assert key_sum(emusum, [a, b]) == (a + b) % R, (hex(a), hex(b))
    assert key_sum(emusum, EDGE) == sum(EDGE) % R


def test_key_sum_crossings_and_zero(emusum):
    """sums that cross r once and many times, and sums that are 0 mod r"""
    cases = [[R - 1, 2], [R - 1, 1], [R - 1] * 50, [2 ** 256 - 1] * 77, [R // 2 + 1] * 3, [(R + 1) // 2, (R - 1) // 2],
             [R] * 9, [12345, R - 12345], [5, 7, R - 12], [R - 1] * 1000 + [1000], [2 ** 256 - 1] * 3 + [R - 3 * (2 ** 256 - 1) % R]]
    for keys in cases:
        assert key_sum(emusum, keys) == sum(keys) % R
    zero = [[R - 1, 1], [R] * 9, [12345, R - 12345], [5, 7, R - 12], [R - 1] * 1000 + [1000], cases[-1]]
    assert all(key_sum(emusum, keys) == 0 for keys in zero)


@pytest.mark.parametrize("k", [1, 2, 3, 10, 33, 100, 999, 1000])
def test_key_sum_random(emusum, k):
    rng = random.Random(0x5a3 + k)
    for trial in range(3):
        keys = [rng.randrange(R) if trial == 0 else rng.getrandbits(256) if trial == 1 else rng.choice([rng.randrange(R), R - 1 - rng.getrandbits(8)])
                for _ in range(k)]
        assert key_sum(emusum, keys) == sum(keys) % R


# ------------------------------------------------------------------ GPU
_sig_cache = {}


def want_sig(oracle, k, msg):
    """the oracle's SignHash bytes (cached: the large k reuse them across m)"""
    key = (k % R, bytes(msg[:48]))
    if key not in _sig_cache:
        _sig_cache[key] = oracle.sign_hash(k32(k % R), msg[:48])
    return _sig_cache[key]


def split(blob, w=96):
    return [blob[i:i + w] for i in range(0, len(blob), w)]


def check_call(gbls, oracle, keys, msgs, msg_len=48):
    """every output of one call against the oracle; -> (sigs, aggs, ok)"""
    k, m = len(keys), len(msgs)
    sigs, aggs, ok = gbls.SignHashKeys(b"".join(k32(x) for x in keys), b"".join(msgs), msg_len)
    assert len(sigs) == 96 * m * k and len(aggs) == 96 * m and len(ok) == m
    per = split(sigs)
    for j, msg in enumerate(msgs):
        mapped = oracle.map_to_g2(msg[:48]) is not None
        assert ok[j] == (1 if mapped else 0), j
        row = per[j * k:(j + 1) * k]
        for i, x in enumerate(keys):
            assert row[i] == (want_sig(oracle, x, msg) if mapped else bytes(96)), (j, i, hex(x))
        want_agg = oracle.sign_hash(k32(sum(keys) % R), msg[:48]) if mapped else bytes(96)
        assert aggs[96 * j:96 * j + 96] == want_agg, j
        if mapped:
            assert oracle.aggregate_sigs(row) == want_agg, j
    return sigs, aggs, ok


def seeded_keys(tag, k):
    return [wl.seeded_sk(tag, i) for i in range(k)]


MSGS = [wl.commit_payload("multikey", j) for j in range(3)]


@pytest.mark.gpu
@pytest.mark.parametrize("m", [1, 2, 3])
@pytest.mark.parametrize("k", [1, 2, 10, 33, 1000])
def test_gpu_sign_hash_keys_parity(gbls, oracle, k, m):
    """per-key == oracle SignHash == SignHashBatch over the repeated keys and messages; aggregate == oracle sum == AggregateSigBytes"""
    keys = seeded_keys("multikey", k); msgs = MSGS[:m]
    sigs, aggs, ok = check_call(gbls, oracle, keys, msgs)
    assert ok == b"\x01" * m
    per = split(sigs)
    for j in range(m):
        assert gbls.AggregateSigBytes(per[j * k:(j + 1) * k]) == aggs[96 * j:96 * j + 96]
    bsigs, bok = gbls.SignHashBatch(b"".join(k32(x) for _ in range(m) for x in keys), b"".join(msg for msg in msgs for _ in range(k)), 48)
    assert bok == b"\x01" * (m * k) and bsigs == sigs


@pytest.mark.gpu
def test_gpu_sign_hash_keys_messages(gbls, oracle):
    """an unmappable message among valid ones; 64-byte messages act as their first 48 bytes; a repeated message: same bytes, one hash"""
    keys = seeded_keys("multikey-msg", 10)
    msgs = [wl.commit_payload("multikey-msg", 0), bytes(48), wl.commit_payload("multikey-msg", 1)]
    sigs, aggs, ok = check_call(gbls, oracle, keys, msgs)
    assert ok == b"\x01\x00\x01"
    assert sigs[960:1920] == bytes(960) and aggs[96:192] == bytes(96) and bytes(96) not in split(sigs[:960] + sigs[1920:])
    rng = random.Random(64)
    long_msgs = [msg + bytes(rng.getrandbits(8) for _ in range(16)) for msg in msgs]
    assert gbls.SignHashKeys(b"".join(k32(x) for x in keys), b"".join(long_msgs), 64) == (sigs, aggs, ok)
    fresh = [wl.commit_payload("multikey-rep", j) for j in range(2)]
    h0 = gbls.HashCacheStats()
    rs, ra, rok = check_call(gbls, oracle, keys, [fresh[0], fresh[1], fresh[0]])
    h1 = gbls.HashCacheStats()
    assert h1["misses"] - h0["misses"] == 2 and h1["hits"] == h0["hits"]
    assert rs[:960] == rs[1920:] and ra[:96] == ra[192:] and rok == b"\x01\x01\x01"


@pytest.mark.gpu
def test_gpu_sign_hash_keys_degenerate_keys(gbls, oracle):
    """keys summing to 0 mod r: identity aggregate; summing to 1: the aggregate is H(m); duplicated keys, key 0 and hand-filled keys
    in both outputs"""
    msgs = [wl.commit_payload("multikey-deg", j) for j in range(2)]
    a = wl.seeded_sk("multikey-deg", 0)
    sigs, aggs, ok = check_call(gbls, oracle, [a, R - a], msgs)
    assert ok == b"\x01\x01" and aggs == bytes(192) and bytes(96) not in split(sigs)
    _, aggs, _ = check_call(gbls, oracle, [a, R - a + 1], msgs)
    assert aggs == b"".join(gbls.MapToG2(msg) for msg in msgs)
    _, aggs, _ = check_call(gbls, oracle, [5, 7, R - 11], msgs)
    assert aggs == b"".join(gbls.MapToG2(msg) for msg in msgs)
    check_call(gbls, oracle, [a, a, a, 0, a, 0], msgs)
    big = [k for k in BIG_KEYS if k >= LIM]
    assert big
    mixed = [a, BIG_KEYS[0], 0, big[0], R, R + 1, 2 ** 256 - 1, big[-1], a]        # both ladders, interleaved
    for m in (1, 2):
        check_call(gbls, oracle, mixed, msgs[:m])
    check_call(gbls, oracle, big, msgs)                   # every per-key item on the 256-bit ladder
    check_call(gbls, oracle, BIG_KEYS, [msgs[0], bytes(48)])


@pytest.mark.gpu
def test_gpu_sign_hash_keys_output_selection(gbls, oracle):
    """the aggregates are the same bytes with and without per-key outputs, the per-key bytes the same with and without aggregates"""
    keys = seeded_keys("multikey-sel", 33) + BIG_KEYS
    blob = b"".join(k32(x) for x in keys)
    msgs = b"".join(wl.commit_payload("multikey-sel", j) for j in range(3)) + bytes(48)
    sigs, aggs, ok = gbls.SignHashKeys(blob, msgs, 48)
    assert gbls.SignHashKeys(blob, msgs, 48, per_key=False) == (None, aggs, ok)
    assert gbls.SignHashKeys(blob, msgs, 48, aggregate=False) == (sigs, None, ok)
    assert ok == b"\x01\x01\x01\x00"


@pytest.mark.gpu
@pytest.mark.parametrize("m", [1, 2, 3])
def test_gpu_sign_hash_keys_launches_do_not_grow_with_k(gbls, m):
    """for fixed m and cache state, a call launches as many kernels for 1 000 keys as for one"""
    deltas = {}
    for k in (1, 1000):
        blob = b"".join(k32(x) for x in seeded_keys("multikey-launch", k))
        for state in ("cold", "cached"):
            msgs = b"".join(wl.commit_payload(f"multikey-launch-{k}-{m}", j) for j in range(m))
            if state == "cached":
                gbls.SignHashKeys(blob, msgs, 48)
            else:
                msgs = b"".join(wl.commit_payload(f"multikey-launch-cold-{k}-{m}", j) for j in range(m))
            n0 = gbls.KernelLaunchCount()
            gbls.SignHashKeys(blob, msgs, 48)
            deltas[(k, state)] = gbls.KernelLaunchCount() - n0
    assert deltas[(1, "cold")] == deltas[(1000, "cold")] and deltas[(1, "cached")] == deltas[(1000, "cached")], deltas
    assert deltas[(1, "cached")] < deltas[(1, "cold")], deltas


@pytest.mark.gpu
def test_gpu_sign_hash_keys_hash_cache(gbls):
    """a repeated call is all hits; blsVerifyHash and hbls_aggregate_verify on the message it signed then hit too; with the cache
    off neither counter moves"""
    keys = seeded_keys("multikey-cache", 4)
    blob = b"".join(k32(x) for x in keys)
    msgs = [wl.commit_payload("multikey-cache", j) for j in range(3)]
    sigs, aggs, ok = gbls.SignHashKeys(blob, b"".join(msgs), 48)
    h0 = gbls.HashCacheStats()
    assert gbls.SignHashKeys(blob, b"".join(msgs), 48) == (sigs, aggs, ok)
    h1 = gbls.HashCacheStats()
    assert h1["hits"] - h0["hits"] == 3 and h1["misses"] == h0["misses"]
    pks = split(gbls.GetPublicKeyBatch(blob), 48)
    pk = gbls.PublicKey(); pk.Deserialize(pks[1])
    s = gbls.Sign(); s.Deserialize(sigs[96 * (0 * 4 + 1):96 * (0 * 4 + 2)])
    assert s.VerifyHash(pk, msgs[0])
    h2 = gbls.HashCacheStats()
    assert h2["hits"] - h1["hits"] == 1 and h2["misses"] == h1["misses"]
    com = gbls.Committee(pks)
    assert com.AggregateVerify(b"\x0f", aggs[96:192], msgs[1])
    h3 = gbls.HashCacheStats()
    assert h3["hits"] - h2["hits"] == 1 and h3["misses"] == h2["misses"]
    old = gbls.GetParam("hm_cache")
    gbls.SetParam("hm_cache", 0)
    try:
        fresh = b"".join(wl.commit_payload("multikey-nocache", j) for j in range(2))
        got = gbls.SignHashKeys(blob, fresh, 48)
        again = gbls.SignHashKeys(blob, b"".join(msgs), 48)
        assert gbls.HashCacheStats() == h3
    finally:
        gbls.SetParam("hm_cache", old)
    assert again == (sigs, aggs, ok) and got[2] == b"\x01\x01"


@pytest.mark.gpu
def test_gpu_sign_hash_keys_argument_errors(gbls):
    """HBLS_ERR_ARG before any launch; m == 0 returns 0 and launches nothing"""
    L = gbls.lib(); gbls.HashCacheStats()                 # initialised
    sk = k32(12345) * 2; msg = wl.commit_payload("multikey-arg", 0) * 2
    out = ctypes.create_string_buffer(96 * 4); agg = ctypes.create_string_buffer(96 * 2); ok = ctypes.create_string_buffer(2)
    big = 2 ** 64 - 1
    bad = [(0, sk, 2, msg, 48, out, agg, ok),              # k == 0
           (2, sk, 2, msg, 48, None, None, ok),            # no output
           (2, None, 2, msg, 48, out, agg, ok),            # no keys
           (2, sk, 2, msg, 48, out, agg, None),            # no ok
           (2, sk, 2, None, 48, out, agg, ok),             # no messages
           (2, sk, 2 ** 62, msg, 48, out, agg, ok),        # m (k + 1) items overflow
           (big, sk, 2, msg, 48, out, agg, ok),            # k + 1 overflows
           (2 ** 59, sk, 1, msg, 48, out, agg, ok),        # k x 32 key bytes overflow
           (2, sk, 2 ** 40, msg, 2 ** 30, out, agg, ok)]   # m x msg_len overflows
    n0 = gbls.KernelLaunchCount()
    for args in bad:
        assert L.hbls_sign_hash_keys(*args) == gbls.ERR_ARG, args[:5]
    assert L.hbls_sign_hash_keys(2, sk, 0, None, 48, out, agg, ok) == 0
    assert L.hbls_sign_hash_keys(2, sk, 0, None, 0, None, agg, ok) == 0
    assert L.hbls_sign_hash_keys(2, sk, 1, None, 0, out, None, ok) == 0               # an empty message needs no bytes
    assert ok.raw[0] == 0 and out.raw[:192] == bytes(192)                              # ... and maps to no point
    assert gbls.KernelLaunchCount() - n0 >= 1
    n1 = gbls.KernelLaunchCount()
    assert L.hbls_sign_hash_keys(0, sk, 0, None, 48, out, agg, ok) == gbls.ERR_ARG
    assert gbls.KernelLaunchCount() == n1


@pytest.mark.gpu
def test_gpu_sign_hash_keys_threads_with_verifiers(gbls, oracle):
    """eight threads calling hbls_sign_hash_keys while four call blsVerifyHash: every caller gets its exact result"""
    T, V, ITERS = 8, 4, 3
    keysets = [seeded_keys(f"multikey-thr-{t}", 3 + t) for t in range(T)]
    jobs = {(t, it): [wl.commit_payload(f"multikey-thr-{t}-{it}", j) for j in range(1 + (t + it) % 3)] for t in range(T) for it in range(ITERS)}
    want = {key: ([want_sig(oracle, x, msg) for msg in msgs for x in keysets[key[0]]],
                  [oracle.sign_hash(k32(sum(keysets[key[0]]) % R), msg) for msg in msgs]) for key, msgs in jobs.items()}
    vkeys = seeded_keys("multikey-thr-v", 6)
    vmsg = [wl.commit_payload("multikey-thr-v", j) for j in range(6)]
    vcases = []
    for i, x in enumerate(vkeys):
        pk = gbls.PublicKey(); pk.Deserialize(oracle.get_public_key(k32(x)))
        s = gbls.Sign(); s.Deserialize(want_sig(oracle, x, vmsg[i]))
        vcases.append((s, pk, vmsg[i], True)); vcases.append((s, pk, vmsg[(i + 1) % 6], False))
    errors, got = [], {}
    def signer(t):
        try:
            for it in range(ITERS):
                msgs = jobs[(t, it)]
                got[(t, it)] = gbls.SignHashKeys(b"".join(k32(x) for x in keysets[t]), b"".join(msgs), 48)
        except BaseException as e:
            errors.append(repr(e))
    def verifier(v):
        try:
            for rep in range(4):
                for s, pk, msg, exp in vcases[v::V]:
                    if s.VerifyHash(pk, msg) != exp: errors.append(f"verify {v} {rep}")
        except BaseException as e:
            errors.append(repr(e))
    th = [threading.Thread(target=signer, args=(t,)) for t in range(T)] + [threading.Thread(target=verifier, args=(v,)) for v in range(V)]
    for x in th: x.start()
    for x in th: x.join(timeout=600)
    assert not errors and len(got) == T * ITERS, errors[:3]
    for key, (sigs, aggs, ok) in got.items():
        ws, wa = want[key]
        assert split(sigs) == ws and split(aggs) == wa and ok == b"\x01" * len(jobs[key]), key


@pytest.mark.gpu
def test_gpu_cpp_multibls_mirror(gbls, tmp_path):
    """multibls::PrivateKeys::SignHashAggregate / SignHashEach (hbls_host.hpp) == the SignHash + Add + Serialize loops they replace"""
    from harmony_b200 import build
    lib = build.build_cuda()
    exe = str(tmp_path / "multikey_sign")
    subprocess.check_call(["g++", "-O1", "-std=c++17", "-Wall", "-o", exe, os.path.join(ROOT, "tests", "host", "multikey_sign.cpp"),
                           "-L" + os.path.dirname(lib), "-lhbls", "-Wl,-rpath," + os.path.dirname(lib), "-pthread", "-ldl", "-lrt"])
    r = subprocess.run([exe], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0 and "all checks passed" in r.stdout, r.stdout + r.stderr
