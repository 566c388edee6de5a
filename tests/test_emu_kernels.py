"""CPU-only: the __global__ kernels of harmony_b200/csrc/kernels.cuh run on the host (tests/emu/emu_kernels.cpp) in the launch
order of hbls.cu's aggregate-verify pipeline -- complement-side mask sums, signature decode, hash-to-G2, batched groups of 4 with
the lane-pair pairing kernel on two host threads, finish flags, exact fallback and tail -- against the oracle's per-round verdicts.
Test infrastructure only: the product path has no CPU implementation (tests/test_capi_symbols.py)."""
import ctypes, os, random, subprocess
import pytest
import oracle_lib
from harmony_b200 import workload as wl

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# "default" = the shipped build (shared inversions: one per 8 items of a persistent thread); "plain" = one inversion per item
# (round-1 behaviour, -DHB_BATCH_INV=0); "karatsuba" = products through mul_wide_k (-DHB_KARATSUBA=1, timed variant)
@pytest.fixture(scope="module", params=["default", "plain", "karatsuba"])
def emuk(request):
    variant = request.param
    src = os.path.join(ROOT, "tests", "emu", "emu_kernels.cpp")
    out = os.path.join(ROOT, "tests", "emu", "libhbls_emu_kernels.so" if variant == "default" else f"libhbls_emu_kernels_{variant}.so")
    csrc = os.path.join(ROOT, "harmony_b200", "csrc")
    deps = [src] + [os.path.join(csrc, f) for f in os.listdir(csrc) if f.endswith(".cuh")]
    if not os.path.exists(out) or any(os.path.getmtime(d) > os.path.getmtime(out) for d in deps):
        flags = {"default": [], "plain": ["-DHB_BATCH_INV=0"], "karatsuba": ["-DHB_KARATSUBA=1"]}[variant]
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-pthread"] + flags + ["-o", out, src])
    L = ctypes.CDLL(out)
    L.emu_aggregate_verify_batch.argtypes = [ctypes.c_int, ctypes.c_uint32, ctypes.c_char_p, ctypes.c_size_t, ctypes.c_char_p, ctypes.c_size_t,
                                             ctypes.c_char_p, ctypes.c_char_p, ctypes.c_uint32, ctypes.c_uint64, ctypes.c_uint64,
                                             ctypes.c_char_p, ctypes.POINTER(ctypes.c_int), ctypes.c_char_p, ctypes.c_int, ctypes.POINTER(ctypes.c_int),
                                             ctypes.c_size_t]
    return L

@pytest.fixture(scope="module")
def oracle():
    return oracle_lib.load()

def make_batch(oracle, n, B, seed):
    """n-key committee, B rounds with distinct bitmaps (some above n/2: complement sums) and distinct 48-byte payloads."""
    rng = random.Random(seed)
    sks = [wl.seeded_sk("emuk", i) for i in range(n)]
    pks = [oracle.get_public_key(wl.sk_bytes(k)) for k in sks]
    blen = (n + 7) // 8
    R = 0x73eda753299d7d483339d80809a1d80553bda402fffe5bfeffffffff00000001
    bitmaps, sigs, msgs = [], [], []
    for j in range(B):
        k = [n, n - 1, n // 2, 1, n - 2, 3][j % 6]
        members = rng.sample(range(n), k)
        bm = bytearray(blen)
        for i in members: bm[i >> 3] |= 1 << (i & 7)
        m = wl.commit_payload("emuk", j)
        agg_sk = sum(sks[i] for i in members) % R
        bitmaps.append(bytes(bm)); msgs.append(m); sigs.append(oracle.sign_hash(wl.sk_bytes(agg_sk), m))
    return pks, blen, bitmaps, sigs, msgs

def run_info(emuk, mode, pks, blen, bitmaps, sigs, msgs, seed=(0x1234, 0x9876), G=4, chunk=0):
    """-> per-round results, any round listed, per-group verdicts, groups failed.  chunk > 0: groups per pass of the line buffer."""
    B = len(sigs); res = ctypes.create_string_buffer(B); gok = ctypes.create_string_buffer(B // 4 + 1); af = ctypes.c_int(-1); gf = ctypes.c_int(-1)
    rc = emuk.emu_aggregate_verify_batch(mode, len(pks), b"".join(pks), B, b"".join(bitmaps), blen, b"".join(sigs), b"".join(msgs), 48,
                                         seed[0], seed[1], res, ctypes.byref(af), gok, G, ctypes.byref(gf), chunk)
    assert rc == 0, rc
    return res.raw[:B], af.value, gok.raw[:B // G], gf.value

def run(emuk, mode, pks, blen, bitmaps, sigs, msgs, seed=(0x1234, 0x9876), G=4):
    return run_info(emuk, mode, pks, blen, bitmaps, sigs, msgs, seed, G)[:3]

def expected(oracle, pks, bitmaps, sigs, msgs):
    h = oracle.committee(pks)
    return bytes(1 if oracle.committee_aggregate_verify(h, bm, s, m) else 0 for bm, s, m in zip(bitmaps, sigs, msgs))

def test_pipeline_all_valid_batched(emuk, oracle):
    pks, blen, bitmaps, sigs, msgs = make_batch(oracle, 10, 9, seed=5)          # 2 groups of 4 (strided) + a tail of 1
    res, any_fail, gok = run(emuk, 1, pks, blen, bitmaps, sigs, msgs)
    assert res == b"\x01" * 9 and any_fail == 0 and gok == b"\x01\x01"
    assert expected(oracle, pks, bitmaps, sigs, msgs) == res

def test_pipeline_bad_rounds_fall_back_to_exact(emuk, oracle):
    pks, blen, bitmaps, sigs, msgs = make_batch(oracle, 10, 9, seed=6)
    sigs[5] = sigs[2]                                    # valid point, wrong round: group 1 (rounds 1, 3, 5, 7) must fail
    sigs[8] = b"\xff" * 96                               # undecodable, in the exactly-verified tail
    want = expected(oracle, pks, bitmaps, sigs, msgs)
    assert want == b"\x01\x01\x01\x01\x01\x00\x01\x01\x00"
    res, any_fail, gok = run(emuk, 1, pks, blen, bitmaps, sigs, msgs)
    assert gok == b"\x01\x00" and any_fail == 1 and res == want
    res0, _, _ = run(emuk, 0, pks, blen, bitmaps, sigs, msgs)                   # exact mode gives the same booleans
    assert res0 == want

def test_pipeline_irregular_rounds(emuk, oracle):
    """Empty bitmap (identity aggregate key) and an all-zero signature: the batched form flags them, the exact pass
    (lane-pair kernel result 0xFF -> k_pairing_fixup) decides exactly as the oracle does."""
    pks, blen, bitmaps, sigs, msgs = make_batch(oracle, 10, 8, seed=7)
    bitmaps[1] = bytes(blen)
    sigs[6] = bytes(96)
    want = expected(oracle, pks, bitmaps, sigs, msgs)
    res, any_fail, gok = run(emuk, 1, pks, blen, bitmaps, sigs, msgs)
    assert any_fail == 1 and res == want

def test_pipeline_groups_of_eight(emuk, oracle):
    pks, blen, bitmaps, sigs, msgs = make_batch(oracle, 12, 17, seed=8)         # 2 strided groups of 8 + a tail of 1
    res, any_fail, gok = run(emuk, 1, pks, blen, bitmaps, sigs, msgs, G=8)
    assert res == b"\x01" * 17 and any_fail == 0 and gok == b"\x01\x01"
    msgs[4] = bytes([msgs[4][0] ^ 1]) + msgs[4][1:]      # round 4 = group 0 (even rounds): fails, exact pass sorts it out
    want = expected(oracle, pks, bitmaps, sigs, msgs)
    res, any_fail, gok = run(emuk, 1, pks, blen, bitmaps, sigs, msgs, G=8)
    assert gok == b"\x00\x01" and any_fail == 1 and res == want and want[4] == 0 and sum(want) == 16

# ---- batches beyond one chunk of the line buffer.  On the device a chunk is rlc_chunk_groups() = SM count x 256 groups; here it is a
# few groups, so that the group form, the exact pass over the failed groups' list and the exact form each run over several chunks.
# Groups are strided: round (k, g) = k * ng + g.
def rnd(ng, k, g):
    return k * ng + g

def flip(msg):
    return bytes([msg[0] ^ 1]) + msg[1:]

def check_chunked(emuk, oracle, pks, blen, bitmaps, sigs, msgs, G, chunk, bad):
    """The batch in chunks of `chunk` groups (the exact forms: `chunk` rounds) gives the oracle's verdicts, which are 0 exactly at the
    injected rounds, and the group verdicts, groups_failed and results of the same pipeline in one pass; exact mode in chunks agrees."""
    B = len(sigs); ng = B // G
    want = expected(oracle, pks, bitmaps, sigs, msgs)
    assert {j for j in range(B) if want[j] != 1} == set(bad)
    failed = {j % ng for j in bad if j < ng * G}
    one = run_info(emuk, 1, pks, blen, bitmaps, sigs, msgs, G=G)
    got = run_info(emuk, 1, pks, blen, bitmaps, sigs, msgs, G=G, chunk=chunk)
    assert got == one
    assert got[0] == want and got[1] == (1 if failed else 0) and got[3] == len(failed)
    assert got[2] == bytes(0 if g in failed else 1 for g in range(ng))
    assert run_info(emuk, 0, pks, blen, bitmaps, sigs, msgs, G=G, chunk=chunk)[0] == want

@pytest.mark.parametrize("G", [4, 8])
def test_chunked_irregular_rounds_at_chunk_edges(emuk, oracle, G):
    """7 groups in chunks of 3 (3 + 3 + 1: the last chunk holds one group) and a tail of 2.  A wrong message, an undecodable signature,
    an identity signature, an empty bitmap and another round's signature sit in the first and last group of every chunk, and a wrong
    message in the middle of the first chunk.  Group 4 is the only clean group.  The failed groups' list (6 G rounds) runs in chunks of
    3 rounds, and the loop over the worst case (7 G rounds) runs past it."""
    ng = 7
    pks, blen, bitmaps, sigs, msgs = make_batch(oracle, 10, ng * G + 2, seed=40 + G)
    bad = {rnd(ng, 0, 0), rnd(ng, G - 1, 2), rnd(ng, 0, 3), rnd(ng, G - 1, 5), rnd(ng, 1, 6), rnd(ng, 2, 1), ng * G, ng * G + 1}
    msgs[rnd(ng, 0, 0)] = flip(msgs[rnd(ng, 0, 0)])                 # first group of chunk 0
    sigs[rnd(ng, G - 1, 2)] = b"\xff" * 96                          # last group of chunk 0: does not decode
    sigs[rnd(ng, 0, 3)] = bytes(96)                                 # first group of chunk 1: identity signature
    bitmaps[rnd(ng, G - 1, 5)] = bytes(blen)                        # last group of chunk 1: empty bitmap (identity aggregate key)
    sigs[rnd(ng, 1, 6)] = sigs[rnd(ng, 0, 1)]                       # the one-group chunk: a valid point of another round
    msgs[rnd(ng, 2, 1)] = flip(msgs[rnd(ng, 2, 1)])                 # middle of chunk 0
    sigs[ng * G] = bytes(96); msgs[ng * G + 1] = flip(msgs[ng * G + 1])     # tail
    check_chunked(emuk, oracle, pks, blen, bitmaps, sigs, msgs, G, 3, bad)

@pytest.mark.parametrize("G", [4, 8])
def test_chunked_list_spans_three_chunks_and_a_partial_one(emuk, oracle, G):
    """16 listed rounds (4 failed groups of 4, or 2 of 8) in chunks of 5: 5 + 5 + 5 + 1; the group form in chunks of 5 groups (5 + 2)."""
    ng = 7
    pks, blen, bitmaps, sigs, msgs = make_batch(oracle, 10, ng * G + 1, seed=50 + G)
    groups = [0, 2, 4, 6] if G == 4 else [1, 5]
    bad = {rnd(ng, (3 * i + 1) % G, g) for i, g in enumerate(groups)}
    for j in bad: msgs[j] = flip(msgs[j])
    check_chunked(emuk, oracle, pks, blen, bitmaps, sigs, msgs, G, 5, bad)

@pytest.mark.parametrize("G", [4, 8])
def test_chunked_list_shorter_than_a_chunk(emuk, oracle, G):
    """One failed group: G listed rounds, less than a chunk of G + 2, while the loop over the worst case (7 G rounds) runs 5 or 6 chunks."""
    ng = 7
    pks, blen, bitmaps, sigs, msgs = make_batch(oracle, 10, ng * G + 1, seed=60 + G)
    j = rnd(ng, G - 1, ng - 1)
    msgs[j] = flip(msgs[j])
    check_chunked(emuk, oracle, pks, blen, bitmaps, sigs, msgs, G, G + 2, {j})

@pytest.mark.parametrize("G", [4, 8])
def test_chunked_empty_list(emuk, oracle, G):
    """All valid: the list is empty and every chunk of the exact pass must return at once (chunks of 2)."""
    pks, blen, bitmaps, sigs, msgs = make_batch(oracle, 10, 7 * G + 3, seed=70 + G)
    check_chunked(emuk, oracle, pks, blen, bitmaps, sigs, msgs, G, 2, set())

def test_stage_counts_pinned(emuk, oracle, request):
    """bench.py's roofline counts EXECUTED Fp multiplications / squarings per round for every stage; the figures are those of the
    device kernels themselves, run here on the host over rounds of the benchmark's workload (250 keys, 167/200/250 signers)."""
    import importlib.util
    spec = importlib.util.spec_from_file_location("bench_mod", os.path.join(ROOT, "bench.py")); bench = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(bench)
    batch_inv = "plain" not in request.node.name
    sks = bench.make_committee_sks()
    pks = [oracle.get_public_key(wl.sk_bytes(k)) for k in sks]
    B = 32
    bitmaps, agg_sk, msgs, nsig = bench.make_rounds(sks, B, seed=2024)
    sigs = b"".join(oracle.sign_hash(agg_sk[32 * j:32 * j + 32], msgs[48 * j:48 * j + 48]) for j in range(B))
    emuk.emu_stage_counts.argtypes = [ctypes.c_uint32, ctypes.c_char_p, ctypes.c_size_t, ctypes.c_char_p, ctypes.c_size_t, ctypes.c_char_p, ctypes.c_char_p,
                                      ctypes.c_uint32, ctypes.c_int, ctypes.POINTER(ctypes.c_uint64)]
    t = bench.EXEC_FP_OPS[batch_inv]
    for G in (8, 4):
        out = (ctypes.c_uint64 * 8)()
        assert emuk.emu_stage_counts(250, b"".join(pks), B, bitmaps, 32, sigs, msgs, 48, G, out) == 0
        got = [(out[2 * i] / B, out[2 * i + 1] / B) for i in range(4)]
        want = [t["mask"], t["decode"], t["hash"], (t[G]["scale"][0] / G, t[G]["scale"][1] / G)]
        for (gm, gs), (wm, ws) in zip(got, want):
            assert abs(gm - wm) <= 0.02 * wm and abs(gs - ws) <= 0.02 * ws, (G, got, want)

def test_vm_pairing_device_decoders(emuk, oracle):
    """Latency-mode pairing (csrc/vm.cuh): the generated step programs executed with the device's own instruction decoders
    (vm_mul / vm_sqr / vm_lin over the 25-word slots) give the oracle's verdicts -- valid, wrong message, wrong key."""
    sk = wl.sk_bytes(wl.seeded_sk("vm", 0)); sk2 = wl.sk_bytes(wl.seeded_sk("vm", 1))
    pk, pk2 = oracle.get_public_key(sk), oracle.get_public_key(sk2)
    m = wl.commit_payload("vm", 0); m2 = wl.commit_payload("vm", 1)
    sig = oracle.sign_hash(sk, m)
    for (p_, s_, msg) in ((pk, sig, m), (pk, sig, m2), (pk2, sig, m)):
        assert emuk.emu_vm_pairing(p_, s_, msg, 48) == (1 if oracle.verify_hash(s_, p_, msg) else 0)
    assert emuk.emu_vm_pairing(pk, sig, m, 48) == 1 and emuk.emu_vm_pairing(pk, sig, m2, 48) == 0

def test_vm_hash_cofactor_device_decoders(emuk):
    """Warp-per-message hash-to-G2 (k_hash_to_g2_coop): the Budroni-Pintore cofactor clearing as VM step programs (G2 doubling runs,
    additions, psi / psi^2, one inversion), executed with the device decoders, gives the point of the thread-per-item kernel."""
    for i in range(3):
        assert emuk.emu_vm_hash(wl.commit_payload("vmh", i), 48) == 1
    assert emuk.emu_vm_hash(wl.seeded_bytes("vmh/32", 7, 32), 32) == 1
    assert emuk.emu_vm_hash(bytes(48), 48) == -1                      # t = 0: the map is undefined (SignHash returns nil)

def test_sign_ladder_over_psi(emuk):
    """blsSignHash's 4-dimensional ladder (sk in base |z|, psi = [z] on G2) == the plain 255-bit ladder, for ordinary keys and the
    edge digits: sk = 1, |z|, |z|^3, r - 1."""
    R = 0x73eda753299d7d483339d80809a1d80553bda402fffe5bfeffffffff00000001; Z = 0xd201000000010000
    keys = [wl.seeded_sk("gls", i) for i in range(3)] + [1, Z, Z ** 3, Z ** 3 + Z - 1, R - 1]
    for k in keys:
        assert emuk.emu_sign_gls(wl.sk_bytes(k), wl.commit_payload("gls", k & 7), 48) == 1, hex(k)

def test_lane_pair_decode_and_hash_kernels(emuk, oracle):
    """k_g2_decode_pair / k_hash_to_g2_pair (item per lane pair, latency path) == the thread-per-item kernels: valid signatures,
    a point outside the subgroup / undecodable bytes / the identity, messages incl. one that maps to no point."""
    import random
    rng = random.Random(3)
    sks = [wl.sk_bytes(wl.seeded_sk("lp2", i)) for i in range(3)]
    msgs = [wl.commit_payload("lp2", i) for i in range(3)] + [bytes(48), rng.randbytes(48), rng.randbytes(48)]
    sigs = [oracle.sign_hash(s, m) for s, m in zip(sks, msgs)]
    junk = bytearray(rng.randbytes(96)); junk[95] &= 0x19; junk[47] &= 0x19
    sigs += [bytes(96), b"\xff" * 96, bytes(junk)]
    assert emuk.emu_pair_decode_hash(len(sigs), b"".join(sigs), b"".join(msgs), 48) == 3
