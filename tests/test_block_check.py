"""Blocks of groups in the batched verify (hbls.cu rlc_blocks): HB_RLC_M = 16 groups share ONE final exponentiation and ONE generator
pair; the groups of a failed block are then checked one by one, and the rounds of the failed groups exactly.

CPU: the block path of the aggregate-verify pipeline runs on the host (tests/emu/emu_block.cpp: the device kernels, the warp-per-block
VM check replayed with the device decoders) and must give the oracle's per-round verdicts and, group by group, the verdicts of the group
form without blocks.  Small batches use a small block stride S so that one block holds several groups.
GPU: a 270 336-round batch with 1 % invalid rounds (wrong messages, undecodable signatures and signature pairs moved between two groups
of one block so that they would cancel under equal coefficients) rejects exactly the injected rounds through blocks, through the
group form the device then chooses, and with blocks turned off."""
import ctypes, os, random, subprocess
import pytest
import oracle_lib
from harmony_b200 import workload as wl

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def emub():
    src = os.path.join(ROOT, "tests", "emu", "emu_block.cpp")
    out = os.path.join(ROOT, "tests", "emu", "libhbls_emu_block.so")
    csrc = os.path.join(ROOT, "harmony_b200", "csrc")
    deps = [src, os.path.join(ROOT, "tests", "emu", "emu_kernels.cpp")] + [os.path.join(csrc, f) for f in os.listdir(csrc) if f.endswith(".cuh")]
    if not os.path.exists(out) or any(os.path.getmtime(d) > os.path.getmtime(out) for d in deps):
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-pthread", "-o", out, src])
    L = ctypes.CDLL(out)
    L.emu_block_verify.argtypes = [ctypes.c_uint32, ctypes.c_char_p, ctypes.c_size_t, ctypes.c_char_p, ctypes.c_size_t, ctypes.c_char_p,
                                   ctypes.c_char_p, ctypes.c_uint32, ctypes.c_int, ctypes.c_size_t, ctypes.c_uint64, ctypes.c_uint64, ctypes.c_int,
                                   ctypes.c_char_p, ctypes.c_char_p, ctypes.POINTER(ctypes.c_int), ctypes.POINTER(ctypes.c_int)]
    return L


@pytest.fixture(scope="module")
def oracle():
    return oracle_lib.load()


def make_batch(oracle, n, B, seed):
    rng = random.Random(seed)
    sks = [wl.seeded_sk("emub", i) for i in range(n)]
    pks = [oracle.get_public_key(wl.sk_bytes(k)) for k in sks]
    blen = (n + 7) // 8
    R = 0x73eda753299d7d483339d80809a1d80553bda402fffe5bfeffffffff00000001
    bitmaps, sigs, msgs = [], [], []
    for j in range(B):
        members = rng.sample(range(n), [n, n - 1, n // 2, 1, n - 2, 3][j % 6])
        bm = bytearray(blen)
        for i in members: bm[i >> 3] |= 1 << (i & 7)
        m = wl.commit_payload("emub", j)
        bitmaps.append(bytes(bm)); msgs.append(m); sigs.append(oracle.sign_hash(wl.sk_bytes(sum(sks[i] for i in members) % R), m))
    return pks, blen, bitmaps, sigs, msgs


def run(emub, pks, blen, bitmaps, sigs, msgs, G=4, S=0, equal_members=0, seed=(0x5eed, 0xb10c)):
    B = len(sigs); res = ctypes.create_string_buffer(B); gok = ctypes.create_string_buffer(B // G + 1)
    bf, fb = ctypes.c_int(-1), ctypes.c_int(-1)
    rc = emub.emu_block_verify(len(pks), b"".join(pks), B, b"".join(bitmaps), blen, b"".join(sigs), b"".join(msgs), 48, G, S,
                               seed[0], seed[1], equal_members, res, gok, ctypes.byref(bf), ctypes.byref(fb))
    assert rc == 0, rc
    return res.raw[:B], gok.raw[:B // G], bf.value, fb.value


def expected(oracle, pks, bitmaps, sigs, msgs):
    h = oracle.committee(pks)
    return bytes(1 if oracle.committee_aggregate_verify(h, bm, s, m) else 0 for bm, s, m in zip(bitmaps, sigs, msgs))


def test_block_all_valid(emub, oracle):
    pks, blen, bitmaps, sigs, msgs = make_batch(oracle, 10, 18, seed=1)      # 4 groups of 4 in 2 blocks of 2 (S = 2) + a tail of 2
    res, gok, bf, fb = run(emub, pks, blen, bitmaps, sigs, msgs, S=2)
    assert res == b"\x01" * 18 and gok == b"\x01" * 4 and bf == 0 and fb == 0


def test_block_wrong_message_falls_back_per_group(emub, oracle):
    pks, blen, bitmaps, sigs, msgs = make_batch(oracle, 10, 18, seed=2)
    msgs[5] = bytes([msgs[5][0] ^ 1]) + msgs[5][1:]                          # round 5 = group 1 (position 1) = block 1 with group 3
    want = expected(oracle, pks, bitmaps, sigs, msgs)
    assert want == bytes(0 if j == 5 else 1 for j in range(18))
    res, gok, bf, fb = run(emub, pks, blen, bitmaps, sigs, msgs, S=2)
    assert res == want and gok == b"\x01\x00\x01\x01" and bf == 1 and fb == 2    # both groups of block 1 checked alone


def test_block_undecodable_and_identity_rounds(emub, oracle):
    pks, blen, bitmaps, sigs, msgs = make_batch(oracle, 10, 18, seed=3)
    sigs[2] = b"\xff" * 96                                                   # does not decode: group 2 is flagged bad, no check of its own
    bitmaps[7] = bytes(blen)                                                 # empty bitmap: identity aggregate key
    sigs[12] = bytes(96)                                                     # identity signature
    sigs[17] = b"\xff" * 96                                                  # in the exactly verified tail
    want = expected(oracle, pks, bitmaps, sigs, msgs)
    res, gok, bf, fb = run(emub, pks, blen, bitmaps, sigs, msgs, S=2)
    assert res == want and want.count(0) == 4 and gok == b"\x00\x01\x00\x00" and bf == 2
    assert fb == 1                  # groups 0, 2, 3 hold flagged rounds and need no check of their own; clean group 1 shares block 1 with 3


def test_block_uneven_members_and_tail(emub, oracle):
    """ng = 5 groups (not a multiple of the block size) with S = 2: block 0 = groups 0, 2, 4, block 1 = groups 1, 3; 3 tail rounds.
    Then the library's own stride (S = 32 here: every group its own block)."""
    pks, blen, bitmaps, sigs, msgs = make_batch(oracle, 10, 23, seed=4)
    sigs[9], sigs[13] = sigs[13], sigs[9]                                    # two valid points swapped between groups 4 and 3
    want = expected(oracle, pks, bitmaps, sigs, msgs)
    assert want.count(0) == 2
    res, gok, bf, fb = run(emub, pks, blen, bitmaps, sigs, msgs, S=2)
    assert res == want and bf == 2 and fb == 5 and gok == b"\x01\x01\x01\x00\x00"
    res, gok, bf, fb = run(emub, pks, blen, bitmaps, sigs, msgs, S=0)
    assert res == want and bf == 2 and fb == 2


def test_block_cross_group_cancellation(emub, oracle):
    """sigma_a + D and sigma_b - D at the same position of two groups of one block: with the coefficients of the group form (equal for
    every member of the block) the two errors cancel in the block's product and both rounds pass; with a draw per member they do not."""
    R = 0x73eda753299d7d483339d80809a1d80553bda402fffe5bfeffffffff00000001
    pks, blen, bitmaps, sigs, msgs = make_batch(oracle, 10, 16, seed=5)      # 4 groups of 4, S = 2: block 0 = groups 0 and 2
    d = wl.seeded_sk("emub/D", 0); mD = wl.commit_payload("emub/D", 0)
    D, negD = oracle.sign_hash(wl.sk_bytes(d), mD), oracle.sign_hash(wl.sk_bytes(R - d), mD)
    a, b = 4, 6                                                              # position 1 of groups 0 and 2
    sigs[a] = oracle.aggregate_sigs([sigs[a], D]); sigs[b] = oracle.aggregate_sigs([sigs[b], negD])
    want = expected(oracle, pks, bitmaps, sigs, msgs)
    assert want == bytes(0 if j in (a, b) else 1 for j in range(16))
    fooled, _, bf, _ = run(emub, pks, blen, bitmaps, sigs, msgs, S=2, equal_members=1)
    assert fooled == b"\x01" * 16 and bf == 0
    res, gok, bf, fb = run(emub, pks, blen, bitmaps, sigs, msgs, S=2)
    assert res == want and gok == b"\x00\x01\x00\x01" and bf == 1 and fb == 2


# ---------------------------------------------------------------------------------------------------------------- GPU
@pytest.mark.gpu
def test_block_path_full_batch_one_pct_invalid(gbls, oracle):
    """The benchmark's batch (270 336 rounds = 33 792 groups of 8 = 2 112 blocks of 16, block path chosen automatically) with 1 % of
    the rounds invalid: wrong messages, undecodable signatures, and pairs sigma_a + D / sigma_b - D at one position of two groups of
    one block (they would cancel under equal coefficients).  Exactly the injected rounds are rejected, with the group verdicts of the
    form without blocks."""
    import bench
    R = 0x73eda753299d7d483339d80809a1d80553bda402fffe5bfeffffffff00000001
    B, G = 270336, 8
    ng = B // G; S = ((ng + 15) // 16 + 31) // 32 * 32
    assert S == 2112 and gbls.GetParam("rlc_block") == 0
    sks = bench.make_committee_sks()
    pks_blob = gbls.GetPublicKeyBatch(b"".join(wl.sk_bytes(k) for k in sks))
    com = gbls.Committee([pks_blob[48 * i:48 * i + 48] for i in range(len(sks))])
    bitmaps, agg_sk, msgs, nsig = bench.make_rounds(sks, B, seed=4242)
    sigs, ok = gbls.SignHashBatch(agg_sk, msgs, 48)
    assert ok == b"\x01" * B
    assert com.AggregateVerifyBatch(bitmaps, sigs, msgs, 48) == b"\x01" * B
    assert gbls.LastBatchInfo()["groups_failed"] == 0
    rng = random.Random(91)
    mm = bytearray(msgs); sg = bytearray(sigs); bad = set()
    d = wl.seeded_sk("blk/D", 0); mD = wl.commit_payload("blk/D", 0)
    D, negD = oracle.sign_hash(wl.sk_bytes(d), mD), oracle.sign_hash(wl.sk_bytes(R - d), mD)
    while len(bad) < 900:                                        # 450 cross-group pairs: same position k, groups g and g + m S
        k, g = rng.randrange(G), rng.randrange(ng); g2 = (g % S) + S * rng.randrange(ng // S)
        ja, jb = k * ng + g, k * ng + g2
        if g2 == g or ja in bad or jb in bad: continue
        sg[96 * ja:96 * ja + 96] = oracle.aggregate_sigs([bytes(sg[96 * ja:96 * ja + 96]), D])
        sg[96 * jb:96 * jb + 96] = oracle.aggregate_sigs([bytes(sg[96 * jb:96 * jb + 96]), negD])
        bad |= {ja, jb}
    for j in rng.sample([j for j in range(B) if j not in bad], B // 100 - len(bad)):
        if rng.random() < 0.8: mm[48 * j + 11] ^= 0x08
        else: sg[96 * j:96 * j + 96] = b"\xff" * 96
        bad.add(j)
    res = com.AggregateVerifyBatch(bitmaps, bytes(sg), bytes(mm), 48)
    info = gbls.LastBatchInfo()
    assert {j for j in range(B) if res[j] != 1} == bad
    assert info["group_size"] == G and info["groups_failed"] == len({j % ng for j in bad})
    # 7.7 % of the groups failed: the next call checks its groups one by one (device-side choice, same coefficients), and a clean
    # batch after it goes back to blocks
    assert com.AggregateVerifyBatch(bitmaps, bytes(sg), bytes(mm), 48) == res
    assert gbls.LastBatchInfo()["groups_failed"] == info["groups_failed"]
    assert com.AggregateVerifyBatch(bitmaps, sigs, msgs, 48) == b"\x01" * B
    assert com.AggregateVerifyBatch(bitmaps, sigs, msgs, 48) == b"\x01" * B
    try:
        gbls.SetParam("rlc_block", 2)                            # the same batch, every group checked on its own
        assert com.AggregateVerifyBatch(bitmaps, bytes(sg), bytes(mm), 48) == res
        assert gbls.LastBatchInfo()["groups_failed"] == info["groups_failed"]
    finally:
        gbls.SetParam("rlc_block", 0)
