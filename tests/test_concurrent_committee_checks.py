"""Single committee checks from many threads at once: hbls_aggregate_verify (Committee.AggregateVerify) and hbls_mask_verify
(DeviceMask.VerifyHash) join the turns of the herumi-API combiner (include/hbls.h: threading), beside blsVerifyHash / blsSignHash.

GPU: every caller gets the oracle's boolean and the result of the same call made alone; the combiner shows shared turns; a lone
call launches exactly the kernels it launched before it could be combined and records the same hbls_last_batch_info; argument
errors return HBLS_ERR_ARG before any turn.  CPU: one combined turn of mixed kinds over two committees runs through the turn's
kernels in host emulation (tests/emu/emu_part1_committee.cpp) and gives the oracle's verdicts."""
import ctypes, os, re, subprocess, threading
import pytest
from harmony_b200 import workload as wl

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ERR_ARG = -2
RQ_VERIFY, RQ_AGG, RQ_MASK = 0, 4, 5


def reject_sigs():
    """x >= p, off the curve, outside the subgroup: the G2 reject encodings of the self-test's known answers"""
    src = open(os.path.join(ROOT, "harmony_b200", "csrc", "selftest_kat.h")).read()
    body = re.search(r"st_g2_rej\[3\]\[96\] = \{(.*?)\};", src, re.S).group(1)
    flat = bytes(int(x, 16) for x in re.findall(r"0x([0-9a-f]{2})", body))
    return [flat[96 * i:96 * i + 96] for i in range(3)]


def flip_bit(bm, i):
    b = bytearray(bm); b[i >> 3] ^= 1 << (i & 7); return bytes(b)


def committee_cases(tag, n, sks, pks_h, oracle, sign, rej):
    """(bitmap, sig96, msg, expected) for one committee: valid rounds with messages of 1 to 64 bytes (some sharing their first 48
    bytes), then a wrong message, another round's signature, a flipped bitmap bit, padding bits, an empty bitmap, the three reject
    encodings and the t = 0 message"""
    blen = (n + 7) >> 3
    lens = [1, 7, 32, 48, 49, 64, 64, 56]
    base = wl.seeded_bytes(f"{tag}/shared", 0, 64)
    msgs = []
    for j, ln in enumerate(lens):
        msgs.append(base[:ln] if j >= 4 else wl.seeded_bytes(f"{tag}/m", j, ln))      # j >= 4: the same first 48 bytes
    bms = [wl.bitmap_with_k(tag, j, n, max(1, (2 * n) // 3 + j % 5)) for j in range(len(msgs))]
    sigs = [sign(wl.round_signer_sum(sks, bm), m) for bm, m in zip(bms, msgs)]
    cases = [(bm, s, m) for bm, s, m in zip(bms, sigs, msgs)]
    cases.append((bms[0], sigs[0], bytes([msgs[2][0] ^ 1]) + msgs[2][1:]))                # wrong message
    cases.append((bms[1], sigs[2], msgs[1]))                                                # another round's signature
    cases.append((flip_bit(bms[3], n // 2), sigs[3], msgs[3]))                              # a flipped bitmap bit
    if n % 8:
        pad = bytearray(bms[2]); pad[-1] |= 0xff & ~((1 << (n % 8)) - 1)
        cases.append((bytes(pad), sigs[2], msgs[2]))                                        # padding bits set in the last byte
    cases.append((bytes(blen), sigs[0], msgs[0]))                                           # empty bitmap
    for r in rej: cases.append((bms[0], r, msgs[0]))                                        # x >= p, off the curve, outside the subgroup
    t0 = bytes(48)
    cases.append((bms[0], sigs[0], t0))                                                     # the t = 0 message
    return [(bm, s, m, oracle.committee_aggregate_verify(pks_h, bm, s, m) == 1) for bm, s, m in cases]


@pytest.fixture(scope="module")
def world(gbls, oracle):
    """three committees (16, 250 and 1 000 keys), their check cases, one resident mask per committee with its cases, and
    VerifyHash / SignHash triples"""
    rej = reject_sigs()
    sign = lambda sk_int, m: oracle.sign_hash(wl.sk_bytes(sk_int), m)
    out = {"committees": [], "masks": [], "triples": []}
    for n in (16, 250, 1000):
        tag = f"ccc/{n}"
        sks = [wl.seeded_sk(tag, i) for i in range(n)]
        blob = gbls.GetPublicKeyBatch(b"".join(wl.sk_bytes(k) for k in sks))
        pks = [blob[48 * i:48 * i + 48] for i in range(n)]
        h = oracle.committee(pks)
        com = gbls.Committee(pks)
        cases = committee_cases(tag, n, sks, h, oracle, sign, rej)
        out["committees"].append((com, cases))
        mbm = wl.bitmap_with_k(tag + "/mask", 0, n, (2 * n) // 3 + 1)
        mask = gbls.DeviceMask(com); mask.SetMask(mbm)
        mm = [wl.seeded_bytes(tag + "/mask/m", j, 48) for j in range(3)]
        msig = sign(wl.round_signer_sum(sks, mbm), mm[0])
        mcases = [(msig, mm[0]), (msig, mm[1]), (sign(wl.round_signer_sum(sks, mbm), mm[2]), mm[2]), (rej[2], mm[0]), (msig, bytes(48))]
        out["masks"].append((mask, [(s, m, oracle.committee_aggregate_verify(h, mbm, s, m) == 1) for s, m in mcases]))
    for i in range(6):
        sk = wl.sk_bytes(wl.seeded_sk("ccc/tri", i)); m = wl.seeded_bytes("ccc/tri/m", i, 32)
        pk = oracle.get_public_key(sk); sig = oracle.sign_hash(sk, m)
        vm = m if i % 3 else bytes([m[0] ^ 1]) + m[1:]
        out["triples"].append((sk, pk, sig, vm, oracle.verify_hash(sig, pk, vm), oracle.sign_hash(sk, vm)))
    return out


def ops_of(world, gbls):
    """every call of the mix as (label, zero-argument function returning its result, expected)"""
    ops = []
    for c, (com, cases) in enumerate(world["committees"]):
        for k, (bm, s, m, want) in enumerate(cases):
            ops.append((f"agg{c}.{k}", (lambda com=com, bm=bm, s=s, m=m: com.AggregateVerify(bm, s, m)), want))
    for c, (mask, cases) in enumerate(world["masks"]):
        for k, (s, m, want) in enumerate(cases):
            ops.append((f"mask{c}.{k}", (lambda mask=mask, s=s, m=m: mask.VerifyHash(s, m)), want))
    for t, (sk, pk, sig, vm, want, want_sig) in enumerate(world["triples"]):
        def verify(pk=pk, sig=sig, vm=vm):
            p = gbls.PublicKey(); p.Deserialize(pk); g = gbls.Sign(); g.Deserialize(sig)
            return g.VerifyHash(p, vm)
        def signh(sk=sk, vm=vm):
            x = gbls.SecretKey(); x.Deserialize(sk); r = x.SignHash(vm)
            return None if r is None else r.Serialize()
        ops.append((f"verify{t}", verify, want))
        ops.append((f"sign{t}", signh, want_sig))
    return ops


def run_threads(n, fn):
    errors = []
    def body(t):
        try: fn(t)
        except BaseException as e: errors.append((t, repr(e)))
    th = [threading.Thread(target=body, args=(t,)) for t in range(n)]
    for x in th: x.start()
    for x in th: x.join(timeout=600)
    assert not any(x.is_alive() for x in th), "a caller thread did not finish"
    assert not errors, errors[:5]


@pytest.mark.gpu
@pytest.mark.parametrize("T", [16, 64])
def test_concurrent_committee_and_mask_checks(gbls, world, T):
    ops = ops_of(world, gbls)
    assert sum(1 for _, _, w in ops if w is True) > 10 and sum(1 for _, _, w in ops if w is False) > 10
    alone = [f() for _, f, _ in ops]                                    # the same calls made one at a time
    assert alone == [w for _, _, w in ops], [l for (l, _, w), a in zip(ops, alone) if a != w]
    # each thread runs the whole mix, rotated by its index: the same call from different threads lands in different turns
    got = [[None] * len(ops) for _ in range(T)]
    s0, h0 = gbls.CoalesceStats(), gbls.HashCacheStats()
    def caller(t):
        for k in range(len(ops)):
            i = (k + 3 * t) % len(ops)
            got[t][i] = ops[i][1]()
    run_threads(T, caller)
    s1, h1 = gbls.CoalesceStats(), gbls.HashCacheStats()
    for t in range(T):
        bad = [ops[i][0] for i in range(len(ops)) if got[t][i] != alone[i]]
        assert not bad, (t, bad)
    turns, requests = s1["turns"] - s0["turns"], s1["requests"] - s0["requests"]
    # Deserialize / SignHash structs add requests of their own; every check is one request
    assert requests >= T * len(ops) and turns < requests and s1["max_turn"] > 1, (s0, s1)
    # H(m): at most one cache lookup per request with a message (one per distinct message of a turn), and at least one per distinct
    # message of the mix
    lookups = (h1["hits"] - h0["hits"]) + (h1["misses"] - h0["misses"])
    distinct = {m[:48].ljust(48, b"\0") for c in world["committees"] for _, _, m, _ in c[1]}
    distinct |= {m.ljust(48, b"\0") for c in world["masks"] for _, m, _ in c[1]} | {t[3].ljust(48, b"\0") for t in world["triples"]}
    assert len(distinct) <= lookups <= T * len(ops), (lookups, len(distinct))
    # the last turn that held committee checks recorded an exact-mode, warp-per-round batch
    bi = gbls.LastBatchInfo()
    assert bi["mode"] == 0 and bi["cta_threads"] == 32 and 1 <= bi["rounds"] <= T and bi["groups"] == 0, bi


@pytest.mark.gpu
def test_hash_cache_off_does_not_count(gbls, world):
    ops = [o for o in ops_of(world, gbls) if o[0].startswith(("agg", "mask"))]
    old = gbls.GetParam("hm_cache")
    gbls.SetParam("hm_cache", 0)
    try:
        h0 = gbls.HashCacheStats()
        got = [None] * len(ops)
        def caller(t):
            for i in range(t, len(ops), 16): got[i] = ops[i][1]()
        run_threads(16, caller)
        assert got == [w for _, _, w in ops]
        assert gbls.HashCacheStats() == h0
    finally:
        gbls.SetParam("hm_cache", old)


# one round of the 250-key committee, checked alone: the launches and the batch record of the path a lone call has always taken
# (values of the build before these checks could be combined: H(m) on the warp, decode and hash beside the key sum on two streams,
# the split Miller loop; with the H(m) cache warm, the two Miller values and the subgroup test in parallel)
LONE_AGG_LAUNCHES = {"cold": 7, "miss": 7, "hit": 8}
LONE_MASK_LAUNCHES = {"cold": 5, "miss": 5, "hit": 4}
LONE_AGG_INFO = {"mode": 0, "group_size": 0, "rounds": 1, "groups": 0, "groups_failed": 0, "rounds_rechecked": 0, "tail_rounds": 0,
                 "cta_threads": 32}


@pytest.mark.gpu
def test_lone_calls_keep_their_launches(gbls, world):
    com, cases = world["committees"][1]
    mask, mcases = world["masks"][1]
    bm, s, m, want = cases[0]
    ms, mm, mwant = mcases[0]
    old = gbls.GetParam("hm_cache")
    try:
        for mode in ("cold", "miss", "hit"):
            gbls.SetParam("hm_cache", 0 if mode == "cold" else 1)
            if mode == "miss":
                # messages no earlier call has hashed: the cache misses; the checks are false, the launches are those of any round
                fresh = [wl.seeded_bytes("ccc/lone", j, 48) for j in range(2)]
                k0 = gbls.KernelLaunchCount(); assert com.AggregateVerify(bm, s, fresh[0]) is False
                assert gbls.KernelLaunchCount() - k0 == LONE_AGG_LAUNCHES[mode]
                k0 = gbls.KernelLaunchCount(); assert mask.VerifyHash(ms, fresh[1]) is False
                assert gbls.KernelLaunchCount() - k0 == LONE_MASK_LAUNCHES[mode]
                continue
            if mode == "hit":
                com.AggregateVerify(bm, s, m); mask.VerifyHash(ms, mm)                # both messages in the cache
            k0 = gbls.KernelLaunchCount(); assert com.AggregateVerify(bm, s, m) is want
            assert gbls.KernelLaunchCount() - k0 == LONE_AGG_LAUNCHES[mode], mode
            assert gbls.LastBatchInfo() == LONE_AGG_INFO, mode
            k0 = gbls.KernelLaunchCount(); assert mask.VerifyHash(ms, mm) is mwant
            assert gbls.KernelLaunchCount() - k0 == LONE_MASK_LAUNCHES[mode], mode
            assert gbls.LastBatchInfo() == LONE_AGG_INFO, mode                       # a mask check records no batch
    finally:
        gbls.SetParam("hm_cache", old)


@pytest.mark.gpu
def test_argument_errors_never_join_a_turn(gbls, world):
    L = gbls.lib()
    com, cases = world["committees"][0]
    mask, _ = world["masks"][0]
    bm, s, m, _ = cases[0]
    s0 = gbls.CoalesceStats(); k0 = gbls.KernelLaunchCount()
    assert L.hbls_aggregate_verify(com.h, bm + b"\0", len(bm) + 1, s, m, len(m)) == ERR_ARG         # bitmap length
    assert L.hbls_aggregate_verify(com.h, bm[:-1], len(bm) - 1, s, m, len(m)) == ERR_ARG
    assert L.hbls_aggregate_verify(None, bm, len(bm), s, m, len(m)) == ERR_ARG                      # null committee
    assert L.hbls_aggregate_verify(com.h, bm, len(bm), None, m, len(m)) == ERR_ARG                  # null signature
    assert L.hbls_mask_verify(None, s, m, len(m)) == ERR_ARG
    assert L.hbls_mask_verify(mask.h, None, m, len(m)) == ERR_ARG
    assert gbls.CoalesceStats() == s0 and gbls.KernelLaunchCount() == k0
    with pytest.raises(ValueError): com.AggregateVerify(bm + b"\0", s, m)


# ---------------------------------------------------------------------------------------------------------------- CPU
@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    src = os.path.join(ROOT, "tests", "emu", "emu_part1_committee.cpp")
    out = str(tmp_path_factory.mktemp("emu") / "libhbls_emu_part1_committee.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-pthread", "-o", out, src])
    L = ctypes.CDLL(out)
    P = ctypes.POINTER
    L.emu_committee_turn.argtypes = [ctypes.c_size_t, ctypes.c_char_p, P(ctypes.c_uint32), ctypes.c_size_t, P(ctypes.c_int), P(ctypes.c_int),
                                     ctypes.c_char_p, ctypes.c_char_p, ctypes.c_char_p, ctypes.c_char_p, P(ctypes.c_uint32), ctypes.c_char_p]
    return L


def test_emu_combined_turn_of_mixed_kinds(emu, oracle):
    """one turn: committee checks against a 12-key and a 21-key committee (valid, wrong message, empty bitmap, padding bits, an
    undecodable and an out-of-subgroup signature, messages sharing their first 48 bytes), two mask checks and two VerifyHash
    requests, in arrival order mixed across kinds"""
    rej = reject_sigs()
    coms = []
    for n in (12, 21):
        sks = [wl.seeded_sk(f"emu-cc/{n}", i) for i in range(n)]
        pks = [oracle.get_public_key(wl.sk_bytes(k)) for k in sks]
        coms.append((n, sks, pks, oracle.committee(pks)))
    shared = wl.seeded_bytes("emu-cc/shared", 0, 64)
    reqs = []                                   # (kind, committee, bitmap, pk48, sig96, msg)
    for c, (n, sks, pks, h) in enumerate(coms):
        bm = wl.bitmap_with_k(f"emu-cc/{n}", 0, n, n // 2 + 1)
        m = shared[:40 + 8 * c]                                             # 40 and 48 bytes
        sig = oracle.sign_hash(wl.sk_bytes(wl.round_signer_sum(sks, bm)), m)
        pad = bytearray(bm); pad[-1] |= 0xff & ~((1 << (n % 8)) - 1)
        reqs += [(RQ_AGG, c, bm, None, sig, m), (RQ_AGG, c, bm, None, sig, bytes([m[0] ^ 4]) + m[1:]),
                 (RQ_MASK, c, bm, None, sig, m), (RQ_AGG, c, bytes(len(bm)), None, sig, m), (RQ_AGG, c, bytes(pad), None, sig, m),
                 (RQ_AGG, c, bm, None, rej[1 + c], m)]
    sk = wl.sk_bytes(wl.seeded_sk("emu-cc/tri", 0)); pk = oracle.get_public_key(sk)
    tm = shared[:48] + b"tail"                                                # shares its first 48 bytes with the 48-byte message
    reqs.insert(3, (RQ_VERIFY, 0, b"", pk, oracle.sign_hash(sk, tm), tm))
    reqs.insert(7, (RQ_VERIFY, 0, b"", pk, oracle.sign_hash(sk, tm), wl.seeded_bytes("emu-cc/other", 0, 32)))
    want = []
    for kind, c, bm, p, s, m in reqs:
        want.append(oracle.verify_hash(s, p, m) if kind == RQ_VERIFY else oracle.committee_aggregate_verify(coms[c][3], bm, s, m) == 1)
    assert 3 <= sum(want) < len(want)
    k = len(reqs)
    keys = b"".join(b"".join(pks) for _, _, pks, _ in coms)
    sizes = (ctypes.c_uint32 * 2)(*[n for n, _, _, _ in coms])
    kinds = (ctypes.c_int * k)(*[r[0] for r in reqs]); cidx = (ctypes.c_int * k)(*[r[1] for r in reqs])
    bitmaps = b"".join(r[2] for r in reqs if r[0] != RQ_VERIFY)
    pk48 = b"".join(r[3] if r[3] else bytes(48) for r in reqs); sig96 = b"".join(r[4] for r in reqs)
    msgs = b"".join(r[5].ljust(64, b"\0") for r in reqs); lens = (ctypes.c_uint32 * k)(*[len(r[5]) for r in reqs])
    res = ctypes.create_string_buffer(k)
    assert emu.emu_committee_turn(2, keys, sizes, k, kinds, cidx, bitmaps, pk48, sig96, msgs, lens, res) == 0
    assert [b == 1 for b in res.raw] == want, (list(res.raw), want)
