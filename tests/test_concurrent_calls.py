"""GPU: herumi-API calls from many threads at once (include/hbls.h: threading).  Concurrent calls are combined into shared device
turns; every caller must still get exactly the result of its own call -- the oracle's booleans and bytes, and the struct bytes of
the same call made alone.  ctypes releases the GIL around each call, so the Python threads really overlap."""
import os, subprocess, threading
import pytest
from harmony_b200 import workload as wl

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

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

def test_concurrent_verify_hash(gbls, oracle):
    """64 threads x 32 triples: messages shared across threads and distinct, of 0, 1, 8, 32, 48 and 64 bytes; wrong messages,
    swapped keys, identity keys and other threads' signatures among them."""
    T, K = 64, 32
    lens = [0, 1, 8, 32, 48, 64]
    sks = [wl.sk_bytes(wl.seeded_sk("cc-v", i)) for i in range(T)]
    pks = [oracle.get_public_key(k) for k in sks]
    shared = [wl.seeded_bytes("cc-v/shared", i, ln) for i, ln in enumerate(lens)]
    cases = []                                          # per thread: (key index, sig96, msg, identity key?)
    for t in range(T):
        row = []
        for k in range(K):
            ln = lens[(t + k) % len(lens)]
            msg = shared[(t + k) % len(lens)] if k % 3 == 0 else wl.seeded_bytes(f"cc-v/{t}", k, ln)
            # the empty message (and any that maps to t = 0, e.g. b"\x00") has no signature: sign another one
            sign_msg = msg if oracle.map_to_g2(msg) is not None else shared[3]
            sig = oracle.sign_hash(sks[t], sign_msg)
            key, ident = t, False
            kind = k % 8
            if kind == 1: msg = bytes([msg[0] ^ 1]) + msg[1:] if msg else b"\x01"       # wrong message
            elif kind == 3: key = (t + 5) % T                                            # swapped key
            elif kind == 5: ident = True                                                 # identity key
            elif kind == 7: sig = oracle.sign_hash(sks[(t + 1) % T], sign_msg)           # another thread's signature
            row.append((key, sig, msg, ident))
        cases.append(row)
    want = [[False if ident else oracle.verify_hash(sig, pks[key], msg) for key, sig, msg, ident in row] for row in cases]
    assert sum(map(sum, want)) > T * K // 3 and sum(map(sum, want)) < T * K
    got = [[None] * K for _ in range(T)]
    s0 = gbls.CoalesceStats()
    def caller(t):
        pk_structs = {}
        for i in (t, (t + 5) % T):
            pk_structs[i] = gbls.PublicKey(); pk_structs[i].Deserialize(pks[i])
        for k, (key, sig96, msg, ident) in enumerate(cases[t]):
            s = gbls.Sign(); s.Deserialize(sig96)
            got[t][k] = s.VerifyHash(gbls.PublicKey() if ident else pk_structs[key], msg)
    run_threads(T, caller)
    s1 = gbls.CoalesceStats()
    assert got == want
    turns, requests = s1["turns"] - s0["turns"], s1["requests"] - s0["requests"]
    assert requests == T * (2 + 2 * K) and turns < requests and s1["max_turn"] > 1, (s0, s1)

def test_concurrent_sign_and_public_key(gbls, oracle):
    T, K = 32, 8
    sks = [[wl.sk_bytes(wl.seeded_sk(f"cc-s/{t}", k)) for k in range(K)] for t in range(T)]
    msgs = [[wl.seeded_bytes(f"cc-s/m{t}", k, 32) if k % 2 else wl.commit_payload("cc-s", k) for k in range(K)] for t in range(T)]
    def structs(t):
        out = []
        for k in range(K):
            sk = gbls.SecretKey(); sk.Deserialize(sks[t][k])
            pk = sk.GetPublicKey(); sig = sk.SignHash(msgs[t][k])
            out.append((bytes(pk.v), bytes(sig.v), pk.Serialize(), sig.Serialize()))
        return out
    alone = [structs(t) for t in range(0, T, 4)]                # the same calls made one at a time
    got = [None] * T
    def caller(t): got[t] = structs(t)
    run_threads(T, caller)
    for t in range(T):
        for k in range(K):
            pk_struct, sig_struct, pk48, sig96 = got[t][k]
            assert pk48 == oracle.get_public_key(sks[t][k]) and sig96 == oracle.sign_hash(sks[t][k], msgs[t][k]), (t, k)
            if t % 4 == 0: assert (pk_struct, sig_struct) == alone[t // 4][k][:2], (t, k)

def test_concurrent_single_element_ops(gbls, oracle):
    """Deserialize (valid and undecodable), Serialize, Add, Sub, IsEqual and hbls_map_to_g2 from 16 threads at once."""
    T, K = 16, 6
    sks = [wl.sk_bytes(wl.seeded_sk("cc-o", i)) for i in range(T * K + 1)]
    pks = [oracle.get_public_key(k) for k in sks]
    msgs = [wl.seeded_bytes("cc-o/m", i, 32) for i in range(T * K + 1)]
    sigs = [oracle.sign_hash(k, m) for k, m in zip(sks, msgs)]
    junk = b"\xff" * 48
    def ops(t):
        out = []
        for k in range(K):
            i = t * K + k
            a, b = gbls.PublicKey(), gbls.PublicKey(); a.Deserialize(pks[i]); b.Deserialize(pks[i + 1])
            s, s2 = gbls.Sign(), gbls.Sign(); s.Deserialize(sigs[i]); s2.Deserialize(sigs[i + 1])
            bad = gbls.PublicKey()
            try: bad.Deserialize(junk); bad_ok = True
            except ValueError: bad_ok = False
            c = a.copy(); c.Add(b); added = c.Serialize()
            c.Sub(b); back = c.IsEqual(a)
            d = a.copy(); d.Sub(b); subbed = d.Serialize()
            s.Add(s2)
            out.append((bad_ok, added, back, subbed, s.Serialize(), a.IsEqual(b), gbls.MapToG2(msgs[i]), gbls.MapToG2(bytes(32))))
        return out
    serial = [ops(t) for t in range(0, T, 4)]
    got = [None] * T
    def caller(t): got[t] = ops(t)
    run_threads(T, caller)
    for t in range(T):
        for k in range(K):
            i = t * K + k
            bad_ok, added, back, subbed, sig_sum, eq, h, h0 = got[t][k]
            assert not bad_ok and back and not eq and h0 is None
            assert added == oracle.pk_add(pks[i], pks[i + 1]) and subbed == oracle.pk_add(pks[i], pks[i + 1], sub=True)
            assert sig_sum == oracle.sig_add(sigs[i], sigs[i + 1]) and h == oracle.map_to_g2(msgs[i])
            if t % 4 == 0: assert got[t][k] == serial[t // 4][k]

def test_mask_set_bit_from_threads(gbls, oracle):
    """8 threads set disjoint bits of one 250-slot mask, then clear half of them: no thread undoes another's bits."""
    n = 250
    pks = gbls.GetPublicKeyBatch(b"".join(wl.sk_bytes(wl.seeded_sk("cc-m", i)) for i in range(n)))
    pks = [pks[48 * i:48 * i + 48] for i in range(n)]
    com = gbls.Committee(pks); m = gbls.DeviceMask(com)
    def setter(t):
        for i in range(t, n, 8): m.SetBit(i, True)
        for i in range(t, n, 16): m.SetBit(i, False)
    run_threads(8, setter)
    want = bytearray((n + 7) // 8)
    for i in range(n):
        if i % 16 >= 8: want[i >> 3] |= 1 << (i & 7)
    want = bytes(want)
    assert m.Mask() == want and m.CountEnabled() == sum(bin(x).count("1") for x in want)
    assert m.AggregatePublicBytes() == oracle.mask_aggregate(pks, want)

def test_cpp_threads_through_header(gbls, tmp_path):
    from harmony_b200 import build
    exe = str(tmp_path / "hbls_concurrency_test")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-Wall", "-o", exe, os.path.join(ROOT, "harmony_b200", "host", "hbls_concurrency_test.cpp"),
                           "-L" + build.LIBDIR, "-lhbls", "-Wl,-rpath," + build.LIBDIR, "-pthread"])
    r = subprocess.run([exe], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0 and "all checks passed" in r.stdout, r.stdout + r.stderr
