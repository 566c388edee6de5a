"""Built-in self-test (hbls_self_test, include/hbls.h).

CPU: the known answers in harmony_b200/csrc/selftest_kat.h are what oracle/gen_selftest.py writes, agree with the big-integer
oracle/pyref.py on a sample, and hold every reject class; the legs name every kernel hbls.cu launches; without a GPU the self-test
launches nothing.  GPU: the self-test passes, launches exactly those kernels, notices a flipped answer in each leg, leaves the
caller's state as it found it, and fails initialisation closed when HBLS_SELF_TEST=1 finds a wrong answer."""
import ctypes, os, re, subprocess, sys
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "harmony_b200", "csrc")
sys.path.insert(0, os.path.join(ROOT, "oracle"))


def _kat():
    """selftest_kat.h as {name: bytes or list of rows}"""
    src = open(os.path.join(CSRC, "selftest_kat.h")).read()
    out = {}
    for m in re.finditer(r"static const uint8_t (\w+)((?:\[\d+\])+) = (\{.*?\});", src, re.S):
        name, dims, body = m.group(1), [int(d) for d in re.findall(r"\d+", m.group(2))], m.group(3)
        flat = bytes(int(x, 16) for x in re.findall(r"0x([0-9a-f]{2})", body)) if "0x" in body else bytes(int(x) for x in re.findall(r"\d+", body))
        out[name] = flat if len(dims) == 1 else [flat[i * dims[1]:(i + 1) * dims[1]] for i in range(dims[0])]
    out["st_msg_len"] = [int(x) for x in re.search(r"st_msg_len\[\d+\] = \{([^}]*)\}", src).group(1).split(",")]
    return out


def _launch_set():
    src = open(os.path.join(CSRC, "hbls.cu")).read()
    return set(re.findall(r"\bLAUNCH(?:_SMEM)?\((k_\w+(?:<\w+>)?)", src))


def _leg_table():
    src = open(os.path.join(CSRC, "selftest.cuh")).read()
    body = src[src.index("const StLeg ST_LEGS[] = {"):src.index("constexpr int ST_NLEGS")]
    legs = []
    for m in re.finditer(r'\{"(\w+)",((?:\s*"[^"]*")+)\}', body):
        legs.append((m.group(1), set("".join(re.findall(r'"([^"]*)"', m.group(2))).split())))
    return legs


def test_kat_header_regenerates_byte_for_byte():
    r = subprocess.run([sys.executable, os.path.join(ROOT, "oracle", "gen_selftest.py"), "--check"], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0 and "up to date" in r.stdout, r.stdout + r.stderr


def test_kat_sample_agrees_with_pyref():
    import pyref as o
    k = _kat()
    sk = int.from_bytes(k["st_sk"][5], "little")
    assert o.g1_serialize(o.get_public_key(sk)) == k["st_pk"][5]
    m3 = k["st_msg"][3][:k["st_msg_len"][3]]
    assert o.g2_serialize(o.map_to_g2(m3)) == k["st_hm"][3]
    m5 = k["st_msg"][5][:k["st_msg_len"][5]]                  # 64 bytes: only the first 48 enter the map
    assert len(m5) == 64 and o.g2_serialize(o.map_to_g2(m5[:48])) == k["st_hm"][5]
    sk1 = int.from_bytes(k["st_sk"][1], "little")
    m1 = k["st_msg"][1][:k["st_msg_len"][1]]
    sig = o.g2_deserialize(k["st_sig"][1]); pk = o.g1_deserialize(k["st_pk"][1])
    assert o.g2_serialize(o.sign_hash(sk1, m1)) == k["st_sig"][1]
    assert o.verify_hash(sig, pk, m1) is True                                   # one valid verification
    assert o.verify_hash(sig, o.g1_deserialize(k["st_pk"][2]), m1) is False    # one invalid verification
    big = int.from_bytes(k["st_sk_big"], "little")
    assert big >= o.Z_ABS ** 4
    assert o.g2_serialize(o.pt_mul(o.FP2, o.map_to_g2(k["st_msg"][3][:k["st_msg_len"][3]]), big % o.R)) == k["st_sig_big"]


def test_kat_holds_every_reject_class(oracle):
    import pyref as o
    k = _kat()
    g1r, g2r = k["st_g1_rej"], k["st_g2_rej"]
    # x >= p
    assert int.from_bytes(g1r[0], "little") & ((1 << 383) - 1) >= o.P and int.from_bytes(g2r[0][:48], "little") >= o.P
    # not on the curve / on the curve but outside the subgroup
    assert o.g1_deserialize(g1r[1], False) is None and o.g2_deserialize(g2r[1], False) is None
    assert o.g1_deserialize(g1r[2], False) is not None and o.g1_deserialize(g1r[2], True) is None
    assert o.g2_deserialize(g2r[2], False) is not None and o.g2_deserialize(g2r[2], True) is None
    for b in g1r: assert not oracle.pk_check(b)
    for b in g2r: assert not oracle.sig_check(b)
    assert oracle.pk_check(bytes(48)) and oracle.sig_check(bytes(96))          # identity encodings decode
    # the triples and rounds carry the classes: identity key, empty bitmap, t = 0 message, wrong message, swapped signatures
    assert k["st_tri_pk"][8] == bytes(48) and k["st_tri_msg"][11] == bytes(32) and oracle.map_to_g2(bytes(32)) is None
    assert k["st_rnd_bm"][5] == bytes(2) and k["st_rnd_msg"][14] == bytes(48)
    assert k["st_rnd_sig"][6] == g2r[0] and k["st_rnd_sig"][13] == g2r[1] and k["st_rnd_sig"][10] == g2r[2]
    assert k["st_tri_pk"][6] == g1r[0] and k["st_tri_pk"][7] == g1r[2] and k["st_tri_sig"][9] == g2r[1]
    ok = k["st_rnd_ok"]
    assert [j for j in range(35) if not ok[j]] == [1, 2, 5, 6, 9, 10, 13, 14, 34]
    assert k["st_rnd_sig"][1] != k["st_rnd_sig"][9] and 1 % 4 == 9 % 4 and 1 % 8 == 9 % 8    # the swapped pair shares a group
    assert list(k["st_tri_status"]) == [1] * 6 + [4, 4, 0, 3, 0, 0]


def test_legs_cover_every_launched_kernel():
    covered = set().union(*(ks for _, ks in _leg_table()))
    launched = _launch_set()
    assert len(launched) > 50
    assert launched - covered == {"k_probe_carry<K>"}, launched - covered
    assert covered <= launched, covered - launched


def test_no_gpu_no_self_test():
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    code = ("import ctypes, sys; sys.path.insert(0, %r); from harmony_b200 import bls; L = bls.lib(); "
            "r = bls.SelfTestReport(); rc = L.hbls_self_test(ctypes.byref(r)); "
            "print(rc, L.hbls_kernel_launch_count(), L.hbls_self_test_kernels(None, 0))") % ROOT
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=120, env={**os.environ, "CUDA_VISIBLE_DEVICES": ""})
    assert r.returncode == 0, r.stderr
    assert r.stdout.split() == ["-100", "0", "0"]


# ---------------------------------------------------------------------------------------------------------------- GPU
def _state(gbls):
    from harmony_b200 import bls
    L = gbls.lib()
    names = ["rlc_min", "rlc_g", "tpsm", "tpsm_split", "tpsm_light", "coop_max", "overlap", "coop_wpsm", "hm_cache", "hash_coop_max",
             "mask_sort", "hash_split", "hash_fallback", "rlc_two_phase", "tpsm_cof", "tpsm_dec", "tpsm_scale", "tpsm_scale_g1",
             "scale_split", "decode_split", "exact_two_phase", "tpsm_lines", "tpsm_accum", "tpsm_sw", "selftest_flip"]
    bi = bls.BatchInfo(); rc = L.hbls_last_batch_info(ctypes.byref(bi))
    return {"params": {n: gbls.GetParam(n) for n in names}, "mode": gbls.GetBatchMode(), "stages": gbls.StageTimingGet(),
            "lines": gbls.StageTimingLinesMs(), "info": (rc, bi.as_dict()), "cache": gbls.HashCacheStats(), "coalesce": gbls.CoalesceStats()}


@pytest.mark.gpu
def test_self_test_passes_and_launches_every_kernel(gbls):
    rep = gbls.SelfTest()
    assert rep["rc"] == 0 and rep["failed"] == [] and rep["failed_legs"] == 0, rep
    names = [gbls.SelfTestLegName(i) for i in range(rep["legs"])]
    assert names == [n for n, _ in _leg_table()]
    got = set(gbls.SelfTestKernels())
    assert got == _launch_set() - {"k_probe_carry<K>"}, (sorted(_launch_set() - got), sorted(got - _launch_set()))
    assert rep["kernels"] == len(got)


@pytest.mark.gpu
def test_each_leg_notices_a_flipped_answer(gbls):
    legs = gbls.SelfTest()["legs"]
    for leg in range(legs):
        gbls.SetParam("selftest_flip", leg + 1)
        rep = gbls.SelfTest()
        assert rep["rc"] == 1 and rep["failed_legs"] == 1 << leg, (leg, rep)
        assert gbls.GetParam("selftest_flip") == 0
        assert gbls.SelfTest()["failed_legs"] == 0, leg


@pytest.mark.gpu
def test_self_test_leaves_state_as_found(gbls, oracle, fixtures):
    from harmony_b200 import workload as wl
    # a caller state that differs from the defaults everywhere the self-test forces something
    n = 16
    sks = [wl.seeded_sk("st-state", i) for i in range(n)]
    pks_blob = gbls.GetPublicKeyBatch(b"".join(wl.sk_bytes(k) for k in sks))
    com = gbls.Committee([pks_blob[48 * i:48 * i + 48] for i in range(n)])
    B = 40
    bms = [wl.bitmap_with_k("st-state", j, n, 9 + j % 7) for j in range(B)]
    msgs = [wl.commit_payload("st-state", j) for j in range(B)]
    sigs, _ = gbls.SignHashBatch(b"".join(wl.sk_bytes(wl.round_signer_sum(sks, bm)) for bm in bms), b"".join(msgs), 48)
    names = ("rlc_min", "coop_max", "hash_split", "overlap", "mask_sort", "hm_cache", "rlc_g")
    old = {k: gbls.GetParam(k) for k in names}
    try:
        gbls.SetParam("rlc_min", 32); gbls.SetParam("coop_max", 7); gbls.SetParam("hash_split", 1); gbls.SetParam("overlap", 0)
        gbls.SetParam("mask_sort", 0); gbls.SetParam("rlc_g", 4); gbls.SetParam("hm_cache", 1)
        gbls.StageTimingEnable(True)
        for m in msgs[:5]: gbls.HashPrefetch(m)
        com.AggregateVerifyBatch(b"".join(bms), sigs, b"".join(msgs), 48)
        before = _state(gbls)
        assert gbls.SelfTest()["failed"] == []
        after = _state(gbls)
        assert after == before
        # the H(m) cache entries survived: the prefetched messages are hits, exactly as before
        sk = gbls.SecretKey(); sk.Deserialize(wl.sk_bytes(sks[0]))
        h0 = gbls.HashCacheStats()["hits"]
        sk.SignHash(msgs[2])
        assert gbls.HashCacheStats()["hits"] == h0 + 1
    finally:
        gbls.StageTimingEnable(False); gbls.SetBatchMode(1)
        for k, v in old.items(): gbls.SetParam(k, v)
    # golden calls afterwards give the same bytes
    sv = fixtures["sig_vectors"][0]
    sk = gbls.SecretKey(); sk.DeserializeHexStr(sv["sk"])
    msg = bytes.fromhex(sv["msg"])
    assert sk.SignHash(msg).SerializeToHexStr() == sv["sig"]
    pk = gbls.PublicKey(); pk.DeserializeHexStr(sv["pk"]); s2 = gbls.Sign(); s2.DeserializeHexStr(sv["sig"])
    assert s2.VerifyHash(pk, msg) and not s2.VerifyHash(pk, bytes([msg[0] ^ 1]) + msg[1:])


_INIT_SCRIPT = """
import ctypes, sys
sys.path.insert(0, %r)
from harmony_b200 import bls
L = bls.lib()
rc = L.blsInit(bls.BLS12_381, 46)
out = ctypes.create_string_buffer(96)
rc2 = L.hbls_map_to_g2(b"abc", 3, out)
sec = bls._Sec(); sec.d[0] = 5
pub = bls._Pub(); sig = bls._Sig()
L.blsGetPublicKey(ctypes.byref(pub), ctypes.byref(sec))
rc3 = L.blsSignHash(ctypes.byref(sig), ctypes.byref(sec), b"\\x01" * 32, 32)
ok = L.blsVerifyHash(ctypes.byref(sig), ctypes.byref(pub), b"\\x01" * 32, 32)
print("RESULT", rc, rc2, rc3, ok, L.blsInit(bls.BLS12_381, 46))
"""


def _run_init(env_extra):
    env = {k: v for k, v in os.environ.items() if not k.startswith("HBLS_")}
    env.update(env_extra)
    r = subprocess.run([sys.executable, "-c", _INIT_SCRIPT % ROOT], capture_output=True, text=True, timeout=600, env=env)
    assert r.returncode == 0, r.stderr
    line = [l for l in r.stdout.splitlines() if l.startswith("RESULT")][0]
    return [int(x) for x in line.split()[1:]], r.stderr


@pytest.mark.gpu
def test_init_with_self_test_verifies():
    (rc, rc2, rc3, ok, again), _ = _run_init({"HBLS_SELF_TEST": "1"})
    assert rc == 0 and rc2 == 0 and rc3 == 0 and ok == 1 and again == 0


@pytest.mark.gpu
def test_init_self_test_failure_refuses_work():
    (rc, rc2, rc3, ok, again), err = _run_init({"HBLS_SELF_TEST": "1", "HBLS_SELFTEST_FLIP": "8"})      # leg 7: sign
    assert rc == -4 and rc2 == -4 and rc3 == -4 and ok == 0 and again == -4, err
    assert "self-test leg failed: sign" in err
