"""hbls_aggregate_sigs_batch and its device form: B AggregateSig calls in one device call.

GPU: every set's bytes and status equal what hbls_aggregate_sigs gives for it alone (HBLS_ERR_DECODE <-> AGG_BAD_SIG_ENCODING and the
identity) and what the CPU oracle gives, at B = 1, 64 and 1 024 with set sizes from 0 to 1 000 mixed and one set of 20 000; the device
form writes the same bytes, also when captured once into a CUDA graph and replayed on new inputs, and neither form draws coefficients
or touches hbls_last_batch_info.
CPU: the new leader's GetM2M3Bitmaps equals GetM2Bitmap / GetM3Bitmap over the oracle-backed stand-in backend."""
import random
import pytest
from harmony_b200 import workload as wl
from harmony_b200 import consensus as cs
from test_consensus import OracleBackend, build_storm

AGG_OK, AGG_BAD_SIG_ENCODING, AGG_BAD_RANGE = 32, 33, 34
BAD_ENCODINGS = [b"\xff" * 96, (1).to_bytes(48, "little") + bytes(48)]        # x >= p; x = 1 is not on the curve


# ------------------------------------------------------------------ CPU: the self-test's known answers
def test_aggb_kat_header_regenerates_byte_for_byte():
    """harmony_b200/csrc/selftest_kat_aggb.h (the aggregate_sigs_batch leg) is what tools/gen_selftest_aggb.py writes"""
    import os, subprocess, sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    r = subprocess.run([sys.executable, os.path.join(root, "tools", "gen_selftest_aggb.py"), "--check"], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0 and "up to date" in r.stdout, r.stdout + r.stderr


# ------------------------------------------------------------------ CPU: NEWVIEW aggregates over the oracle backend
class OracleBatchBackend(OracleBackend):
    """the stand-in backend with the batch call: one oracle AggregateSig per set"""
    def aggregate_sigs_batch(self, sets):
        self.calls["aggregate_sigs_batch"] = self.calls.get("aggregate_sigs_batch", 0) + 1
        ident = self.o.aggregate_sigs([])
        aggs, st = [], []
        for s in sets:
            a = self.o.aggregate_sigs(list(s))
            aggs.append(a if a is not None else ident); st.append(AGG_OK if a is not None else AGG_BAD_SIG_ENCODING)
        return aggs, st


def test_m2m3_bitmaps_one_call_host_logic(oracle):
    n, viewID = 24, 77
    sign = lambda sk, m: oracle.sign_hash(wl.sk_bytes(sk), m)
    sks, pks, msgs, faults, payload = build_storm(n, 18, sign, lambda ks: [oracle.get_public_key(wl.sk_bytes(k)) for k in ks], viewID)
    be = OracleBatchBackend(oracle)
    vc = cs.viewChange(pks, backend=be)
    vc.ProcessViewChangeMsgs(msgs)
    m2, m3 = vc.GetM2Bitmap(viewID), vc.GetM3Bitmap(viewID)
    assert m2[0] is not None and m3[0] is not None
    assert vc.GetM2M3Bitmaps(viewID) == (m2, m3) and be.calls["aggregate_sigs_batch"] == 1
    # the other view id of the storm has M2 and M3 of one sender; an unknown view id has neither (no call)
    assert vc.GetM2M3Bitmaps(viewID + 5) == (vc.GetM2Bitmap(viewID + 5), vc.GetM3Bitmap(viewID + 5))
    assert vc.GetM2M3Bitmaps(viewID + 99) == ((None, None), (None, None)) and be.calls["aggregate_sigs_batch"] == 2
    # only M3 signatures (every sender sent M1): M2 stays (None, None)
    vc.nilSigs.pop(viewID)
    assert vc.GetM2M3Bitmaps(viewID) == ((None, None), m3)
    # a stored signature that does not decode fails as AggregateSigBytes does
    vc.viewIDSigs[viewID]["bad"] = BAD_ENCODINGS[0]
    with pytest.raises(ValueError):
        vc.GetM2M3Bitmaps(viewID)


def test_m2m3_bitmaps_device_backend_calls_the_batch(monkeypatch):
    """the product backend forwards to bls.AggregateSigsBatch (one call for both aggregates)"""
    from harmony_b200 import bls
    seen = []
    monkeypatch.setattr(bls, "AggregateSigsBatch", lambda sets: (seen.append(sets), ([b"\x01" * 96] * len(sets), [AGG_OK] * len(sets)))[1])
    vc = cs.viewChange.__new__(cs.viewChange)
    vc.be = cs.DeviceBackend(); vc.nilSigs = {3: {"a": b"s" * 96}}; vc.viewIDSigs = {3: {"a": b"s" * 96, "b": b"t" * 96}}
    vc.nilBitmap = {3: bytearray(b"\x01")}; vc.viewIDBitmap = {3: bytearray(b"\x03")}
    assert vc.GetM2M3Bitmaps(3) == ((b"\x01" * 96, b"\x01"), (b"\x01" * 96, b"\x03"))
    assert seen == [[[b"s" * 96], [b"s" * 96, b"t" * 96]]]


# ------------------------------------------------------------------ GPU
_POOL = {}


def _pool(gbls):
    """256 valid signatures (distinct keys and messages), signed on the device"""
    if "sigs" not in _POOL:
        sks = b"".join(wl.sk_bytes(wl.seeded_sk("aggb", i)) for i in range(256))
        msgs = b"".join(wl.commit_payload("aggb", i) for i in range(256))
        sigs, ok = gbls.SignHashBatch(sks, msgs, 48)
        assert ok == b"\x01" * 256
        _POOL["sigs"] = [sigs[96 * i:96 * i + 96] for i in range(256)]
    return _POOL["sigs"]


def _sets(gbls, sizes, seed, bad_sets=0.2):
    """sets of the given sizes drawn from the pool; a share bad_sets of them gets one undecodable signature"""
    rng = random.Random(seed)
    pool = _pool(gbls)
    sets = []
    for sz in sizes:
        s = [rng.choice(pool) for _ in range(sz)]
        if s and rng.random() < bad_sets: s[rng.randrange(sz)] = rng.choice(BAD_ENCODINGS)
        sets.append(s)
    return sets


def _sizes(B, seed):
    rng = random.Random(seed)
    fixed = [0, 1, 127, 128, 129, 1000, 256, 0]
    return (fixed + [rng.randrange(1001) for _ in range(B)])[:B]


def _single(gbls, s):
    try: return gbls.AggregateSigBytes(s), AGG_OK
    except ValueError: return gbls.AggregateSigBytes([]), AGG_BAD_SIG_ENCODING


def _check_host(gbls, oracle, sets, oracle_every=1):
    aggs, st = gbls.AggregateSigsBatch(sets)
    ident = oracle.aggregate_sigs([])
    for j, s in enumerate(sets):
        assert (aggs[j], st[j]) == _single(gbls, s), j
        if j % oracle_every == 0:
            o = oracle.aggregate_sigs(s)
            assert aggs[j] == (o if o is not None else ident) and st[j] == (AGG_OK if o is not None else AGG_BAD_SIG_ENCODING), j
    return aggs, st


@pytest.mark.gpu
@pytest.mark.parametrize("B", [1, 64, 1024])
def test_batch_matches_single_calls_and_oracle(gbls, oracle, B):
    sets = _sets(gbls, _sizes(B, B), seed=B)
    aggs, st = _check_host(gbls, oracle, sets, oracle_every=1 if B <= 64 else 61)
    if B > 1: assert AGG_OK in st and AGG_BAD_SIG_ENCODING in st


@pytest.mark.gpu
def test_batch_with_a_set_of_20000(gbls, oracle):
    sets = _sets(gbls, [3, 20000, 0, 1000], seed=20000, bad_sets=0)
    sets.append(list(sets[1][:19999]) + [BAD_ENCODINGS[1]])
    aggs, st = _check_host(gbls, oracle, sets, oracle_every=1)
    assert st == [AGG_OK] * 4 + [AGG_BAD_SIG_ENCODING]


@pytest.mark.gpu
def test_empty_and_argument_errors(gbls):
    import ctypes
    L = gbls.lib()
    assert gbls.AggregateSigsBatch([]) == ([], [])
    aggs, st = gbls.AggregateSigsBatch([[], []])
    assert st == [AGG_OK] * 2 and aggs == [gbls.AggregateSigBytes([])] * 2
    out = ctypes.create_string_buffer(96 * 2); s = ctypes.create_string_buffer(2)
    sig = _pool(gbls)[0]
    for offs in ([1, 1, 1], [0, 1, 0]):                                     # offsets[0] != 0, decreasing
        assert L.hbls_aggregate_sigs_batch(2, (ctypes.c_uint64 * 3)(*offs), sig, out, s) == gbls.ERR_ARG
    assert L.hbls_aggregate_sigs_batch(2, None, sig, out, s) == gbls.ERR_ARG
    assert L.hbls_aggregate_sigs_batch(1, (ctypes.c_uint64 * 2)(0, 1), None, out, s) == gbls.ERR_ARG
    assert L.hbls_aggregate_sigs_batch(1, (ctypes.c_uint64 * 2)(0, 1), sig, None, s) == gbls.ERR_ARG
    assert L.hbls_aggregate_sigs_batch(0, None, None, None, None) == 0


def _dev_inputs(sets):
    import torch
    offs = [0]
    for s in sets: offs.append(offs[-1] + len(s))
    blob = b"".join(r for s in sets for r in s)
    sigs = torch.frombuffer(bytearray(blob or b"\x00" * 96), dtype=torch.uint8).cuda().view(-1, 96)[:offs[-1]]
    return torch.tensor(offs, dtype=torch.int64, device="cuda"), sigs


def _host_bytes(aggs, st):
    import torch
    torch.cuda.synchronize()
    out = aggs.cpu().numpy().tobytes()
    return [out[96 * j:96 * j + 96] for j in range(aggs.shape[0])], list(st.cpu().numpy().tobytes())


@pytest.mark.gpu
@pytest.mark.parametrize("B", [1, 64, 1024])
def test_device_form_equals_host_form(gbls, B):
    import torch
    sets = _sets(gbls, _sizes(B, B + 1), seed=B + 1)
    want = gbls.AggregateSigsBatch(sets)
    offs, sigs = _dev_inputs(sets)
    assert _host_bytes(*gbls.AggregateSigsBatchDevice(offs, sigs)) == want
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    got = gbls.AggregateSigsBatchDevice(offs, sigs, stream=side)
    side.synchronize()
    assert _host_bytes(*got) == want


@pytest.mark.gpu
def test_device_form_bad_ranges(gbls):
    """ranges the host form refuses: a reversed range or one past row n -> BAD_RANGE and the identity; the other sets as the host
    form gives them, overlapping ones included"""
    import torch
    pool = _pool(gbls)
    rows = [pool[i % len(pool)] for i in range(300)]
    _, sigs = _dev_inputs([rows])
    ident = gbls.AggregateSigBytes([])
    def run(offsets):
        aggs, st = _host_bytes(*gbls.AggregateSigsBatchDevice(torch.tensor(offsets, dtype=torch.int64, device="cuda"), sigs))
        exp_st, exp_out = [], []
        for j in range(len(offsets) - 1):
            lo, hi = offsets[j], offsets[j + 1]
            if lo > hi or hi > 300: exp_st.append(AGG_BAD_RANGE); exp_out.append(ident)
            else: a, s = _single(gbls, rows[lo:hi]); exp_st.append(s); exp_out.append(a)
        assert st == exp_st and aggs == exp_out
        return st
    st = run([0, 300, 100, 250, 300, 301, 0, 200, 10 ** 12])
    assert st == [AGG_OK, AGG_BAD_RANGE, AGG_OK, AGG_OK, AGG_BAD_RANGE, AGG_BAD_RANGE, AGG_OK, AGG_BAD_RANGE]
    # five overlapping copies of all 300 rows: 15 chunks of 128 for a table of ceil(300 / 128) + 9 = 12 -- the sets past the table
    # are summed by their fold warps
    st = run([0, 300] * 5)
    assert st == [AGG_OK, AGG_BAD_RANGE] * 4 + [AGG_OK]


@pytest.mark.gpu
def test_launches_do_not_grow_with_B(gbls):
    counts = []
    for B in (2, 300):
        sets = _sets(gbls, [5] * B, seed=3, bad_sets=0)
        before = gbls.KernelLaunchCount()
        gbls.AggregateSigsBatch(sets)
        counts.append(gbls.KernelLaunchCount() - before)
    assert counts[0] == counts[1] <= 6


@pytest.mark.gpu
def test_graph_capture_and_replay(gbls):
    """captured once on torch.cuda.graph's stream; replays with new offsets and signatures copied into the captured tensors give the
    host form's bytes; no coefficient is drawn and hbls_last_batch_info keeps describing the last direct batch call"""
    import torch
    B, n = 48, 6000
    def inputs(seed):
        r = random.Random(seed)
        cut = sorted(r.randrange(n + 1) for _ in range(B - 1))
        sizes = [b - a for a, b in zip([0] + cut, cut + [n])]
        return _sets(gbls, sizes, seed=seed)
    sets0 = inputs(100)
    offs, sigs = _dev_inputs(sets0)
    com_sigs = _pool(gbls)[:4]
    pks = gbls.GetPublicKeyBatch(b"".join(wl.sk_bytes(wl.seeded_sk("aggb", i)) for i in range(4)))
    gbls.VerifyBatch(pks, b"".join(com_sigs), b"".join(wl.commit_payload("aggb", i) for i in range(4)), 48)   # a direct batch call
    info0 = gbls.LastBatchInfo()
    draws0 = gbls.GetParam("rlc_draws")
    gbls.AggregateSigsBatchDevice(offs, sigs)                     # warm the caching allocator; not needed by the library
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        out, st = gbls.AggregateSigsBatchDevice(offs, sigs)
    for seed in (101, 102, 103):
        sets = inputs(seed) if seed != 103 else sets0
        o2, s2 = _dev_inputs(sets)
        offs.copy_(o2); sigs.copy_(s2)
        g.replay()
        assert _host_bytes(out, st) == gbls.AggregateSigsBatch(sets), seed
    assert gbls.GetParam("rlc_draws") == draws0
    assert gbls.LastBatchInfo() == info0
