"""Device forms of the batch verifiers (hbls_verify_batch_status_device, hbls_verify_headers_device,
hbls_aggregate_verify_items_device) through the CUDA-tensor wrappers of harmony_b200/bls.py: byte for byte what the host forms
write, in every batching regime, for inputs at odd byte offsets, on two streams at once, asynchronously, without touching the H(m)
cache; the wrappers reject unusable tensors before any launch."""
import random
import pytest
from harmony_b200 import workload as wl

pytestmark = pytest.mark.gpu


def _dev(b, width, offset=0):
    """bytes -> uint8 CUDA tensor [len / width, width], starting `offset` bytes into its allocation"""
    import torch
    n = len(b) // width if width else 0
    buf = torch.zeros(len(b) + offset, dtype=torch.uint8, device="cuda")
    if b: buf[offset:] = torch.frombuffer(bytearray(b), dtype=torch.uint8).cuda()
    return buf[offset:].view(n, width) if width else buf[offset:].view(n, 0)


def _host(t):
    import torch
    torch.cuda.synchronize()
    return t.cpu().numpy().tobytes()


def _triples(gbls, tag, k, nmsg=None):
    """k triples, messages from a pool of nmsg (None: all distinct), with every reject class at seeded positions"""
    sks = b"".join(wl.sk_bytes(wl.seeded_sk(tag, i % 64)) for i in range(k))
    msgs = b"".join(wl.seeded_bytes(tag + "/m", i if nmsg is None else i % nmsg, 32) for i in range(k))
    pks = bytearray(gbls.GetPublicKeyBatch(sks))
    sigs, _ = gbls.SignHashBatch(sks, msgs, 32)
    sigs, msgs = bytearray(sigs), bytearray(msgs)
    rng = random.Random(tag)
    for t, i in enumerate(rng.sample(range(k), min(k, 10)) if k > 1 else []):
        kind = t % 5
        if kind == 0: pks[48 * i:48 * i + 48] = b"\xff" * 48                     # key does not decode
        elif kind == 1: sigs[96 * i:96 * i + 96] = b"\xff" * 96                  # signature does not decode
        elif kind == 2: msgs[32 * i + 3] ^= 0x40                                 # wrong message
        elif kind == 3: pks[48 * i:48 * i + 48] = pks[48 * ((i + 1) % k):48 * ((i + 1) % k) + 48]   # wrong key
        else: pks[48 * i:48 * i + 48] = b"\xff" * 48; sigs[96 * i:96 * i + 96] = b"\xff" * 96    # both: the key is reported
    return bytes(pks), bytes(sigs), bytes(msgs)


class _Params:
    def __init__(self, gbls, **kv): self.g, self.kv = gbls, kv
    def __enter__(self):
        self.old = {k: self.g.GetParam(k) for k in self.kv}
        for k, v in self.kv.items(): self.g.SetParam(k, v)
    def __exit__(self, *a):
        for k, v in self.old.items(): self.g.SetParam(k, v)


@pytest.mark.parametrize("k,nmsg,params", [
    (1, None, {}),
    (97, None, {}),                                    # below coop_max: warp per round, warp per message
    (500, 3, {}),                                      # the view-change shape: 500 triples over 3 messages
    (600, 40, {"hash_coop_max": 8}),                   # lane pair per message
    (5000, None, {}),                                  # between coop_max and rlc_min: thread per message, exact checks
    (5000, 7, {"coop_max": 16}),                       # few messages beyond the latency path
    (2000, None, {"rlc_min": 16}),                     # batched groups with bad rounds and the exact pass
])
def test_triples_match_host_form(gbls, oracle, k, nmsg, params):
    pks, sigs, msgs = _triples(gbls, f"dev-tri-{k}-{nmsg}", k, nmsg)
    with _Params(gbls, **params):
        want = gbls.VerifyBatchStatus(pks, sigs, msgs, 32)
        info_host = gbls.LastBatchInfo()
        got = _host(gbls.VerifyBatchStatusDevice(_dev(pks, 48), _dev(sigs, 96), _dev(msgs, 32)))
        info_dev = gbls.LastBatchInfo()
    assert got == want
    assert {k_: v for k_, v in info_dev.items() if k_ not in ("groups_failed", "rounds_rechecked")} == \
           {k_: v for k_, v in info_host.items() if k_ not in ("groups_failed", "rounds_rechecked")}
    if params.get("rlc_min") == 16:
        assert info_dev["mode"] == 1 and info_dev["groups_failed"] > 0
    assert {4, 3, 0} <= set(got) or k == 1
    for i in [i for i in range(k) if got[i] != 1][:12]:
        p, s, m = pks[48 * i:48 * i + 48], sigs[96 * i:96 * i + 96], msgs[32 * i:32 * i + 32]
        exp = 4 if not oracle.pk_check(p) else 3 if not oracle.sig_check(s) else (1 if oracle.verify_hash(s, p, m) else 0)
        assert got[i] == exp, i


def _committee(gbls, tag, n):
    sks = [wl.seeded_sk(tag, i) for i in range(n)]
    blob = gbls.GetPublicKeyBatch(b"".join(wl.sk_bytes(s) for s in sks))
    return sks, gbls.Committee([blob[48 * i:48 * i + 48] for i in range(n)])


def _headers(gbls, oracle, sks, n, N, npay):
    bms = [bytearray(wl.bitmap_with_k("dev-hdr", j, n, [167, 200, 250, 120][j % 4])) for j in range(N)]
    pays = [bytearray(wl.commit_payload("dev-hdr", j % npay)) for j in range(N)]
    sig_blob, _ = gbls.SignHashBatch(b"".join(wl.sk_bytes(wl.round_signer_sum(sks, bytes(b))) for b in bms), b"".join(bytes(m) for m in pays), 48)
    sigs = bytearray(sig_blob)
    pays[3][12] ^= 1
    bms[9][31] |= 0xfc                                   # padding bits never count
    sigs[96 * 5:96 * 6] = b"\xff" * 96
    sigs[96 * 6:96 * 7] = sigs[96 * 7:96 * 8]
    return bytes(sigs), b"".join(bytes(b) for b in bms), b"".join(bytes(p) for p in pays)


@pytest.mark.parametrize("N,npay,params", [(40, 5, {}), (300, 300, {"rlc_min": 16}), (64, 2, {"coop_max": 0})])
def test_headers_match_host_form(gbls, oracle, N, npay, params):
    n = 250
    sks, com = _committee(gbls, "dev-hdr", n)
    sigs, bms, pays = _headers(gbls, oracle, sks, n, N, npay)
    with _Params(gbls, **params):
        for q in (wl.quorum_k(n), 0):
            want = com.VerifyHeaders(sigs, bms, pays, 48, q)
            got = _host(com.VerifyHeadersDevice(_dev(sigs, 96, 1), _dev(bms, 32, 3), _dev(pays, 48, 5), q))
            assert got == want, q
            assert (gbls.HDR_NO_QUORUM in set(got)) == (q != 0) and gbls.HDR_BAD_ENCODING in set(got) and gbls.HDR_BAD_SIG in set(got)


def test_items_over_committees_of_different_sizes(gbls, oracle):
    sizes = [50, 130, 250, 13]
    coms, skss = [], []
    for s in sizes:
        sks, com = _committee(gbls, f"dev-items-{s}", s); coms.append(com); skss.append(sks)
    K = 48; which = [j % len(sizes) for j in range(K)]
    bms = [wl.bitmap_with_k(f"dev-items/{j}", j, sizes[which[j]], max(1, sizes[which[j]] * 2 // 3 + j % 5)) for j in range(K)]
    msgs = [wl.commit_payload("dev-items", j % 4) for j in range(K)]                # 4 messages, as in a crosslink batch
    sigs = bytearray(gbls.SignHashBatch(b"".join(wl.sk_bytes(wl.round_signer_sum(skss[which[j]], bms[j])) for j in range(K)), b"".join(msgs), 48)[0])
    sigs[96 * 7:96 * 8] = sigs[96 * 8:96 * 9]; sigs[96 * 30:96 * 31] = b"\xff" * 96
    items = [coms[w] for w in which]
    for params in ({}, {"rlc_min": 16}):
        with _Params(gbls, **params):
            want = gbls.AggregateVerifyItems(items, bms, bytes(sigs), b"".join(msgs), 48)
            got = _host(gbls.AggregateVerifyItemsDevice(items, _dev(b"".join(bms), 1, 1).view(-1), _dev(bytes(sigs), 96, 7), _dev(b"".join(msgs), 48, 3)))
        assert got == want and [j for j in range(K) if got[j] == 0] == [7, 30], params
    # one committee: the bitmaps as [k, blen]
    sel = list(range(2, K, 4))
    sb, ss, sm = [bms[j] for j in sel], b"".join(bytes(sigs[96 * j:96 * j + 96]) for j in sel), b"".join(msgs[j] for j in sel)
    got = _host(gbls.AggregateVerifyItemsDevice([coms[2]] * len(sel), _dev(b"".join(sb), 32), _dev(ss, 96), _dev(sm, 48)))
    assert got == gbls.AggregateVerifyItems([coms[2]] * len(sel), sb, ss, sm, 48)
    assert [i for i in range(len(sel)) if got[i] == 0] == [sel.index(30)]                  # item 30's undecodable signature


def test_two_streams_in_flight_and_cache_untouched(gbls):
    import torch
    a = _triples(gbls, "dev-s0", 3000, 5); b = _triples(gbls, "dev-s1", 3000)
    want_a = gbls.VerifyBatchStatus(*a, 32); want_b = gbls.VerifyBatchStatus(*b, 32)
    ta = [_dev(x, w) for x, w in zip(a, (48, 96, 32))]; tb = [_dev(x, w) for x, w in zip(b, (48, 96, 32))]
    s0, s1 = torch.cuda.Stream(), torch.cuda.Stream()
    torch.cuda.synchronize()
    cache = gbls.HashCacheStats()
    outs = []
    for _ in range(3):
        outs.append((gbls.VerifyBatchStatusDevice(*ta, stream=s0), gbls.VerifyBatchStatusDevice(*tb, stream=s1)))
    torch.cuda.synchronize()
    for oa, ob in outs:
        assert _host(oa) == want_a and _host(ob) == want_b
    assert gbls.HashCacheStats() == cache


def test_calls_return_before_the_stream_runs(gbls):
    import torch
    n = 250
    sks, com = _committee(gbls, "dev-async", n)
    sigs, bms, pays = _headers(gbls, None, sks, n, 24, 3)
    tri = _triples(gbls, "dev-async", 400, 3)
    tt = [_dev(x, w) for x, w in zip(tri, (48, 96, 32))]
    th = (_dev(sigs, 96), _dev(bms, 32), _dev(pays, 48))
    bmi = _dev(bms, 32).view(-1)
    st = torch.cuda.Stream()
    calls = [lambda: gbls.VerifyBatchStatusDevice(*tt, stream=st), lambda: com.VerifyHeadersDevice(*th, 0, stream=st),
             lambda: gbls.AggregateVerifyItemsDevice([com] * 24, bmi, th[0], th[2], stream=st)]
    first = [c() for c in calls]                                                   # scratch and staging exist from here on
    torch.cuda.synchronize()
    for c, f in zip(calls, first):
        with torch.cuda.stream(st):
            torch.cuda._sleep(200_000_000)                                         # ~0.1 s of device time queued before the call
        out = c()
        assert not st.query()
        st.synchronize()
        assert _host(out) == _host(f)
    assert _host(first[0]) == gbls.VerifyBatchStatus(*tri, 32)
    assert _host(first[1]) == com.VerifyHeaders(sigs, bms, pays, 48, 0)
    assert _host(first[2]) == gbls.AggregateVerifyItems([com] * 24, [bms[32 * j:32 * j + 32] for j in range(24)], sigs, pays, 48)


def test_tensor_validation(gbls):
    import torch
    pks, sigs, msgs = (_dev(bytes(48 * 4), 48), _dev(bytes(96 * 4), 96), _dev(bytes(32 * 4), 32))
    bad = [
        (pks.cpu(), sigs, msgs),                                   # on the CPU
        (pks, sigs.to(torch.int16), msgs),                         # wrong dtype
        (pks, torch.zeros(96, 4, dtype=torch.uint8, device="cuda").t(), msgs),     # non-contiguous
        (pks[:3], sigs, msgs),                                     # inconsistent rows
        (pks, sigs, msgs.view(-1)),                                # not [k, len]
        (pks, _dev(bytes(95 * 4), 95), msgs),                      # wrong width
        (b"\x00" * 192, sigs, msgs),                               # not a tensor
    ]
    if torch.cuda.device_count() > 1:
        bad.append((pks.to("cuda:1"), sigs, msgs))                 # another device
    _, com = _committee(gbls, "dev-val", 20)
    torch.cuda.synchronize()
    launches = gbls.KernelLaunchCount()
    for args in bad:
        with pytest.raises(gbls.HblsError):
            gbls.VerifyBatchStatusDevice(*args)
    with pytest.raises(gbls.HblsError):
        com.VerifyHeadersDevice(sigs, _dev(bytes(4 * 2), 2), msgs, 0)                 # blen 3 expected
    with pytest.raises(gbls.HblsError):
        gbls.AggregateVerifyItemsDevice([com] * 4, _dev(bytes(11), 1).view(-1), sigs, msgs)      # 12 bitmap bytes expected
    assert gbls.KernelLaunchCount() == launches
    L = gbls.lib()
    assert L.hbls_verify_headers_device(com.h, 4, sigs.data_ptr(), 0, 2, msgs.data_ptr(), 32, 0, 0, None) == gbls.ERR_ARG
    assert L.hbls_verify_batch_status_device(4, pks.data_ptr(), sigs.data_ptr(), msgs.data_ptr(), 32, None, None) == gbls.ERR_ARG
    assert L.hbls_verify_batch_status_device(0, None, None, None, 32, None, None) == 0


def test_default_stream_orders_inputs_and_output(gbls):
    """stream=None runs on torch's current stream even when that is the legacy default stream: inputs written there after a long
    sleep are read after they land, and `.cpu()` of the output (no device-wide synchronise) sees the finished statuses."""
    import torch
    pks, sigs, msgs = _triples(gbls, "dev-default", 300, 3)
    want = gbls.VerifyBatchStatus(pks, sigs, msgs, 32)
    gbls.VerifyBatchStatusDevice(_dev(pks, 48), _dev(sigs, 96), _dev(msgs, 32))             # scratch for this size exists from here on
    torch.cuda.synchronize()
    host = [torch.frombuffer(bytearray(b), dtype=torch.uint8).view(-1, w).pin_memory() for b, w in ((pks, 48), (sigs, 96), (msgs, 32))]
    assert torch.cuda.current_stream().cuda_stream == 0
    for _ in range(2):
        dev = [torch.empty(h.shape, dtype=torch.uint8, device="cuda") for h in host]
        torch.cuda._sleep(200_000_000)                                                        # the inputs land ~0.1 s from now
        for d, h in zip(dev, host): d.copy_(h, non_blocking=True)
        out = gbls.VerifyBatchStatusDevice(*dev)
        assert not torch.cuda.current_stream().query()
        assert out.cpu().numpy().tobytes() == want


def test_single_triple_every_reject_class(gbls, oracle):
    sks = b"".join(wl.sk_bytes(wl.seeded_sk("dev-one", i)) for i in range(2))
    pks = gbls.GetPublicKeyBatch(sks)
    m = wl.seeded_bytes("dev-one/m", 0, 32)
    p, s = pks[:48], gbls.SignHashBatch(sks[:32], m, 32)[0]
    cases = {"valid": (p, s, m), "bad key": (b"\xff" * 48, s, m), "bad signature": (p, b"\xff" * 96, m),
             "wrong message": (p, s, bytes([m[0] ^ 1]) + m[1:]), "wrong key": (pks[48:], s, m), "both encodings": (b"\xff" * 48, b"\xff" * 96, m)}
    got = {}
    for name, (cp, cs, cm) in cases.items():
        want = gbls.VerifyBatchStatus(cp, cs, cm, 32)
        got[name] = _host(gbls.VerifyBatchStatusDevice(_dev(cp, 48, 1), _dev(cs, 96, 3), _dev(cm, 32, 5)))
        assert got[name] == want, name
    assert got == {"valid": b"\x01", "bad key": b"\x04", "bad signature": b"\x03", "wrong message": b"\x00", "wrong key": b"\x00",
                   "both encodings": b"\x04"}


def test_empty_batches(gbls):
    import torch
    _, com = _committee(gbls, "dev-empty", 20)
    e = lambda w: torch.empty(0, w, dtype=torch.uint8, device="cuda")
    assert gbls.VerifyBatchStatusDevice(e(48), e(96), e(32)).numel() == 0
    assert com.VerifyHeadersDevice(e(96), e(3), e(48), 14).numel() == 0 and com.VerifyHeaders(b"", b"", b"", 48, 14) == b""
    assert gbls.AggregateVerifyItemsDevice([], torch.empty(0, dtype=torch.uint8, device="cuda"), e(96), e(48)).numel() == 0
