"""Committee sets (hbls_committee_set_*, hbls_aggregate_verify_set_device) through bls.CommitteeSet: the items of a multi-committee
batch name their committee by an int32 index tensor on the device.  The results are byte for byte what hbls_aggregate_verify_items
writes for the same items (and what the oracle says), in every batching regime; a bad index gives SET_BAD_INDEX and changes no other
byte; the call is asynchronous on its stream, leaves the H(m) cache alone, sets hbls_last_batch_info like the items forms, and can be
captured into a CUDA graph with no warm-up, replayed on new indices and inputs, drawing on the device at every replay."""
import ctypes, random
import pytest
from harmony_b200 import workload as wl

pytestmark = pytest.mark.gpu

SIZES = [50, 130, 250, 13, 1]


def _dev(b, width, offset=0):
    """bytes -> uint8 CUDA tensor [len / width, width], starting `offset` bytes into its allocation"""
    import torch
    n = len(b) // width
    buf = torch.zeros(len(b) + offset, dtype=torch.uint8, device="cuda")
    if b: buf[offset:] = torch.frombuffer(bytearray(b), dtype=torch.uint8).cuda()
    return buf[offset:].view(n, width)


def _idx(index):
    import torch
    return torch.tensor(index, dtype=torch.int32, device="cuda")


def _host(t):
    import torch
    torch.cuda.synchronize()
    return t.cpu().numpy().tobytes()


class _Params:
    def __init__(self, gbls, **kv): self.g, self.kv = gbls, kv
    def __enter__(self):
        self.old = {k: self.g.GetParam(k) for k in self.kv}
        for k, v in self.kv.items(): self.g.SetParam(k, v)
    def __exit__(self, *a):
        for k, v in self.old.items(): self.g.SetParam(k, v)


_C = {}


def _committees(gbls):
    """committees of SIZES slots (a one-slot committee included), their secret keys and public keys"""
    if "coms" not in _C:
        out = []
        for s in SIZES:
            sks = [wl.seeded_sk(f"cset-{s}", i) for i in range(s)]
            blob = gbls.GetPublicKeyBatch(b"".join(wl.sk_bytes(x) for x in sks))
            pks = [blob[48 * i:48 * i + 48] for i in range(s)]
            out.append((sks, pks, gbls.Committee(pks)))
        _C["coms"] = out
        _C["set"] = gbls.CommitteeSet([c for _, _, c in out])
    return _C["coms"], _C["set"]


def _items(gbls, index, tag, nmsg=4, bad_sigs=()):
    """items over the committees named by index (entries outside the set get a valid-looking signature and no bitmap): bitmaps back to
    back, signatures, 48-byte messages from nmsg payloads; bad_sigs = positions whose signature is another item's or undecodable"""
    coms, _ = _committees(gbls)
    m = len(coms)
    K = len(index)
    bms, agg = [], []
    for j, i in enumerate(index):
        if 0 <= i < m:
            n = SIZES[i]
            bm = wl.bitmap_with_k(f"{tag}/{j}", j, n, min(n, max(1, n * 2 // 3 + j % 5)))
            bms.append(bm); agg.append(wl.sk_bytes(wl.round_signer_sum(coms[i][0], bm)))
        else:
            bms.append(b""); agg.append(wl.sk_bytes(wl.seeded_sk(tag, j)))
    msgs = [wl.commit_payload(tag, j % nmsg) for j in range(K)]
    sigs = bytearray(gbls.SignHashBatch(b"".join(agg), b"".join(msgs), 48)[0])
    for t, j in enumerate(bad_sigs):
        if t % 2 == 0: o = (j + 1) % K; sigs[96 * j:96 * j + 96] = sigs[96 * o:96 * o + 96]
        else: sigs[96 * j:96 * j + 96] = b"\xff" * 96
    return bms, bytes(sigs), b"".join(msgs)


def _items_form(gbls, index, bms, sigs, msgs):
    """hbls_aggregate_verify_items over the items whose index is in the set, SET_BAD_INDEX elsewhere"""
    coms, _ = _committees(gbls)
    m = len(coms)
    good = [j for j, i in enumerate(index) if 0 <= i < m]
    res = gbls.AggregateVerifyItems([coms[index[j]][2] for j in good], [bms[j] for j in good],
                                    b"".join(sigs[96 * j:96 * j + 96] for j in good), b"".join(msgs[48 * j:48 * j + 48] for j in good), 48)
    out = bytearray([gbls.SET_BAD_INDEX] * len(index))
    for r, j in zip(res, good): out[j] = r
    return bytes(out)


def _set_call(gbls, index, bms, sigs, msgs, stream=None, offsets=(0, 0, 0, 0)):
    _, cset = _committees(gbls)
    return cset.AggregateVerifyDevice(_idx(index), _dev(b"".join(bms), 1, offsets[1]).view(-1), _dev(sigs, 96, offsets[2]),
                                      _dev(msgs, 48, offsets[3]), stream=stream)


REGIMES = [("warp", 48, {}), ("lane_pair", 64, {"coop_max": 0}), ("groups", 300, {"rlc_min": 16}),
           ("groups8", 600, {"rlc_min": 16, "rlc_g": 8})]


@pytest.mark.parametrize("regime,K,params", REGIMES, ids=[r[0] for r in REGIMES])
def test_matches_items_form_every_regime(gbls, oracle, regime, K, params):
    rng = random.Random(regime)
    index = [rng.randrange(len(SIZES)) for _ in range(K)]
    bad = [7, 8, 30] + ([161, 162] if K > 200 else [])         # 161 / 162: invalid rounds inside a batched group
    bms, sigs, msgs = _items(gbls, index, f"cset-{regime}", bad_sigs=bad)
    coms, cset = _committees(gbls)
    with _Params(gbls, **params):
        want = _items_form(gbls, index, bms, sigs, msgs)
        info_items = gbls.LastBatchInfo()
        got = _host(_set_call(gbls, index, bms, sigs, msgs, offsets=(0, 1, 7, 3)))
        assert gbls.LastBatchInfo() == info_items
        dev_items = _host(gbls.AggregateVerifyItemsDevice([coms[i][2] for i in index], _dev(b"".join(bms), 1).view(-1), _dev(sigs, 96), _dev(msgs, 48)))
    assert got == want == dev_items
    assert sorted(j for j in range(K) if got[j] != 1) == sorted(bad)
    if params.get("rlc_min"):
        assert info_items["mode"] == 1 and info_items["groups_failed"] >= 1
    for j in range(0, K, max(1, K // 24)):                                       # the oracle on a sample
        i = index[j]
        if ("och", i) not in _C: _C[("och", i)] = oracle.committee(coms[i][1])
        och = _C[("och", i)]
        assert got[j] == (1 if oracle.committee_aggregate_verify(och, bms[j], sigs[96 * j:96 * j + 96], msgs[48 * j:48 * j + 48]) == 1 else 0), j


@pytest.mark.parametrize("regime,K,params", REGIMES[:3], ids=[r[0] for r in REGIMES[:3]])
def test_bad_indices_change_no_other_byte(gbls, regime, K, params):
    coms, cset = _committees(gbls)
    m = len(coms)
    rng = random.Random("bad-" + regime)
    base = [rng.randrange(m) for _ in range(K)]
    bms, sigs, msgs = _items(gbls, base, f"cset-bad-{regime}", bad_sigs=[5])
    with _Params(gbls, **params):
        ref = _host(_set_call(gbls, base, bms, sigs, msgs))
        for places, value in (([0], -1), ([K // 2], m), ([K - 1], 2 ** 31 - 1), ([0, K // 2, K - 1], -7), (list(range(8, 16)), m + 3)):
            index = list(base)
            for p in places: index[p] = value
            ibms = [b"" if j in places else bms[j] for j in range(K)]               # a bad index occupies no bitmap bytes
            got = _host(_set_call(gbls, index, ibms, sigs, msgs))
            assert got == bytes(gbls.SET_BAD_INDEX if j in places else ref[j] for j in range(K)), places
            assert got == _items_form(gbls, index, ibms, sigs, msgs)


def test_empty_batch_and_argument_errors(gbls):
    import torch
    coms, cset = _committees(gbls)
    assert len(cset) == len(SIZES) and gbls.lib().hbls_committee_set_size(cset.h) == len(SIZES)
    e = lambda w: torch.empty(0, w, dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    launches = gbls.KernelLaunchCount()
    assert cset.AggregateVerifyDevice(torch.empty(0, dtype=torch.int32, device="cuda"), torch.empty(0, dtype=torch.uint8, device="cuda"),
                                      e(96), e(48)).numel() == 0
    L = gbls.lib()
    assert L.hbls_aggregate_verify_set_device(cset.h, 0, None, None, None, None, 48, None, None) == 0
    assert gbls.KernelLaunchCount() == launches                                   # k = 0 launches nothing
    idx = _idx([0, 1, 2, 3]); bm = _dev(bytes(64), 1).view(-1); sg = _dev(bytes(96 * 4), 96); ms = _dev(bytes(48 * 4), 48)
    out = torch.empty(4, dtype=torch.uint8, device="cuda")
    p = lambda t: t.data_ptr()
    assert L.hbls_aggregate_verify_set_device(None, 4, p(idx), p(bm), p(sg), p(ms), 48, p(out), None) == gbls.ERR_ARG
    assert L.hbls_aggregate_verify_set_device(cset.h, 4, None, p(bm), p(sg), p(ms), 48, p(out), None) == gbls.ERR_ARG
    assert L.hbls_aggregate_verify_set_device(cset.h, 4, p(idx), p(bm), p(sg), p(ms), 48, None, None) == gbls.ERR_ARG
    assert L.hbls_aggregate_verify_set_device(cset.h, 3, p(idx) + 2, p(bm), p(sg), p(ms), 48, p(out), None) == gbls.ERR_ARG   # not 4-byte aligned
    h = ctypes.c_void_p()
    arr = (ctypes.c_void_p * 2)(coms[0][2].h, None)
    assert L.hbls_committee_set_create(ctypes.byref(h), arr, 2) == gbls.ERR_ARG                  # a null entry
    assert L.hbls_committee_set_create(ctypes.byref(h), arr, 0) == gbls.ERR_ARG                  # m == 0
    assert L.hbls_committee_set_create(None, arr, 1) == gbls.ERR_ARG
    assert L.hbls_committee_set_create(ctypes.byref(h), None, 1) == gbls.ERR_ARG
    assert gbls.KernelLaunchCount() == launches
    for bad_idx in (idx.to(torch.int64), idx.cpu(), idx[:3], idx.view(2, 2)):
        with pytest.raises(gbls.HblsError):
            cset.AggregateVerifyDevice(bad_idx, bm, sg, ms)
    with pytest.raises(gbls.HblsError):
        cset.AggregateVerifyDevice(idx, bm.view(8, 8), sg, ms)                   # [rows, blen] with rows != k
    with pytest.raises(ValueError):
        gbls.CommitteeSet([])
    assert gbls.KernelLaunchCount() == launches


def test_two_streams_in_flight_and_cache_untouched(gbls):
    import torch
    ia = [j % len(SIZES) for j in range(400)]; ib = [(3 * j + 1) % len(SIZES) for j in range(700)]
    a = _items(gbls, ia, "cset-s0", bad_sigs=[3]); b = _items(gbls, ib, "cset-s1", nmsg=700, bad_sigs=[9, 10])
    want_a, want_b = _items_form(gbls, ia, *a), _items_form(gbls, ib, *b)
    _, cset = _committees(gbls)
    ta = (_idx(ia), _dev(b"".join(a[0]), 1).view(-1), _dev(a[1], 96), _dev(a[2], 48))
    tb = (_idx(ib), _dev(b"".join(b[0]), 1).view(-1), _dev(b[1], 96), _dev(b[2], 48))
    s0, s1 = torch.cuda.Stream(), torch.cuda.Stream()
    torch.cuda.synchronize()
    cache = gbls.HashCacheStats()
    outs = [(cset.AggregateVerifyDevice(*ta, stream=s0), cset.AggregateVerifyDevice(*tb, stream=s1)) for _ in range(3)]
    torch.cuda.synchronize()
    for oa, ob in outs:
        assert _host(oa) == want_a and _host(ob) == want_b
    assert gbls.HashCacheStats() == cache


def test_default_stream_orders_inputs_and_output(gbls):
    """stream=None on torch's legacy default stream: inputs written there after a long sleep are read after they land, and `.cpu()`
    of the output sees the finished results; the call returns before the stream runs"""
    import torch
    index = [j % len(SIZES) for j in range(40)]; index[11] = -1
    bms, sigs, msgs = _items(gbls, index, "cset-default", bad_sigs=[4])
    want = _items_form(gbls, index, bms, sigs, msgs)
    _, cset = _committees(gbls)
    assert _host(_set_call(gbls, index, bms, sigs, msgs)) == want                  # scratch for this size exists from here on
    host = [torch.tensor(index, dtype=torch.int32).pin_memory()] + \
           [torch.frombuffer(bytearray(b), dtype=torch.uint8).view(-1, w).pin_memory() for b, w in ((b"".join(bms), 1), (sigs, 96), (msgs, 48))]
    assert torch.cuda.current_stream().cuda_stream == 0
    for _ in range(2):
        dev = [torch.empty(h.shape, dtype=h.dtype, device="cuda") for h in host]
        torch.cuda._sleep(200_000_000)                                            # the inputs land ~0.1 s from now
        for d, h in zip(dev, host): d.copy_(h, non_blocking=True)
        out = cset.AggregateVerifyDevice(dev[0], dev[1].view(-1), dev[2], dev[3])
        assert not torch.cuda.current_stream().query()
        assert out.cpu().numpy().tobytes() == want


# ---- CUDA graphs
def _graph_inputs(gbls, K, seed):
    """K items over the set with a seeded index vector (bad indices included), bitmaps padded to the most bytes K items can take"""
    coms, _ = _committees(gbls)
    rng = random.Random(f"cset-graph/{K}/{seed}")
    index = [rng.randrange(len(SIZES)) for _ in range(K)]
    for j in rng.sample(range(K), 3): index[j] = rng.choice([-1, len(SIZES), -(2 ** 31)])
    bms, sigs, msgs = _items(gbls, index, f"cset-graph/{K}/{seed}", bad_sigs=rng.sample(range(K), 4))
    blob = b"".join(bms)
    return index, bms, blob + bytes(K * ((max(SIZES) + 7) >> 3) - len(blob)), sigs, msgs


def _capture(fn, stream=None):
    import torch
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=stream):
        out = fn()
    return g, out


@pytest.mark.parametrize("regime,K,params", REGIMES[:3], ids=[r[0] for r in REGIMES[:3]])
def test_replays_match_host_items_form(gbls, regime, K, params):
    import torch
    _, cset = _committees(gbls)
    with _Params(gbls, **params):
        index, bms, blob, sigs, msgs = _graph_inputs(gbls, K, 0)
        static = [_idx(index), _dev(blob, 1).view(-1), _dev(sigs, 96), _dev(msgs, 48)]
        g, out = _capture(lambda: cset.AggregateVerifyDevice(*static), torch.cuda.Stream())      # a stream the library has never seen
        for seed in (1, 2, 3):
            index, bms, blob, sigs, msgs = _graph_inputs(gbls, K, seed)
            static[0].copy_(torch.tensor(index, dtype=torch.int32))
            for t, b in zip(static[1:], (blob, sigs, msgs)): t.copy_(torch.frombuffer(bytearray(b), dtype=torch.uint8).view(t.shape))
            d0 = gbls.GetParam("rlc_draws")
            g.replay()
            got = _host(out)
            assert gbls.GetParam("rlc_draws") == d0 + 1                            # one draw per replay
            assert got == _items_form(gbls, index, bms, sigs, msgs), seed
            assert {0, 1, gbls.SET_BAD_INDEX} <= set(got)
        d0 = gbls.GetParam("rlc_draws")
        assert _host(_set_call(gbls, index, bms, sigs, msgs)) == got               # a direct call draws on the host
        assert gbls.GetParam("rlc_draws") == d0


def test_graph_owns_its_scratch_and_leaves_batch_info(gbls):
    import torch
    _, cset = _committees(gbls)
    s, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    with _Params(gbls, rlc_min=16):
        index, bms, blob, sigs, msgs = _graph_inputs(gbls, 600, 0)
        static = [_idx(index), _dev(blob, 1).view(-1), _dev(sigs, 96), _dev(msgs, 48)]
        g, out = _capture(lambda: cset.AggregateVerifyDevice(*static), s)
        big = _graph_inputs(gbls, 3000, 9)
        direct = [_graph_inputs(gbls, 600, 10 + i) for i in range(2)]
        tdirect = [[_idx(d[0]), _dev(d[2], 1).view(-1), _dev(d[3], 96), _dev(d[4], 48)] for d in direct]
        tbig = [_idx(big[0]), _dev(big[2], 1).view(-1), _dev(big[3], 96), _dev(big[4], 48)]
        want = _items_form(gbls, *[index, bms, sigs, msgs])
        torch.cuda.synchronize()
        for _ in range(2):
            with torch.cuda.stream(s2):
                g.replay()                                         # the graph on a second stream ...
            with torch.cuda.stream(s):                             # ... while direct calls reuse (and grow) the capture stream's arena
                outs = [cset.AggregateVerifyDevice(*tdirect[0]), cset.AggregateVerifyDevice(*tbig), cset.AggregateVerifyDevice(*tdirect[1])]
            torch.cuda.synchronize()
            assert _host(out) == want
            assert _host(outs[0]) == _items_form(gbls, direct[0][0], direct[0][1], direct[0][3], direct[0][4])
            assert _host(outs[2]) == _items_form(gbls, direct[1][0], direct[1][1], direct[1][3], direct[1][4])
            assert _host(outs[1]) == _items_form(gbls, big[0], big[1], big[3], big[4])
        # the batch info is the last direct call's: replays leave it alone
        _host(cset.AggregateVerifyDevice(*tbig))
        info = gbls.LastBatchInfo()
        assert info["rounds"] == 3000 and info["mode"] == 1
        for _ in range(2):
            g.replay(); _host(out)
        assert gbls.LastBatchInfo() == info
