"""Device forms captured into CUDA graphs (include/hbls.h, "CUDA graphs"): hbls_verify_batch_status_device,
hbls_verify_headers_device and hbls_aggregate_verify_batch_device captured once with torch.cuda.graph and replayed on new inputs copied
into the static tensors give what the host forms give, in every batching regime; every replay draws its coefficients and grouping
salt on the device (rlc_draws), owns its scratch, and leaves the library's state alone; the items form refuses cleanly; and a
global-mode capture on one thread does not break the library's synchronising calls on others."""
import random, threading
import pytest
from harmony_b200 import workload as wl

pytestmark = pytest.mark.gpu


def _dev(b, width):
    import torch
    n = len(b) // width
    return torch.frombuffer(bytearray(b), dtype=torch.uint8).cuda().view(n, width)


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


# ---- inputs: a valid base set signed once, then per replay a seeded rotation with every reject class at new positions
_BASE = {}


def _triples_base(gbls, k):
    if ("tri", k) not in _BASE:
        pool = min(k, 256)
        sks = b"".join(wl.sk_bytes(wl.seeded_sk("gc-tri", i % 64)) for i in range(pool))
        msgs = b"".join(wl.seeded_bytes("gc-tri/m", i % 37, 32) for i in range(pool))
        pks = gbls.GetPublicKeyBatch(sks)
        sigs, _ = gbls.SignHashBatch(sks, msgs, 32)
        idx = [i % pool for i in range(k)]
        _BASE[("tri", k)] = (b"".join(pks[48 * i:48 * i + 48] for i in idx), b"".join(sigs[96 * i:96 * i + 96] for i in idx),
                             b"".join(msgs[32 * i:32 * i + 32] for i in idx))
    return _BASE[("tri", k)]


def _triples(gbls, k, seed):
    """k triples: the base set rotated by a seeded offset, with every reject class at seeded positions"""
    pks0, sigs0, msgs0 = _triples_base(gbls, k)
    rng = random.Random(f"gc-tri/{k}/{seed}")
    r = rng.randrange(k)
    pks = bytearray(pks0[48 * r:] + pks0[:48 * r]); sigs = bytearray(sigs0[96 * r:] + sigs0[:96 * r]); msgs = bytearray(msgs0[32 * r:] + msgs0[:32 * r])
    for t, i in enumerate(rng.sample(range(k), min(k, 10)) if k > 1 else []):
        kind = t % 5
        if kind == 0: pks[48 * i:48 * i + 48] = b"\xff" * 48                     # key does not decode
        elif kind == 1: sigs[96 * i:96 * i + 96] = b"\xff" * 96                  # signature does not decode
        elif kind == 2: msgs[32 * i + 3] ^= 0x40                                 # wrong message
        elif kind == 3: pks[48 * i:48 * i + 48] = pks[48 * ((i + 1) % k):48 * ((i + 1) % k) + 48]   # wrong key
        else: pks[48 * i:48 * i + 48] = b"\xff" * 48; sigs[96 * i:96 * i + 96] = b"\xff" * 96    # both: the key is reported
    return bytes(pks), bytes(sigs), bytes(msgs)


_N = 64                                                   # committee slots (blen 8)


def _committee(gbls):
    if "com" not in _BASE:
        sks = [wl.seeded_sk("gc-com", i) for i in range(_N)]
        blob = gbls.GetPublicKeyBatch(b"".join(wl.sk_bytes(s) for s in sks))
        _BASE["com"] = (sks, gbls.Committee([blob[48 * i:48 * i + 48] for i in range(_N)]))
    return _BASE["com"]


def _rounds_base(gbls, N):
    if ("rnd", N) not in _BASE:
        sks, _ = _committee(gbls)
        pool = min(N, 96)
        bms = [wl.bitmap_with_k("gc-rnd", j, _N, [44, 50, 60, 64][j % 4]) for j in range(pool)]
        pays = [wl.commit_payload("gc-rnd", j % 5) for j in range(pool)]
        sigs, _ = gbls.SignHashBatch(b"".join(wl.sk_bytes(wl.round_signer_sum(sks, b)) for b in bms), b"".join(pays), 48)
        idx = [j % pool for j in range(N)]
        _BASE[("rnd", N)] = (b"".join(sigs[96 * j:96 * j + 96] for j in idx), b"".join(bms[j] for j in idx), b"".join(pays[j] for j in idx))
    return _BASE[("rnd", N)]


def _rounds(gbls, N, seed):
    """N rounds against the committee: rotated by a seeded offset; wrong payload, undecodable signature, another round's signature
    and a bitmap below quorum at seeded positions"""
    sigs0, bms0, pays0 = _rounds_base(gbls, N)
    rng = random.Random(f"gc-rnd/{N}/{seed}")
    r = rng.randrange(N)
    sigs = bytearray(sigs0[96 * r:] + sigs0[:96 * r]); bms = bytearray(bms0[8 * r:] + bms0[:8 * r]); pays = bytearray(pays0[48 * r:] + pays0[:48 * r])
    for t, j in enumerate(rng.sample(range(N), min(N, 8)) if N > 1 else []):
        kind = t % 4
        if kind == 0: pays[48 * j + 12] ^= 1
        elif kind == 1: sigs[96 * j:96 * j + 96] = b"\xff" * 96
        elif kind == 2: o = (j + 1) % N; sigs[96 * j:96 * j + 96] = sigs[96 * o:96 * o + 96]
        else: bms[8 * j:8 * j + 8] = bytes([1]) + bytes(7)
    return bytes(sigs), bytes(bms), bytes(pays)


# ---- the three capturable forms: (make inputs, device call on static tensors, host form)
def _form(gbls, name, k):
    _, com = _committee(gbls) if name != "triples" else (None, None)
    q = wl.quorum_k(_N)
    if name == "triples":
        make = lambda seed: _triples(gbls, k, seed)
        widths = (48, 96, 32)
        dev = lambda t: gbls.VerifyBatchStatusDevice(t[0], t[1], t[2])
        host = lambda a: gbls.VerifyBatchStatus(a[0], a[1], a[2], 32)
    elif name == "headers":
        make = lambda seed: _rounds(gbls, k, seed)
        widths = (96, 8, 48)
        dev = lambda t: com.VerifyHeadersDevice(t[0], t[1], t[2], q)
        host = lambda a: com.VerifyHeaders(a[0], a[1], a[2], 48, q)
    else:
        make = lambda seed: _rounds(gbls, k, seed)
        widths = (96, 8, 48)
        dev = lambda t: com.AggregateVerifyBatchDevice(t[1], t[0], t[2])
        host = lambda a: com.AggregateVerifyBatch(a[1], a[0], a[2], 48)
    return make, widths, dev, host


def _capture(dev, static, stream=None):
    import torch
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=stream):
        out = dev(static)
    return g, out


def _load(static, arrays):
    import torch
    for t, a in zip(static, arrays):
        t.copy_(torch.frombuffer(bytearray(a), dtype=torch.uint8).view(t.shape))


FORMS = ["triples", "headers", "batch"]
REGIMES = [("warp", 40, {}), ("lane_pair", 64, {"coop_max": 0}), ("groups", 300, {"rlc_min": 16}), ("default_rlc", 13000, {})]


@pytest.mark.parametrize("regime,k,params", REGIMES, ids=[r[0] for r in REGIMES])
@pytest.mark.parametrize("form", FORMS)
def test_replays_match_host_form(gbls, form, regime, k, params):
    make, widths, dev, host = _form(gbls, form, k)
    with _Params(gbls, **params):
        static = [_dev(a, w) for a, w in zip(make(0), widths)]
        g, out = _capture(dev, static)
        for seed in (1, 2, 3):
            arrays = make(seed)
            _load(static, arrays)
            d0 = gbls.GetParam("rlc_draws")
            g.replay()
            got = _host(out)
            assert gbls.GetParam("rlc_draws") == d0 + 1               # one draw per replay: coefficients (when batched) and salt
            want = host(arrays)
            assert got == want, (form, regime, seed)
            assert len(set(got)) > 1
        if regime in ("groups", "default_rlc"):
            assert gbls.LastBatchInfo()["mode"] == 1                  # the host form checked the same size in batched groups


def test_direct_calls_do_not_draw_on_the_device(gbls):
    make, widths, dev, host = _form(gbls, "headers", 300)
    t = [_dev(a, w) for a, w in zip(make(4), widths)]
    with _Params(gbls, rlc_min=16):
        d0 = gbls.GetParam("rlc_draws")
        got = _host(dev(t))
        assert gbls.GetParam("rlc_draws") == d0
        assert got == host(make(4))


def test_capture_needs_no_warm_up(gbls):
    import torch
    # a stream the library has never seen
    make, widths, dev, host = _form(gbls, "triples", 500)
    static = [_dev(a, w) for a, w in zip(make(5), widths)]
    g, out = _capture(dev, static, torch.cuda.Stream())
    for seed in (6, 7):
        _load(static, make(seed)); g.replay()
        assert _host(out) == host(make(seed))
    # a capture larger than any earlier call on its stream
    s = torch.cuda.Stream()
    make_s, widths_s, dev_s, host_s = _form(gbls, "headers", 16)
    small = [_dev(a, w) for a, w in zip(make_s(1), widths_s)]
    with torch.cuda.stream(s):
        assert _host(dev_s(small)) == host_s(make_s(1))
    make_l, widths_l, dev_l, host_l = _form(gbls, "headers", 2000)
    static = [_dev(a, w) for a, w in zip(make_l(2), widths_l)]
    g, out = _capture(dev_l, static, s)
    for seed in (3, 4):
        _load(static, make_l(seed)); g.replay()
        assert _host(out) == host_l(make_l(seed))


@pytest.mark.parametrize("form", FORMS)
def test_graph_owns_its_scratch(gbls, form):
    import torch
    s, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    make, widths, dev, host = _form(gbls, form, 600)
    static = [_dev(a, w) for a, w in zip(make(0), widths)]
    g, out = _capture(dev, static, s)
    make_big, _, dev_big, host_big = _form(gbls, form, 3000)
    direct = [[_dev(a, w) for a, w in zip(make(10 + i), widths)] for i in range(2)]
    big = [_dev(a, w) for a, w in zip(make_big(12), widths)]
    torch.cuda.synchronize()
    for seed in (1, 2):
        _load(static, make(seed))
        torch.cuda.synchronize()
        with torch.cuda.stream(s2):
            g.replay()                                         # the graph on a second stream ...
        outs = []
        with torch.cuda.stream(s):                             # ... while direct calls reuse (and grow) the capture stream's arena
            outs.append(dev(direct[0])); outs.append(dev_big(big)); outs.append(dev(direct[1]))
        torch.cuda.synchronize()
        assert _host(out) == host(make(seed)), seed
        assert _host(outs[0]) == host(make(10)) and _host(outs[2]) == host(make(11))
        assert _host(outs[1]) == host_big(make_big(12))


def test_replays_leave_library_state_alone(gbls):
    make, widths, dev, host = _form(gbls, "batch", 300)
    with _Params(gbls, rlc_min=16):
        static = [_dev(a, w) for a, w in zip(make(0), widths)]
        g, out = _capture(dev, static)
        host(make(0))                                          # a direct batch call: the info replays must leave in place
        sk = gbls.SecretKey(); sk.Deserialize(wl.sk_bytes(wl.seeded_sk("gc-state", 1)))
        sk.SignHash(b"gc-state" * 4)
        before = (gbls.LastBatchInfo(), gbls.HashCacheStats(), gbls.CoalesceStats())
        for seed in (1, 2, 3):
            _load(static, make(seed)); g.replay(); _host(out)
        assert (gbls.LastBatchInfo(), gbls.HashCacheStats(), gbls.CoalesceStats()) == before


def test_items_form_refuses_capture(gbls):
    import torch
    sks, com = _committee(gbls)
    sigs, bms, pays = _rounds(gbls, 8, 0)
    ts, tb, tp = _dev(sigs, 96), _dev(bms, 8), _dev(pays, 48)
    x = torch.arange(16, dtype=torch.int32, device="cuda")
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        y = x * 3
        with pytest.raises(gbls.HblsError, match="HBLS_ERR_CAPTURE"):
            gbls.AggregateVerifyItemsDevice([com] * 8, tb, ts, tp)
        z = y + 1
    x.copy_(torch.arange(16, 32, dtype=torch.int32, device="cuda"))
    g.replay()
    torch.cuda.synchronize()
    assert z.cpu().tolist() == [3 * i + 1 for i in range(16, 32)]
    # outside a capture the same call works
    assert _host(gbls.AggregateVerifyItemsDevice([com] * 8, tb, ts, tp)) == gbls.AggregateVerifyItems([com] * 8, [bms[8 * j:8 * j + 8] for j in range(8)], sigs, pays, 48)


def test_other_threads_work_during_a_global_capture(gbls):
    import torch
    sks, com = _committee(gbls)
    sigs, bms, pays = _rounds(gbls, 8, 1)
    want_agg = com.AggregateVerifyBatch(bms, sigs, pays, 48)
    pks, tsigs, msgs = _triples(gbls, 12, 1)
    want_vb = gbls.VerifyBatchStatus(pks, tsigs, msgs, 32)
    sk = gbls.SecretKey(); sk.Deserialize(wl.sk_bytes(wl.seeded_sk("gc-thr", 0)))
    pk = sk.GetPublicKey(); h = wl.seeded_bytes("gc-thr", 0, 32)
    sig = sk.SignHash(h)
    bad_h = bytes([h[0] ^ 1]) + h[1:]
    errors, counts = [], [0, 0, 0]

    def worker(w):
        try:
            for it in range(6):
                if w == 0:
                    assert sig.VerifyHash(pk, h) and not sig.VerifyHash(pk, bad_h)
                elif w == 1:
                    assert gbls.VerifyBatchStatus(pks, tsigs, msgs, 32) == want_vb
                else:
                    j = it % 8
                    assert com.AggregateVerify(bms[8 * j:8 * j + 8], sigs[96 * j:96 * j + 96], pays[48 * j:48 * j + 48]) == bool(want_agg[j])
                counts[w] += 1
        except BaseException as e:          # noqa: BLE001 -- reported on the main thread
            errors.append((w, repr(e)))

    x = torch.arange(8, dtype=torch.float32, device="cuda")
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):                                  # capture_error_mode "global" (torch's default)
        y = x * 2
        th = [threading.Thread(target=worker, args=(w,)) for w in range(3)]
        for t in th: t.start()
        for t in th: t.join()
        z = y + 1
    g.replay()
    torch.cuda.synchronize()
    assert errors == [] and counts == [6, 6, 6], errors
    assert z.cpu().tolist() == [2 * i + 1 for i in range(8)]
