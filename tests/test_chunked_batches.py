"""Batches beyond one chunk of the line buffer.  The two-kernel pairing (hbls.cu launch_verify_tail) checks W = SM count x 256 groups
per pass (rlc_chunk_groups(): 33 792 on a 132-SM H100), and the kernels index the rounds of a chunk from its first group g0.  Three
loops depend on that offset: the groups of the batched form once a batch has more than W groups, the exact pass over the rounds of the
failed groups (sized for the worst case on the host; the real list length exists only on the device), and the exact form of batch
mode 0 (launch_exact_two_phase).  Each test runs one of them over two or more chunks with invalid and irregular rounds at the chunk
seams and checks the per-round verdicts against the C oracle, and against the same batch through a form that has no chunks.

Every test takes a prefix of one signed batch of 8 (W + 5) + 3 rounds of the benchmark's workload: a prefix of a valid batch is valid,
so every round that is not injected must pass.  Knobs and the batch mode are restored whatever happens."""
import contextlib, random
import pytest
from harmony_b200 import workload as wl

pytestmark = pytest.mark.gpu

BLEN = 32                       # 250-key committee
KINDS = ("msg", "swap", "undecodable", "identity", "empty")


@pytest.fixture(scope="module")
def W():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count * 256


@pytest.fixture(scope="module")
def batch(gbls, oracle, W):
    import bench
    sks = bench.make_committee_sks()
    pks_blob = gbls.GetPublicKeyBatch(b"".join(wl.sk_bytes(k) for k in sks))
    pks = [pks_blob[48 * i:48 * i + 48] for i in range(len(sks))]
    B = 8 * (W + 5) + 3
    bitmaps, agg_sk, msgs, _ = bench.make_rounds(sks, B, seed=3131)
    sigs, ok = gbls.SignHashBatch(agg_sk, msgs, 48)
    assert ok == b"\x01" * B
    return {"com": gbls.Committee(pks), "och": oracle.committee(pks), "bitmaps": bitmaps, "agg_sk": agg_sk, "msgs": msgs, "sigs": sigs}


@contextlib.contextmanager
def knobs(gbls, mode=1, **kv):
    saved = {k: gbls.GetParam(k) for k in ("rlc_g", "rlc_block", "rlc_two_phase", "exact_two_phase")}
    saved_mode = gbls.GetBatchMode()
    try:
        gbls.SetBatchMode(mode)
        for k, v in kv.items(): gbls.SetParam(k, v)
        yield
    finally:
        for k, v in saved.items(): gbls.SetParam(k, v)
        gbls.SetBatchMode(saved_mode)


class Rounds:
    """Mutable copy of the first B rounds of the batch."""
    def __init__(self, batch, B):
        self.B = B
        self.bm = bytearray(batch["bitmaps"][:BLEN * B]); self.sg = bytearray(batch["sigs"][:96 * B]); self.ms = bytearray(batch["msgs"][:48 * B])
        self.clean_sig = batch["sigs"]
        self.bad = set()

    def inject(self, j, kind, donor=1):
        assert j not in self.bad and (kind != "swap" or donor not in self.bad)
        if kind == "msg": self.ms[48 * j + 11] ^= 0x08
        elif kind == "swap": self.sg[96 * j:96 * j + 96] = self.clean_sig[96 * donor:96 * donor + 96]     # a valid point of another round
        elif kind == "undecodable": self.sg[96 * j:96 * j + 96] = b"\xff" * 96
        elif kind == "identity": self.sg[96 * j:96 * j + 96] = bytes(96)
        elif kind == "empty": self.bm[BLEN * j:BLEN * j + BLEN] = bytes(BLEN)                     # identity aggregate key
        else: raise ValueError(kind)
        self.bad.add(j)

    def verify(self, batch):
        return batch["com"].AggregateVerifyBatch(bytes(self.bm), bytes(self.sg), bytes(self.ms), 48)

    def oracle(self, oracle, batch, j):
        return 1 if oracle.committee_aggregate_verify(batch["och"], self.bm[BLEN * j:BLEN * j + BLEN], self.sg[96 * j:96 * j + 96],
                                                      self.ms[48 * j:48 * j + 48]) == 1 else 0


def sample(B, seed, k=1000):
    return set(random.Random(seed).sample(range(B), min(k, B)))


def seam_rounds(G, ng, W, groups):
    """Every round of the given groups and of the first and last group of each chunk of W groups."""
    gs = set(groups)
    for g0 in range(0, ng, W): gs |= {g0, min(g0 + W, ng) - 1}
    return {k * ng + g for g in gs for k in range(G)}


def bad_groups(r, G, ng):
    return {j % ng for j in r.bad if j < G * ng}


def check_verdicts(oracle, batch, r, res, idx):
    """Exactly the injected rounds fail (every other round is a valid signature), and the oracle agrees on the rounds in idx."""
    assert len(res) == r.B and set(res) <= {0, 1}
    assert {j for j in range(r.B) if res[j] != 1} == r.bad and sum(res) == r.B - len(r.bad)
    wrong = [j for j in sorted(idx) if res[j] != r.oracle(oracle, batch, j)]
    assert not wrong, wrong[:20]


def check_info(gbls, r, G, ng):
    failed = bad_groups(r, G, ng)
    info = gbls.LastBatchInfo()
    assert (info["mode"], info["group_size"], info["groups"], info["tail_rounds"]) == (1, G, ng, r.B - G * ng)
    assert info["groups_failed"] == len(failed) and info["rounds_rechecked"] == G * len(failed)
    return info


def test_one_group_past_a_chunk(gbls, oracle, batch, W):
    """G = 8 and W + 1 groups: the second chunk holds one group, and blocks cannot run.  Every kind of bad round at positions 0 and 7
    of groups 0, W - 1 and W, and in the 3-round tail.  Then a wrong message in group W alone: read through a chunk offset that
    pointed at group 0 instead, it would pass."""
    G, ng = 8, W + 1
    B = G * ng + 3
    with knobs(gbls):
        clean = Rounds(batch, B)
        assert clean.verify(batch) == b"\x01" * B
        check_info(gbls, clean, G, ng)
        r = Rounds(batch, B)
        slots = [k * ng + g for g in (0, W - 1, W) for k in (0, 7)] + [G * ng, G * ng + 1, G * ng + 2]
        for i, j in enumerate(slots): r.inject(j, KINDS[i % len(KINDS)])
        res = r.verify(batch)
        check_verdicts(oracle, batch, r, res, seam_rounds(G, ng, W, bad_groups(r, G, ng)) | set(range(G * ng, B)) | sample(B, 11))
        info = check_info(gbls, r, G, ng)
        alone = Rounds(batch, B)
        alone.inject(3 * ng + W, "msg")
        check_verdicts(oracle, batch, alone, alone.verify(batch), seam_rounds(G, ng, W, {W}))
        check_info(gbls, alone, G, ng)
        gbls.SetParam("rlc_block", 1)           # forcing blocks must not make a block span two chunks
        assert r.verify(batch) == res and gbls.LastBatchInfo() == info


def test_groups_of_four_across_three_chunks(gbls, oracle, batch, W):
    """G = 4 and 2 W + 5 groups: two full chunks and one of 5 groups.  Bad rounds at groups W - 1, W, 2 W - 1, 2 W, 2 W + 4 and in the
    tail; then the same batch through the fused pairing kernel (rlc_two_phase = 0: all groups in one launch, no line buffer, and the
    exact pass through k_pairing_verify_split_list)."""
    G, ng = 4, 2 * W + 5
    B = G * ng + 3
    with knobs(gbls, rlc_g=4):
        r = Rounds(batch, B)
        for i, g in enumerate((W - 1, W, 2 * W - 1, 2 * W, 2 * W + 4)): r.inject((i * 3) % G * ng + g, KINDS[i])
        r.inject(G * ng + 2, "msg")
        res = r.verify(batch)
        check_verdicts(oracle, batch, r, res, seam_rounds(G, ng, W, bad_groups(r, G, ng)) | set(range(G * ng, B)) | sample(B, 12))
        info = check_info(gbls, r, G, ng)
        gbls.SetParam("rlc_two_phase", 0)
        assert r.verify(batch) == res
        assert gbls.LastBatchInfo()["groups_failed"] == info["groups_failed"]


def test_exact_pass_list_longer_than_a_chunk(gbls, oracle, batch, W):
    """G = 8 and W groups (one chunk for the groups).  One wrong message in each of W / 8 + 500 groups lists more than W rounds, so the
    exact pass runs over two list chunks; then position 0 of every group: all 8 W rounds listed, 8 chunks.  Both again through
    k_pairing_verify_split_list (exact_two_phase = 0)."""
    G, ng = 8, W
    B = G * ng
    rng = random.Random(13)
    with knobs(gbls):
        r1 = Rounds(batch, B)
        for g in rng.sample(range(ng), W // 8 + 500): r1.inject(rng.randrange(G) * ng + g, "msg")
        assert G * len(r1.bad) > W
        r2 = Rounds(batch, B)
        for g in range(ng): r2.inject(g, "msg")
        results = []
        for r, seed in ((r1, 14), (r2, 15)):
            res = r.verify(batch)
            check_verdicts(oracle, batch, r, res, sample(B, seed))
            results.append((res, check_info(gbls, r, G, ng)["groups_failed"]))
        gbls.SetParam("exact_two_phase", 0)
        for r, (res, gf) in zip((r1, r2), results):
            assert r.verify(batch) == res and gbls.LastBatchInfo()["groups_failed"] == gf
        assert Rounds(batch, B).verify(batch) == b"\x01" * B      # a clean batch: the next call of this size may use blocks again


def test_exact_mode_beyond_a_chunk(gbls, oracle, batch, W):
    """Batch mode 0 with W + 37 rounds: launch_exact_two_phase in two chunks (W and 37 rounds).  Bad and irregular rounds at W - 1, W,
    W + 36 and at random places; identity signatures and empty bitmaps take the k_pairing_fixup path.  Then exact_two_phase = 0."""
    B = W + 37
    rng = random.Random(17)
    with knobs(gbls, mode=0):
        r = Rounds(batch, B)
        for i, j in enumerate([W - 1, W, W + 36] + rng.sample(range(2, W - 1), 7)): r.inject(j, KINDS[i % len(KINDS)], donor=0)
        res = r.verify(batch)
        check_verdicts(oracle, batch, r, res, r.bad | set(range(W - 8, W + 9)) | set(range(B - 8, B)) | sample(B, 18))
        assert gbls.LastBatchInfo()["mode"] == 0
        gbls.SetParam("exact_two_phase", 0)
        assert r.verify(batch) == res


def test_triples_beyond_a_chunk(gbls, oracle, batch, W):
    """hbls_verify_batch_status over 8 (W + 1) + 3 independent triples (each round's aggregate key, message and signature): undecodable
    keys (ok_pk flags of listed rounds and of the tail), undecodable signatures and wrong messages at the chunk seam and in the tail.
    Group W, alone in the second chunk, holds only wrong messages, which no flag marks.  Statuses in the reference's order of errors:
    key, then signature encoding, then VerifyHash."""
    G, ng = 8, W + 1
    B = G * ng + 3
    pks = bytearray(gbls.GetPublicKeyBatch(batch["agg_sk"][:32 * B]))
    sigs = bytearray(batch["sigs"][:96 * B]); msgs = bytearray(batch["msgs"][:48 * B])
    bad = {}
    slots = [W - 1, 7 * ng + W - 1, 3 * ng + W - 1, W, 7 * ng + W, 3 * ng + 5, G * ng, G * ng + 1, G * ng + 2]
    kinds = ["key", "key+sig", "sig", "msg", "msg", "key", "key", "sig", "msg"]
    for j, kind in zip(slots, kinds):
        if "key" in kind: pks[48 * j:48 * j + 48] = b"\xff" * 48
        if "sig" in kind: sigs[96 * j:96 * j + 96] = b"\xff" * 96
        if kind == "msg": msgs[48 * j + 11] ^= 0x08
        bad[j] = {"key": 4, "key+sig": 4, "sig": 3, "msg": 0}[kind]
    with knobs(gbls):
        st = gbls.VerifyBatchStatus(bytes(pks), bytes(sigs), bytes(msgs), 48)
        assert len(st) == B and {j: st[j] for j in range(B) if st[j] != gbls.VB_OK} == bad
        failed = {j % ng for j in bad if j < G * ng}
        info = gbls.LastBatchInfo()
        assert (info["group_size"], info["groups"], info["tail_rounds"]) == (G, ng, 3)
        assert info["groups_failed"] == len(failed) and info["rounds_rechecked"] == G * len(failed)

    def want(j):
        pk, sg, m = pks[48 * j:48 * j + 48], sigs[96 * j:96 * j + 96], msgs[48 * j:48 * j + 48]
        if not oracle.pk_check(pk): return 4
        if not oracle.sig_check(sg): return 3
        return 1 if oracle.verify_hash(sg, pk, m) else 0
    idx = seam_rounds(G, ng, W, failed) | set(bad) | set(range(G * ng, B)) | sample(B, 19)
    wrong = [j for j in sorted(idx) if st[j] != want(j)]
    assert not wrong, wrong[:20]
