"""A leader's vote queue checked against the committee table and collected into the device ballot box in one call
(hbls_ballot_box_submit_votes, bls.BallotBox.SubmitVotes, consensus.BallotBoxCollector).

CPU: the known answers of the self-test's vote-queue leg regenerate byte for byte; the admission and fold kernels run on the host
(tests/emu/emu_ballot.cpp, under the build variants of tools/build_variants.sh) agree with a restatement of leader.go + quorum.go over
the oracle; the collector's host logic over an oracle-backed box agrees with VoteCollector over the oracle.
GPU: on 250- and 1 000-key committees the collector gives VoteCollector's errors, quorum index, ballots, bitmap and aggregate on seeded
queues with every fault the handlers distinguish; a queue of distinct members is one library call with no Part-1 request and no key
decode; argument errors; the box keeps working with add_vote."""
import ctypes, os, random, re, subprocess, sys
import pytest
from harmony_b200 import consensus as cs
from harmony_b200 import workload as wl
from test_consensus import OracleVoteBackend

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ACC, COL, BENC, BSIG = 16, 17, 18, 19                     # include/hbls.h HBLS_BALLOT_*
BAD_SIG = b"\xff" * 96                                   # x >= p: does not decode


def slots_of(bm, n):
    return {i for i in range(n) if bm[i >> 3] >> (i & 7) & 1}


def bitmap_of(slots, n):
    bm = bytearray((n + 7) >> 3)
    for i in slots: bm[i >> 3] |= 1 << (i & 7)
    return bytes(bm)


class OracleBallotBox:
    """hbls_ballot_box_* restated over the oracle: the ballot rules of leader.go:227-290 in arrival order (already collected, then
    Sign.Deserialize, then VerifyHash over the signers' key sum), AggregateVotes of quorum.go:164-196 over the accepted ballots."""
    def __init__(self, orc, och, n):
        self.o, self.h, self.n = orc, och, n
        self.collected, self.sigs, self.calls = set(), [], {"submit": 0, "add": 0}
    def SubmitVotes(self, bitmaps, sigs, msg):
        self.calls["submit"] += 1
        out = bytearray()
        for bm, sg in zip(bitmaps, sigs):
            s = slots_of(bm, self.n)
            if s & self.collected: out.append(COL)
            elif not self.o.sig_check(sg): out.append(BENC)
            elif self.o.committee_aggregate_verify(self.h, bm, sg, msg) != 1: out.append(BSIG)
            else: out.append(ACC); self.collected |= s; self.sigs.append(bytes(sg))
        return bytes(out)
    def AddVote(self, bm, sg):
        self.calls["add"] += 1
        s = slots_of(bm, self.n)
        if s & self.collected: return False
        if not self.o.sig_check(sg): raise ValueError("err blsSignatureDeserialize")
        self.collected |= s; self.sigs.append(bytes(sg))
        return True
    def Aggregate(self):
        return (self.o.aggregate_sigs(self.sigs) if self.sigs else bytes(96)), bitmap_of(self.collected, self.n)


class OracleBoxBackend(OracleVoteBackend):
    def ballot_box(self, com): return OracleBallotBox(self.o, com["h"], len(com["pks"]))


# ------------------------------------------------------------------ seeded queues
class Signer:
    def __init__(self, orc, n, tag, message, extra=3):
        self.o, self.n, self.message = orc, n, message
        self.sks = [wl.seeded_sk(tag, i) for i in range(n + extra)]
        self.cache = {}
    def pks(self, pk_of):
        self.pk = pk_of(self.sks); self.members = self.pk[:self.n]; self.outsiders = self.pk[self.n:]
        return self.members
    def sign(self, idx, msg=None):
        key = (tuple(idx), msg)
        if key not in self.cache:
            self.cache[key] = self.o.sign_hash(wl.sk_bytes(sum(self.sks[i] for i in idx) % wl.R_ORDER), msg or self.message)
        return self.cache[key]
    def vote(self, idx, sig_idx=None):
        return cs.Vote([self.pk[i] for i in idx], self.sign(sig_idx if sig_idx is not None else idx))


def random_queue(sg, rng, n_votes, faults=True):
    """one-key and multi-key votes over a pool of members (signers repeat within and across queues); with faults: undecodable,
    wrong and someone else's signatures, short payloads, repeated keys, non-member keys, an empty key list"""
    n = sg.n; votes = []
    for _ in range(n_votes):
        r = rng.randrange(20) if faults else 0
        idx = rng.sample(range(n), 1 if rng.randrange(3) else rng.randrange(2, 5))
        if r == 1: v = sg.vote(idx); v.Payload = BAD_SIG
        elif r == 2: v = sg.vote(idx, [(idx[0] + 1) % n])                              # someone else's signature
        elif r == 3: v = sg.vote(idx); v.Payload = sg.sign(idx, wl.commit_payload("vq/other", 0))     # another message
        elif r == 4: v = sg.vote(idx); v.Payload = v.Payload[:95]
        elif r == 5: v = sg.vote([idx[0], idx[0]], [idx[0], idx[0]])                   # repeated key
        elif r == 6: o = n + rng.randrange(len(sg.outsiders)); v = sg.vote(idx[:1] + [o] if rng.randrange(2) else [o])      # non-member
        elif r == 7: v = cs.Vote([], sg.sign(idx))
        else: v = sg.vote(idx)
        votes.append(v)
    return votes


def compare_ticks(col, ref, ticks):
    """every tick: the same errors and quorum index; at the end the same ballots and the same AggregateVotes bytes"""
    for votes in ticks:
        assert col.onVotes(votes) == ref.onVotes(votes)
        assert col.SignersCount() == ref.SignersCount() and col.IsQuorumAchieved() == ref.IsQuorumAchieved()
    assert col.BallotBox == ref.BallotBox
    assert col.AggregateVotes() == ref.AggregateVotes()


def cut(rng, votes):
    out, pos = [], 0
    while pos < len(votes):
        step = rng.randrange(1, 9); out.append(votes[pos:pos + step]); pos += step
    return out


# ------------------------------------------------------------------ CPU
def test_vote_queue_kat_header_regenerates_byte_for_byte():
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "gen_selftest_votes.py"), "--check"], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0 and "up to date" in r.stdout, r.stdout + r.stderr


def test_collector_host_logic_matches_vote_collector(oracle):
    """BallotBoxCollector over an oracle-backed box == VoteCollector over the oracle, on queues in one tick and cut into many; a queue
    of distinct members is one box call and nothing else."""
    n = 18; message = wl.commit_payload("vq/host", 0)
    sg = Signer(oracle, n, "vq/host", message)
    members = sg.pks(lambda ks: [oracle.get_public_key(wl.sk_bytes(k)) for k in ks])
    for seed in range(6):
        rng = random.Random(seed)
        votes = random_queue(sg, rng, 30)
        ticks = [votes] if seed % 2 == 0 else cut(rng, votes)
        be = OracleBoxBackend(oracle)
        col = cs.BallotBoxCollector(members, message, backend=be)
        compare_ticks(col, cs.VoteCollector(members, message, backend=OracleVoteBackend(oracle)), ticks + [random_queue(sg, rng, 10)])
    # honest queue: one box call, no key sum, no status triple
    be = OracleBoxBackend(oracle)
    col = cs.BallotBoxCollector(members, message, backend=be)
    honest = [sg.vote([i]) for i in range(8)] + [sg.vote([8, 9, 10]), sg.vote([3]), sg.vote([11, 12])]
    be.aggregate_keys = be.verify_status = lambda *a: pytest.fail("the queue left the box path")
    errs, q = col.onVotes(honest)
    assert errs == [None] * 9 + [cs.errAlreadyReceived, None]
    assert col.box.calls == {"submit": 1, "add": 0}
    assert q == 10 and col.SignersCount() == 13 == col.quorum


def test_cpp_collector_matches_cpp_vote_collector(oracle, tmp_path):
    """The C++ consensus::BallotBoxCollector == consensus::VoteCollector (harmony_b200/host/hbls_consensus.hpp), both over the CPU
    oracle standing in for libhbls.so (tests/host/oracle_abi.cpp): seeded queues with every fault, one tick or many, and an honest
    queue that is one box call with no key decoded."""
    from harmony_b200 import build
    orc = build.build_oracle()
    exe = str(tmp_path / "vote_collectors")
    host = os.path.join(ROOT, "tests", "host")
    subprocess.check_call(["g++", "-O1", "-std=c++17", "-Wall", "-o", exe, os.path.join(host, "vote_collectors.cpp"), os.path.join(host, "oracle_abi.cpp"),
                           orc, "-Wl,-rpath," + os.path.dirname(orc), "-pthread"])
    r = subprocess.run([exe], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0 and "all checks passed" in r.stdout, r.stdout + r.stderr


@pytest.fixture(scope="module", params=["default", "noinv", "batchinv4", "chunks"])
def emub(request):
    """emu_ballot.cpp built like the library variants of tools/build_variants.sh (default = batchinv8); "chunks" shrinks the
    admission kernel's shared-memory box and staging area (128 / 256 bytes) so that queues are staged in chunks of 2 to 128 votes"""
    variant = request.param
    src = os.path.join(ROOT, "tests", "emu", "emu_ballot.cpp")
    out = os.path.join(ROOT, "tests", "emu", "libhbls_emu_ballot.so" if variant == "default" else f"libhbls_emu_ballot_{variant}.so")
    csrc = os.path.join(ROOT, "harmony_b200", "csrc")
    deps = [src, os.path.join(ROOT, "tests", "emu", "emu_kernels.cpp")] + [os.path.join(csrc, f) for f in os.listdir(csrc) if f.endswith(".cuh")]
    if not os.path.exists(out) or any(os.path.getmtime(d) > os.path.getmtime(out) for d in deps):
        flags = {"default": [], "noinv": ["-DHB_BATCH_INV=0"], "batchinv4": ["-DHB_BATCH_INV=1", "-DHB_BATCH_K=4"],
                 "chunks": ["-DHB_BALLOT_MAX_BYTES=128", "-DHB_BALLOT_STAGE=256"]}[variant]
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-pthread"] + flags + ["-o", out, src])
    L = ctypes.CDLL(out)
    L.emu_ballot_submit.argtypes = [ctypes.c_uint32, ctypes.c_char_p, ctypes.c_size_t, ctypes.c_char_p, ctypes.c_size_t, ctypes.c_char_p,
                                    ctypes.c_char_p, ctypes.c_uint32, ctypes.c_char_p, ctypes.c_char_p, ctypes.c_char_p, ctypes.c_char_p]
    L.emu_g2_jac_bytes.restype = ctypes.c_size_t
    return L


class EmuBox:
    def __init__(self, L, pks):
        self.L, self.pks, self.n = L, pks, len(pks)
        self.col = ctypes.create_string_buffer((self.n + 7) >> 3)
        self.sum = ctypes.create_string_buffer(L.emu_g2_jac_bytes())
    def submit(self, bms, sigs, msg):
        k = len(sigs); st = ctypes.create_string_buffer(k or 1); s96 = ctypes.create_string_buffer(96)
        rc = self.L.emu_ballot_submit(self.n, b"".join(self.pks), k, b"".join(bms), len(self.col), b"".join(sigs), msg, len(msg),
                                      self.col, self.sum, st, s96)
        assert rc == 0, rc
        return st.raw[:k], s96.raw, self.col.raw


_COMMITTEES = {}
def committee(oracle, n):
    if n not in _COMMITTEES:
        sks = [wl.seeded_sk("vq/emu", i) for i in range(n)]
        _COMMITTEES[n] = (sks, [oracle.get_public_key(wl.sk_bytes(k)) for k in sks], oracle.committee([oracle.get_public_key(wl.sk_bytes(k)) for k in sks]))
    return _COMMITTEES[n]


@pytest.mark.parametrize("n", [16, 250, 1000])
def test_emulated_admission_and_fold_match_restatement(emub, oracle, n):
    """Two ticks into one box.  Tick 1 opens with a signer already in the box and ends with an accepted vote in the last slot, and holds a
    multi-key vote, a repeated signer, an undecodable, a wrong and an empty-bitmap vote; tick 2 repeats signers of tick 1 only: every
    vote is already collected, even the undecodable one."""
    sks, pks, och = committee(oracle, n)
    msg = wl.commit_payload("vq/emu", n)
    rng = random.Random(n)
    sign = lambda idx, m=msg: oracle.sign_hash(wl.sk_bytes(sum(sks[i] for i in idx) % wl.R_ORDER), m)
    a, b, c, d, e, f = rng.sample(range(n - 1), 6)
    ref = OracleBallotBox(oracle, och, n); box = EmuBox(emub, pks)
    pre = [bitmap_of([a], n)], [sign([a])]
    assert ref.SubmitVotes(*pre, msg) == bytes([ACC]) and box.submit(*pre, msg)[0] == bytes([ACC])
    tick1 = [([a], sign([a])), ([b, c], sign([b, c])), ([c], sign([c])), ([d], BAD_SIG), ([e], sign([f])), ([], sign([d])),
             ([d], sign([d]), ), ([e, f], sign([e, f], wl.commit_payload("vq/emu", n + 1))), ([n - 1], sign([n - 1]))]
    tick2 = [([b], sign([b])), ([c, d], sign([c, d])), ([n - 1], BAD_SIG), ([a, e], sign([a, e]))]
    for tick in (tick1, tick2):
        bms = [bitmap_of(s, n) for s, _ in tick]; sigs = [g for _, g in tick]
        want = ref.SubmitVotes(bms, sigs, msg)
        got, agg, col = box.submit(bms, sigs, msg)
        assert got == want and (agg, col) == ref.Aggregate()
    assert list(want) == [COL] * 4


# ------------------------------------------------------------------ GPU
def _gpu_signer(gbls, oracle, n, tag, message):
    sg = Signer(oracle, n, tag, message)
    def pk_of(ks):
        blob = gbls.GetPublicKeyBatch(b"".join(wl.sk_bytes(k) for k in ks)); return [blob[48 * i:48 * i + 48] for i in range(len(ks))]
    return sg, sg.pks(pk_of)


@pytest.mark.gpu
@pytest.mark.parametrize("n", [250, 1000])
def test_collector_matches_vote_collector_on_device(gbls, oracle, n):
    message = wl.commit_payload("vq/gpu", n)
    sg, members = _gpu_signer(gbls, oracle, n, "vq/gpu", message)
    for seed in range(3):
        rng = random.Random(1000 * n + seed)
        votes = random_queue(sg, rng, n // 3)
        ticks = [votes] if seed == 0 else cut(rng, votes)
        ticks.append(random_queue(sg, rng, n // 2, faults=seed != 2))        # signers repeated across ticks; quorum reached here
        col = cs.BallotBoxCollector(members, message)
        ref = cs.VoteCollector(members, message, backend=OracleVoteBackend(oracle))
        compare_ticks(col, ref, ticks)
        sig, bm = col.AggregateVotes()
        if not col.unbitted:                                                    # no non-member ballot: the payload verifies
            assert gbls.Committee(members).AggregateVerify(bm, sig, message)


@pytest.mark.gpu
def test_box_submit_matches_restatement_and_keeps_add_vote(gbls, oracle):
    """SubmitVotes statuses over two ticks (empty bitmaps, undecodable / wrong signatures, signers repeated within and across ticks),
    then add_vote on the same box, against the restatement; the bitmap and the aggregate after each step."""
    for n in (250, 1000):
        message = wl.commit_payload("vq/box", n)
        sg, members = _gpu_signer(gbls, oracle, n, "vq/box", message)
        com = gbls.Committee(members); box = gbls.BallotBox(com)
        ref = OracleBallotBox(oracle, oracle.committee(members), n)
        rng = random.Random(n)
        for tick in range(2):
            bms, sigs = [], []
            for j in range(40):
                idx = rng.sample(range(n), rng.choice((1, 1, 2, 4)))
                r = rng.randrange(8)
                bms.append(bitmap_of([] if r == 0 else idx, n))
                sigs.append(BAD_SIG if r == 1 else sg.sign([(idx[0] + 1) % n]) if r == 2 else sg.sign(idx))
            got = box.SubmitVotes(bms, sigs, message)
            assert got == ref.SubmitVotes(bms, sigs, message)
            assert box.Aggregate() == ref.Aggregate()
            assert {ACC, COL, BENC, BSIG} <= set(got)
        free = sorted(set(range(n)) - ref.collected)[:2]
        for idx in ([free[0]], [free[0], free[1]], [free[1]]):
            assert box.AddVote(bitmap_of(idx, n), sg.sign(idx)) == ref.AddVote(bitmap_of(idx, n), sg.sign(idx))
        assert box.Aggregate() == ref.Aggregate()
        assert box.SubmitVotes([], [], message) == b""


@pytest.mark.gpu
def test_distinct_member_queue_is_one_call_without_key_decode(gbls, oracle):
    import torch
    from torch.profiler import profile, ProfilerActivity
    n = 250; message = wl.commit_payload("vq/one", 0)
    sg, members = _gpu_signer(gbls, oracle, n, "vq/one", message)
    col = cs.BallotBoxCollector(members, message)
    calls = {"submit": 0}
    real = col.box.SubmitVotes
    def counted(*a):
        calls["submit"] += 1; return real(*a)
    col.box.SubmitVotes = counted
    for name in ("aggregate_keys", "verify_status", "verify_headers", "aggregate_sigs"):
        setattr(col.be, name, lambda *a, _n=name: pytest.fail(f"{_n} called"))
    names = ("rlc_min", "rlc_g", "coop_max", "overlap", "hm_cache", "hash_split", "mask_sort", "rlc_block")
    params = {k: gbls.GetParam(k) for k in names}; mode = gbls.GetBatchMode()
    q1 = [sg.vote([i]) for i in range(50)] + [sg.vote([50 + 4 * j + t for t in range(4)]) for j in range(25)]       # 50 one-key, 25 four-key
    c0 = gbls.CoalesceStats()
    assert col.onVotes(q1) == ([None] * 75, None) and calls["submit"] == 1
    # the second queue: H(m) is cached now; its launches are those of the same-message verification of as many rounds, plus two
    q2 = [sg.vote([150 + i]) for i in range(75)]
    bms = [bitmap_of([150 + i], n) for i in range(75)]
    com = gbls.Committee(members)
    l0 = gbls.KernelLaunchCount()
    com.AggregateVerifyBatch(b"".join(bms), b"".join(v.Payload for v in q2), message * 75, len(message))
    verify_launches = gbls.KernelLaunchCount() - l0
    l0 = gbls.KernelLaunchCount()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        errs, q = col.onVotes(q2)
        torch.cuda.synchronize()
    assert gbls.KernelLaunchCount() - l0 == verify_launches + 2
    assert errs == [None] * 75 and q == 16 and calls["submit"] == 2
    assert gbls.CoalesceStats()["requests"] == c0["requests"]                 # no Part-1 Deserialize / Add
    kern = [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
    assert any("k_ballot_admit" in k for k in kern) and any("k_ballot_fold" in k for k in kern), kern
    assert not any("k_g1_decode" in k for k in kern), kern
    assert sum(1 for k in kern if re.search(r"k_g2_decode(_pair)?\b", k)) == 1, kern
    assert {k: gbls.GetParam(k) for k in names} == params and gbls.GetBatchMode() == mode
    assert gbls.LastBatchInfo()["rounds"] == 75


@pytest.mark.gpu
def test_submit_votes_argument_errors(gbls):
    L = gbls.lib(); c = ctypes
    members = [gbls.GetPublicKeyBatch(wl.sk_bytes(wl.seeded_sk("vq/arg", i)))[:48] for i in range(10)]
    com = gbls.Committee(members); box = gbls.BallotBox(com)
    st = c.create_string_buffer(4); bm = bytes(2); sig = bytes(96); m = b"m" * 32
    assert L.hbls_ballot_box_submit_votes(None, 1, bm, 2, sig, m, 32, st) == gbls.ERR_ARG
    assert L.hbls_ballot_box_submit_votes(box.h, 1, bm, 2, sig, m, 32, None) == gbls.ERR_ARG
    assert L.hbls_ballot_box_submit_votes(box.h, 1, bytes(3), 3, sig, m, 32, st) == gbls.ERR_ARG
    assert L.hbls_ballot_box_submit_votes(box.h, 1, bm, 2, sig, b"m" * 65, 65, st) == gbls.ERR_ARG
    assert L.hbls_ballot_box_submit_votes(box.h, 0, bm, 2, sig, m, 32, st) == 0
    with pytest.raises(ValueError): box.SubmitVotes([bm], [sig, sig], m)


# every form of the verification pipeline feeds the admission and the fold: {knobs}, queue length.  Up to coop_max votes the exact
# check runs a warp per vote with lane-pair decode (the other tests); past it the signatures go through k_g2_decode + k_g2_subgroup and
# the exact check through the line / accumulator kernels or the lane-pair kernel; from rlc_min on through the batched groups (failed
# groups re-verified exactly); from 256 votes per SM on the keys are summed one vote per thread (k_mask_aggregate_serial)
_FORMS = {"exact_two_kernel": ({"coop_max": 0}, 150),
          "exact_lane_pair": ({"coop_max": 0, "exact_two_phase": 0}, 150),
          "rlc_groups": ({"rlc_min": 16}, 150),
          "mask_serial_rlc": ({}, 34000)}


@pytest.mark.gpu
@pytest.mark.parametrize("form", sorted(_FORMS))
def test_box_submit_through_every_verify_form(gbls, oracle, form):
    knobs, B = _FORMS[form]
    n = 250; message = wl.commit_payload("vq/forms", 0)
    sg, members = _gpu_signer(gbls, oracle, n, "vq/forms", message)
    rng = random.Random(len(form))
    base = []                                             # 80 distinct votes of every kind; the queue repeats them up to B votes
    for j in range(80):
        idx = rng.sample(range(n), rng.choice((1, 1, 2, 4)))
        r = rng.randrange(8)
        base.append((bitmap_of([] if r == 0 else idx, n), BAD_SIG if r == 1 else sg.sign([(idx[0] + 1) % n]) if r == 2 else sg.sign(idx)))
    queue = base + [base[rng.randrange(len(base))] for _ in range(B - len(base))]
    rng.shuffle(queue)
    # the restatement, with the oracle's verdict on each distinct vote computed once
    och = oracle.committee(members); verdict = {}; collected = 0; want = bytearray(); acc = []
    for bm, sig in queue:
        bits = int.from_bytes(bm, "little")
        if bits & collected: want.append(COL); continue
        if (bm, sig) not in verdict:
            verdict[(bm, sig)] = BENC if not oracle.sig_check(sig) else ACC if oracle.committee_aggregate_verify(och, bm, sig, message) == 1 else BSIG
        v = verdict[(bm, sig)]; want.append(v)
        if v == ACC: collected |= bits; acc.append(sig)
    assert {ACC, COL, BENC, BSIG} <= set(want)
    old = {k: gbls.GetParam(k) for k in knobs}
    try:
        for k, v in knobs.items(): gbls.SetParam(k, v)
        box = gbls.BallotBox(gbls.Committee(members))
        got = box.SubmitVotes([bm for bm, _ in queue], [s for _, s in queue], message)
        info = gbls.LastBatchInfo()
    finally:
        for k, v in old.items(): gbls.SetParam(k, v)
    assert got == bytes(want)
    assert box.Aggregate() == (oracle.aggregate_sigs(acc), collected.to_bytes((n + 7) >> 3, "little"))
    assert info["rounds"] == B and info["mode"] == (1 if form in ("rlc_groups", "mask_serial_rlc") else 0)
