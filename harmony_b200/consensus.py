"""harmony_b200/consensus.py -- the signature checks of Harmony's FBFT message handlers, batched (SURVEY.md 8f rank 3 and the
callers behind BASELINE configs[3], the view-change storm).

Host mirror of
  * consensus/consensus_service.go:115-133 signMessage / signConsensusMessage and consensus/checks.go:20-56 verifyMessageSig /
    senderKeySanityChecks (keccak256 of the marshalled message, SignHash / VerifyHash),
  * consensus/view_change_msg.go:139-190 ParseViewChangeMessage (what must decode), consensus/checks.go:139-193
    onViewChangeSanityCheck (the viewID signature), consensus/view_change_construct.go:237-375 ProcessViewChangeMsg,
    :122-151 GetM2Bitmap / GetM3Bitmap, :154-234 VerifyNewViewMsg and consensus/view_change.go:445-500 onNewView.

The reference runs these checks one cgo call at a time under consensus.mutex: a new leader that receives N VIEWCHANGE messages
pays 2 N VerifyHash + up to N (SetMask + VerifyHash) calls.  Here the cryptographic booleans of a whole batch of messages come
from TWO device calls (hbls_verify_batch_status over the 2 N independent triples, hbls_verify_headers over the embedded PREPARED
proofs) and the reference's stateful bookkeeping (duplicate checks, bitmaps, first M1 payload) then runs over them in arrival
order, so every message gets exactly the error the sequential code would have returned.

Messages of different lengths share a batch: the hash-to-G2 map reads min(len, 48) bytes as a little-endian integer (SURVEY
A.3), so the 1-byte NIL, the 8-byte viewID and a >= 128-byte M1 payload are zero-padded / cut to 48 bytes without changing H(m).

Out of scope (callers' business, passed in as callbacks or bytes): protobuf marshalling, RLP decoding and block verification.
"""
from dataclasses import dataclass
from typing import Callable, List, Optional
from . import bls

NIL = b"\x01"                                                   # consensus/config.go:49-52
ValidPayloadLength = 32 + bls.BLSSignatureSizeInBytes           # consensus/view_change_construct.go:25-26

# error values, spelled as in the reference
errDupM1 = "received M1 (prepared) message already"             # view_change_construct.go:225-234
errDupM2 = "received M2 (NIL) message already"
errDupM3 = "received M3 (ViewID) message already"
errVerifyM1 = "failed to verfiy signature for M1 message"
errVerifyM2 = "failed to verfiy signature for M2 message"
errM1Payload = "failed to verify multi signature for M1 prepared payload"
errNoQuorum = "no quorum on M1 (prepared) payload"
errViewIDSig = "[onViewChangeSanityCheck] Failed to Verify viewID Signature"        # checks.go:186-191
errSigDeserialize = "err blsSignatureDeserialize"                # herumi's Go wrapper, Sign.Deserialize
errKeyDeserialize = "err blsPublicKeyDeserialize"                # crypto/bls/mask.go:35-55 BytesToBLSPublicKey
errMsgSig = "failed to verify the signature"                    # checks.go:35
errMultiSigDeserialize = "unable to deserialize multi-signature from payload"       # internal/chain/sig.go:42
errSetMask = "mask.SetMask failed"                              # internal/chain/sig.go:47
errM3Nil = "[VerifyNewViewMsg] M3AggSig or M3Bitmap is nil"
errM3Verify = "[VerifyNewViewMsg] Unable to Verify Aggregated Signature of M3 (ViewID) payload"
errM2Verify = "[VerifyNewViewMsg] Unable to Verify Aggregated Signature of M2 (NIL) payload"
errNewViewQuorum = "[onNewView] Quorum Not achieved"
errNewViewM1 = "[onNewView] Failed to Verify Signature for M1 (prepare) message"
errPayloadLength = "payload not have enough length"              # consensus_service.go:313-315, sig.go:23-25
errAlreadyReceived = "already received message from the validator"          # leader.go:127-136,233-241 (logged, message dropped)
errVoteSig = "received invalid BLS signature"                                # leader.go:171-180,287-290
errDuplicateKey = "duplicate key found in votes"                              # quorum.go:361-363
errAlreadySubmitted = "vote is already submitted"                             # quorum.go:366-368
errKeyNotFound = "key not found"                                              # crypto/bls/mask.go:226-233 SetKeysAtomic

# ------------------------------------------------------------------ crypto/hash/hash.go:9-17 (sha3.NewLegacyKeccak256)
_RC = [0x0000000000000001, 0x0000000000008082, 0x800000000000808A, 0x8000000080008000, 0x000000000000808B, 0x0000000080000001,
       0x8000000080008081, 0x8000000000008009, 0x000000000000008A, 0x0000000000000088, 0x0000000080008009, 0x000000008000000A,
       0x000000008000808B, 0x800000000000008B, 0x8000000000008089, 0x8000000000008003, 0x8000000000008002, 0x8000000000000080,
       0x000000000000800A, 0x800000008000000A, 0x8000000080008081, 0x8000000000008080, 0x0000000080000001, 0x8000000080008008]
_ROT = [[0, 36, 3, 41, 18], [1, 44, 10, 45, 2], [62, 6, 43, 15, 61], [28, 55, 25, 21, 56], [27, 20, 39, 8, 14]]
_M64 = (1 << 64) - 1

def _keccak_f(a):
    rol = lambda v, n: ((v << n) | (v >> (64 - n))) & _M64 if n else v
    for rc in _RC:
        c = [a[x][0] ^ a[x][1] ^ a[x][2] ^ a[x][3] ^ a[x][4] for x in range(5)]
        d = [c[(x - 1) % 5] ^ rol(c[(x + 1) % 5], 1) for x in range(5)]
        a = [[a[x][y] ^ d[x] for y in range(5)] for x in range(5)]
        b = [[0] * 5 for _ in range(5)]
        for x in range(5):
            for y in range(5):
                b[y][(2 * x + 3 * y) % 5] = rol(a[x][y], _ROT[x][y])
        a = [[b[x][y] ^ (~b[(x + 1) % 5][y] & b[(x + 2) % 5][y]) for y in range(5)] for x in range(5)]
        a[0][0] ^= rc
    return a

def Keccak256(*data) -> bytes:
    """Legacy Keccak-256 (multi-rate padding 0x01 .. 0x80, rate 136), as golang.org/x/crypto/sha3.NewLegacyKeccak256."""
    rate = 136
    p = bytearray(b"".join(bytes(d) for d in data))
    p.append(0x01)
    while len(p) % rate: p.append(0)
    p[-1] |= 0x80
    a = [[0] * 5 for _ in range(5)]
    for off in range(0, len(p), rate):
        for i in range(rate // 8):
            a[i % 5][i // 5] ^= int.from_bytes(p[off + 8 * i:off + 8 * i + 8], "little")
        a = _keccak_f(a)
    return b"".join(a[i % 5][i // 5].to_bytes(8, "little") for i in range(4))

# ------------------------------------------------------------------ the device calls behind the checks (one per method)
def _m48(m: bytes) -> bytes:
    """what hash-to-G2 reads of a message (SURVEY A.3): its first 48 bytes as a little-endian integer == zero-padded to 48."""
    return bytes(m[:48]).ljust(48, b"\x00")

class DeviceBackend:
    """The product path: every method is ONE call into libhbls.so (no CPU fallback -- bls raises without a GPU)."""
    def committee(self, pks48): return bls.Committee(pks48)
    def verify_status(self, pks48, sigs96, msgs) -> bytes:
        return bls.VerifyBatchStatus(b"".join(pks48), b"".join(sigs96), b"".join(_m48(m) for m in msgs), 48)
    def verify_headers(self, com, sigs96, bitmaps, msgs, quorum) -> bytes:
        return com.VerifyHeaders(b"".join(sigs96), b"".join(bitmaps), b"".join(_m48(m) for m in msgs), 48, quorum)
    def aggregate_sigs(self, sigs96) -> bytes: return bls.AggregateSigBytes(sigs96)
    def aggregate_keys(self, pks48) -> bytes:
        """sum of a multi-key vote's sender keys (consensus/leader.go:161-169): PublicKey.Add over the LRU-decoded keys"""
        acc = bls.PublicKey()
        for k in pks48: acc.Add(bls.BytesToBLSPublicKey(k))          # ValueError when a key does not decode
        return acc.Serialize()

def _le64(v: int) -> bytes: return int(v).to_bytes(8, "little")
def _popcount_slots(bitmap: bytes, n: int) -> int:
    return sum(1 for i in range(n) if bitmap[i >> 3] & (1 << (i & 7)))

# ------------------------------------------------------------------ consensus message signatures
def signMessage(message: bytes, priKey: "bls.SecretKey") -> bytes:
    """consensus/consensus_service.go:115-119: SignHash(keccak256(message)).Serialize()."""
    sig = priKey.SignHash(Keccak256(message))
    return sig.Serialize()

def verifyMessageSig(signerPubKey: "bls.PublicKey", message: bytes, signature: bytes) -> Optional[str]:
    """consensus/checks.go:20-39 on the marshalled message (Signature field cleared by the caller): None or the error."""
    msgSig = bls.Sign()
    try: msgSig.Deserialize(signature)
    except ValueError: return errSigDeserialize
    if not msgSig.VerifyHash(signerPubKey, Keccak256(message)): return errMsgSig
    return None

def verifyMessageSigBatch(senderKeys48: List[bytes], messages: List[bytes], signatures: List[bytes], backend=None) -> List[Optional[str]]:
    """senderKeySanityChecks (consensus/checks.go:41-56) for a queue of received messages in ONE device call: per message None,
    or the error BytesToBLSPublicKey / Sign.Deserialize / VerifyHash would have produced, in that order."""
    be = backend or DeviceBackend()
    n = len(messages)
    if n == 0: return []
    well = [len(senderKeys48[i]) == 48 and len(signatures[i]) == 96 for i in range(n)]
    st = be.verify_status([senderKeys48[i] if well[i] else bytes(48) for i in range(n)],
                          [signatures[i] if well[i] else bytes(96) for i in range(n)],
                          [Keccak256(m) for m in messages])
    out = []
    for i in range(n):
        if len(senderKeys48[i]) != 48 or st[i] == bls.VB_BAD_KEY_ENCODING: out.append(errKeyDeserialize)
        elif len(signatures[i]) != 96 or st[i] == bls.VB_BAD_SIG_ENCODING: out.append(errSigDeserialize)
        else: out.append(None if st[i] == bls.VB_OK else errMsgSig)
    return out

# ------------------------------------------------------------------ view change
@dataclass
class FBFTMessage:
    """The fields of consensus/fbft_log.go FBFTMessage the view-change checks read; signatures and keys as wire bytes."""
    ViewID: int
    BlockNum: int
    SenderPubkey: bytes                      # 48 bytes; VIEWCHANGE / NEWVIEW carry a single sender (HasSingleSender)
    LeaderPubkey: bytes = b""
    Payload: bytes = b""                     # M1: blockHash32 || preparedAggSig96 || preparedBitmap ; empty otherwise
    Block: bytes = b""                       # RLP of the prepared block (opaque here)
    ViewchangeSig: bytes = b""               # over Payload (M1) or NIL (M2)
    ViewidSig: bytes = b""                   # over LE64(ViewID) (M3)
    M2AggSig: Optional[bytes] = None
    M2Bitmap: Optional[bytes] = None
    M3AggSig: Optional[bytes] = None
    M3Bitmap: Optional[bytes] = None

class viewChange:
    """consensus/view_change_construct.go:31-51: the new leader's collection of M1 / M2 / M3 signatures, device-backed."""
    def __init__(self, members: List[bytes], backend=None, verifyBlock: Optional[Callable[[bytes], Optional[str]]] = None,
                 isQuorumAchievedByMask: Optional[Callable[[bytes], bool]] = None):
        self.members = [bytes(m) for m in members]
        self.index = {m: i for i, m in enumerate(self.members)}
        self.be = backend or DeviceBackend()
        self.com = self.be.committee(self.members)
        self.blen = (len(self.members) + 7) >> 3
        self.verifyBlock = verifyBlock or (lambda block: None)
        # uniform vote by default (consensus/quorum/one-node-one-vote.go:57-72); a staked-vote decider passes its own predicate
        self.isQuorum = isQuorumAchievedByMask
        self.quorum = 2 * len(self.members) // 3 + 1
        self.Reset()
    def Reset(self):                         # view_change_construct.go:85-95
        self.bhpSigs, self.nilSigs, self.viewIDSigs = {}, {}, {}
        self.bhpBitmap, self.nilBitmap, self.viewIDBitmap = {}, {}, {}
        self.newViewMsg = {}
        self.m1Payload = b""
    def IsM1PayloadEmpty(self) -> bool: return len(self.m1Payload) == 0
    def GetM1Payload(self) -> bytes: return self.m1Payload
    def _set_key(self, table, viewID, pk48):               # Mask.SetKey(key, true); "key not found" is ignored like the caller does
        bm = table.setdefault(viewID, bytearray(self.blen))
        i = self.index.get(bytes(pk48))
        if i is not None: bm[i >> 3] |= 1 << (i & 7)

    # ---- the storm: n VIEWCHANGE messages, two device calls
    def ProcessViewChangeMsgs(self, msgs: List[FBFTMessage]) -> List[Optional[str]]:
        """onViewChangeSanityCheck's signature check + ProcessViewChangeMsg for every message, in arrival order.
        Returns None (accepted) or the error per message; the state afterwards equals that of the sequential reference."""
        n = len(msgs)
        if n == 0: return []
        is_m1 = [len(m.Payload) >= ValidPayloadLength and len(m.Block) != 0 for m in msgs]
        well = [len(m.SenderPubkey) == 48 and len(m.ViewchangeSig) == 96 and len(m.ViewidSig) == 96 for m in msgs]
        # call 1: 2 n independent triples -- (sender, Payload | NIL, ViewchangeSig) and (sender, LE64(ViewID), ViewidSig)
        pks, sigs, ms = [], [], []
        for m, w, m1 in zip(msgs, well, is_m1):
            pk = m.SenderPubkey if w else bytes(48)
            pks += [pk, pk]
            sigs += [m.ViewchangeSig if w else bytes(96), m.ViewidSig if w else bytes(96)]
            ms += [m.Payload if m1 else NIL, _le64(m.ViewID)]
        st = self.be.verify_status(pks, sigs, ms)
        # call 2: the PREPARED proof inside every M1 payload: Deserialize ; SetMask ; quorum ; aggSig.VerifyHash(apk, blockHash)
        m1_idx = [i for i in range(n) if is_m1[i]]
        hdr = {}
        if m1_idx:
            hs, hb, hp, short = [], [], [], {}
            for i in m1_idx:
                body = msgs[i].Payload[32:]
                bm = body[96:]
                short[i] = len(bm) != self.blen          # mask.SetMask: "mismatching bitmap lengths" (crypto/bls/mask.go:114-120)
                hs.append(body[:96]); hb.append(bytes(self.blen) if short[i] else bytes(bm)); hp.append(msgs[i].Payload[:32])
            res = self.be.verify_headers(self.com, hs, hb, hp, 0 if self.isQuorum else self.quorum)
            for k, i in enumerate(m1_idx): hdr[i] = (res[k], short[i], hb[k])
        # the reference's bookkeeping, message by message
        out = []
        for i, m in enumerate(msgs):
            out.append(self._process_one(m, is_m1[i], well[i], st[2 * i], st[2 * i + 1], hdr.get(i)))
        return out

    def _process_one(self, m, m1, well, st_vc, st_vid, hdr) -> Optional[str]:
        # ParseViewChangeMessage (view_change_msg.go:159-179): sender key, ViewchangeSig, ViewidSig must decode
        if len(m.SenderPubkey) != 48 or (well and st_vc == bls.VB_BAD_KEY_ENCODING): return errKeyDeserialize
        if len(m.ViewchangeSig) != 96 or st_vc == bls.VB_BAD_SIG_ENCODING: return errSigDeserialize
        if len(m.ViewidSig) != 96 or st_vid == bls.VB_BAD_SIG_ENCODING: return errSigDeserialize
        # onViewChangeSanityCheck (checks.go:184-191)
        if st_vid != bls.VB_OK: return errViewIDSig
        # ProcessViewChangeMsg (view_change_construct.go:237-375)
        sender = bytes(m.SenderPubkey).hex()
        if sender in self.viewIDSigs.get(m.ViewID, {}): return errDupM3
        if m1:
            err = self.verifyBlock(m.Block)
            if err: return err
            if sender in self.bhpSigs.get(m.ViewID, {}): return errDupM1
            if st_vc != bls.VB_OK: return errVerifyM1
            status, short, bitmap = hdr
            if status == bls.HDR_BAD_ENCODING: return errMultiSigDeserialize
            if short: return errSetMask
            if self.isQuorum:
                if not self.isQuorum(bitmap): return errNoQuorum
            elif status == bls.HDR_NO_QUORUM: return errNoQuorum
            if status != bls.HDR_OK: return errM1Payload
            self.bhpSigs.setdefault(m.ViewID, {})[sender] = bytes(m.ViewchangeSig)
            self._set_key(self.bhpBitmap, m.ViewID, m.SenderPubkey)
            self.viewIDSigs.setdefault(m.ViewID, {})[sender] = bytes(m.ViewidSig)
            self._set_key(self.viewIDBitmap, m.ViewID, m.SenderPubkey)
            if self.IsM1PayloadEmpty(): self.m1Payload = bytes(m.Payload)
            return None
        if sender in self.nilSigs.get(m.ViewID, {}): return errDupM2
        if st_vc != bls.VB_OK: return errVerifyM2
        self.nilSigs.setdefault(m.ViewID, {})[sender] = bytes(m.ViewchangeSig)
        self._set_key(self.nilBitmap, m.ViewID, m.SenderPubkey)
        self.viewIDSigs.setdefault(m.ViewID, {})[sender] = bytes(m.ViewidSig)
        self._set_key(self.viewIDBitmap, m.ViewID, m.SenderPubkey)
        return None

    def ProcessViewChangeMsg(self, m: FBFTMessage) -> Optional[str]:
        return self.ProcessViewChangeMsgs([m])[0]

    # ---- what the new leader puts into NEWVIEW (view_change_construct.go:122-151): aggregate bytes do not depend on the order of
    # the map iteration the reference sums in (SURVEY A.6)
    def GetM2Bitmap(self, viewID: int):
        sigs = list(self.nilSigs.get(viewID, {}).values())
        if not sigs: return None, None
        return self.be.aggregate_sigs(sigs), bytes(self.nilBitmap[viewID])
    def GetM3Bitmap(self, viewID: int):
        sigs = list(self.viewIDSigs.get(viewID, {}).values())
        if not sigs: return None, None
        return self.be.aggregate_sigs(sigs), bytes(self.viewIDBitmap[viewID])

    # ---- a validator receiving NEWVIEW: ParseNewViewMessage (view_change_msg.go:191-250), VerifyNewViewMsg (:154-234), the M3 quorum
    # and the M1 proof of onNewView (view_change.go:470-500) -- up to three aggregate checks over messages of 8 / 1 / 32 bytes in ONE
    # device call (hbls_verify_headers with the quorum gate off: the statuses tell "does not decode" from "does not verify")
    def OnNewViewChecks(self, m: FBFTMessage) -> Optional[str]:
        n = len(self.members)
        def mask_of(bm):        # NewMask + SetMask with the error ignored, as the parser does: a wrong length leaves the mask empty
            return bytes(bm) if bm is not None and len(bm) == self.blen else bytes(self.blen)
        has_m3 = m.M3AggSig is not None and len(m.M3AggSig) > 0
        has_m2 = m.M2AggSig is not None and len(m.M2AggSig) > 0
        m3_mask = mask_of(m.M3Bitmap) if has_m3 else None
        m2_mask = mask_of(m.M2Bitmap) if has_m2 else None
        need_m1 = has_m3 and (m2_mask is None or _popcount_slots(m3_mask, n) > _popcount_slots(m2_mask, n))
        items = []
        if has_m3: items.append(("m3", m3_mask, m.M3AggSig, _le64(m.ViewID)))
        if has_m2: items.append(("m2", m2_mask, m.M2AggSig, NIL))
        m1_err = None
        if need_m1:
            if 32 + 96 > len(m.Payload): m1_err = errPayloadLength
            else:
                body = m.Payload[32:]
                if len(body) - 96 != self.blen: m1_err = errSetMask
                items.append(("m1", bytes(self.blen) if m1_err else body[96:], body[:96], m.Payload[:32]))
        for it in items:
            if len(it[2]) != 96: return errSigDeserialize if it[0] != "m1" else errMultiSigDeserialize
        st = {}
        if items:
            res = self.be.verify_headers(self.com, [it[2] for it in items], [it[1] for it in items], [it[3] for it in items], 0)
            st = {it[0]: res[k] for k, it in enumerate(items)}
        # ParseNewViewMessage: the aggregate signatures must decode
        if st.get("m3") == bls.HDR_BAD_ENCODING or st.get("m2") == bls.HDR_BAD_ENCODING: return errSigDeserialize
        # VerifyNewViewMsg
        if not has_m3 or m.M3Bitmap is None: return errM3Nil
        self.newViewMsg.setdefault(m.ViewID, {})[bytes(m.SenderPubkey).hex()] = m.BlockNum
        if st["m3"] != bls.HDR_OK: return errM3Verify
        if has_m2 and st["m2"] != bls.HDR_OK: return errM2Verify
        if len(m.Payload) >= ValidPayloadLength and len(m.Block) != 0:
            err = self.verifyBlock(m.Block)
            if err: return err
        # onNewView: quorum over M3, then the PREPARED proof when the M3 signers outnumber the M2 signers
        if not (self.isQuorum(m3_mask) if self.isQuorum else _popcount_slots(m3_mask, n) >= self.quorum): return errNewViewQuorum
        if need_m1:
            if m1_err == errPayloadLength: return m1_err
            if st["m1"] == bls.HDR_BAD_ENCODING: return errMultiSigDeserialize
            if m1_err: return m1_err
            if st["m1"] != bls.HDR_OK: return errNewViewM1
        return None

# ------------------------------------------------------------------ the leader's vote collection (SURVEY 8a R9: "the real CPU bottleneck")
@dataclass
class Vote:
    """A PREPARE / COMMIT message as the leader reads it (consensus/leader.go:110-201, 203-345): one or several sender keys (a
    validator running several BLS keys signs once with their sum) and the signature bytes in Payload."""
    SenderPubkeys: List[bytes]
    Payload: bytes

class VoteCollector:
    """onPrepare / onCommit over a QUEUE of votes for one phase of one block: every vote of the queue is checked against the same
    message (block hash, or the commit payload) in ONE device call -- H(m) is hashed once --, then the reference's bookkeeping
    (already-received test, decider.AddNewVote -> submitVote, bitmap.SetKeysAtomic, quorum transition) runs over the booleans in
    arrival order.  The reference pays Deserialize + VerifyHash (~2 ms of cgo) per vote under consensus.mutex."""
    def __init__(self, members: List[bytes], message: bytes, backend=None):
        self.members = [bytes(m) for m in members]
        self.index = {m: i for i, m in enumerate(self.members)}
        self.message = bytes(message)
        self.be = backend or DeviceBackend()
        self.blen = (len(self.members) + 7) >> 3
        self.quorum = 2 * len(self.members) // 3 + 1            # uniform vote: TwoThirdsSignersCount (quorum.go:409-411)
        self.BallotBox = {}                                       # votepower.Round.BallotBox: key -> (SignerPubKeys, Signature)
        self.bitmap = bytearray(self.blen)
    def SignersCount(self) -> int: return len(self.BallotBox)                     # quorum.go:340-352
    def IsQuorumAchieved(self) -> bool: return self.SignersCount() >= self.quorum  # one-node-one-vote.go:46-54
    def onVotes(self, votes: List[Vote]):
        """Returns (errors, quorum_at): errors[i] is None when vote i was counted, else why it was dropped; quorum_at = index of the
        vote with which the quorum was first reached during this call (None if it was not, or was there before)."""
        n = len(votes)
        if n == 0: return [], None
        pre = [None] * n; pks, sigs = [], []
        for i, v in enumerate(votes):
            pk = bytes(48)
            if len(v.SenderPubkeys) == 1 and len(v.SenderPubkeys[0]) == 48: pk = bytes(v.SenderPubkeys[0])
            elif len(v.SenderPubkeys) > 1:
                try: pk = self.be.aggregate_keys(v.SenderPubkeys)
                except ValueError: pre[i] = errKeyDeserialize
            else: pre[i] = errKeyDeserialize
            pks.append(pk); sigs.append(bytes(v.Payload) if len(v.Payload) == 96 else bytes(96))
        st = self.be.verify_status(pks, sigs, [self.message] * n)
        out, quorum_at = [], None
        for i, v in enumerate(votes):
            was = self.IsQuorumAchieved()
            e = self._one(v, st[i], pre[i])
            out.append(e)
            if e is None and not was and self.IsQuorumAchieved() and quorum_at is None: quorum_at = i
        return out, quorum_at
    def _one(self, v, st, pre):
        keys = [bytes(k) for k in v.SenderPubkeys]
        if pre is not None or st == bls.VB_BAD_KEY_ENCODING: return errKeyDeserialize       # the message parser decodes the sender keys
        if any(k in self.BallotBox for k in keys): return errAlreadyReceived       # leader.go:127-136
        if len(v.Payload) != 96 or st == bls.VB_BAD_SIG_ENCODING: return errSigDeserialize
        if st != bls.VB_OK: return errVoteSig
        if len(set(keys)) != len(keys): return errDuplicateKey                      # submitVote (quorum.go:354-377)
        if any(k not in self.index for k in keys):                                  # SetKeysAtomic fails AFTER the ballots were recorded
            for k in keys: self.BallotBox[k] = (keys, bytes(v.Payload))
            return errKeyNotFound
        for k in keys: self.BallotBox[k] = (keys, bytes(v.Payload))
        for k in keys: i = self.index[k]; self.bitmap[i >> 3] |= 1 << (i & 7)
        return None
    def AggregateVotes(self):
        """consensus/quorum/quorum.go:164-196: one signature per ballot (a multi-key ballot is stored under each of its keys), then
        the aggregate in one device call; with the bitmap this is the payload of PREPARED / COMMITTED."""
        sigs, seen = [], set()
        for key, (keys, sig) in self.BallotBox.items():
            if any(k in seen for k in keys): continue
            seen.update(keys); sigs.append(sig)
        return (self.be.aggregate_sigs(sigs) if sigs else bytes(96)), bytes(self.bitmap)

class BoxBackend(DeviceBackend):
    """DeviceBackend plus the device ballot box that BallotBoxCollector collects into."""
    def ballot_box(self, com): return bls.BallotBox(com)

_UNDECODABLE = b"\xff" * 96             # x >= p: stands in for a payload of the wrong length, which Sign.Deserialize rejects too

class BallotBoxCollector:
    """VoteCollector's interface and results, collected into a device ballot box (hbls_ballot_box_submit_votes).  The leader maps
    sender keys to committee slots on the host; a queue whose votes each name distinct committee members goes to the device in ONE
    call -- signer keys summed from the committee table (no key decoded), H(m) hashed once, the already-received / Deserialize /
    VerifyHash rules applied in arrival order on the device, accepted signatures folded into the box's running sum without being
    decoded again.  A vote with a repeated key, a non-member key or a key held by a ballot without a bit (below) cuts the queue there
    and goes through VoteCollector's path (key sum, status triple); honest queues never hold one.
    The reference records a ballot of a non-member key (decider.AddNewVote) before bitmap.SetKeysAtomic fails (leader.go:185-196), so
    its signature counts in AggregateVotes without a bit: such a ballot enters the box with an empty bitmap, and its keys are kept
    here so that a later vote by one of them is "already received"."""
    def __init__(self, members: List[bytes], message: bytes, backend=None):
        self.members = [bytes(m) for m in members]
        self.index = {m: i for i, m in enumerate(self.members)}
        self.message = bytes(message)
        self.be = backend or BoxBackend()
        self.blen = (len(self.members) + 7) >> 3
        self.quorum = 2 * len(self.members) // 3 + 1            # uniform vote: TwoThirdsSignersCount (quorum.go:409-411)
        self.box = self.be.ballot_box(self.be.committee(self.members))
        self.BallotBox = {}                                       # votepower.Round.BallotBox: key -> (SignerPubKeys, Signature)
        self.unbitted = set()                                     # keys of ballots recorded without a bit
    def SignersCount(self) -> int: return len(self.BallotBox)
    def IsQuorumAchieved(self) -> bool: return self.SignersCount() >= self.quorum
    def _slots(self, v):
        """the vote's committee slots when the device can judge it alone, else None"""
        keys = [bytes(k) for k in v.SenderPubkeys]
        if not keys or len(set(keys)) != len(keys): return None
        if any(k not in self.index or k in self.unbitted for k in keys): return None
        return [self.index[k] for k in keys]
    def onVotes(self, votes: List[Vote]):
        """(errors, quorum_at) exactly as VoteCollector.onVotes."""
        n = len(votes)
        out, quorum_at = [None] * n, None
        i = 0
        while i < n:
            j, slots = i, []
            while j < n:
                s = self._slots(votes[j])
                if s is None: break
                slots.append(s); j += 1
            errs = self._device(votes[i:j], slots) if j > i else []
            if j < n: errs.append(self._irregular(votes[j])); j += 1
            for t, e in enumerate(errs):
                out[i + t] = e
            i = j
        # quorum transition, vote by vote (a vote changes the count only when it is counted)
        count = self.SignersCount() - sum(len(votes[t].SenderPubkeys) for t in range(n) if out[t] in (None, errKeyNotFound))
        for t in range(n):
            was = count >= self.quorum
            if out[t] in (None, errKeyNotFound): count += len(votes[t].SenderPubkeys)
            if out[t] is None and not was and count >= self.quorum and quorum_at is None: quorum_at = t
        return out, quorum_at
    def _device(self, votes, slots):
        bms = []
        for s in slots:
            bm = bytearray(self.blen)
            for x in s: bm[x >> 3] |= 1 << (x & 7)
            bms.append(bytes(bm))
        sigs = [bytes(v.Payload) if len(v.Payload) == 96 else _UNDECODABLE for v in votes]
        st = self.box.SubmitVotes(bms, sigs, _m48(self.message))             # what H(m) reads, as VoteCollector's backend passes it
        errs = []
        for v, s in zip(votes, st):
            if s == bls.BALLOT_ACCEPTED:
                keys = [bytes(k) for k in v.SenderPubkeys]
                for k in keys: self.BallotBox[k] = (keys, bytes(v.Payload))
                errs.append(None)
            else:
                errs.append(errAlreadyReceived if s == bls.BALLOT_COLLECTED else errSigDeserialize if s == bls.BALLOT_BAD_SIG_ENCODING else errVoteSig)
        return errs
    def _irregular(self, v):
        """VoteCollector's path for one vote (key sum, status triple, the reference's checks in order)"""
        keys = [bytes(k) for k in v.SenderPubkeys]
        pk, pre = bytes(48), None
        if len(keys) == 1 and len(keys[0]) == 48: pk = keys[0]
        elif len(keys) > 1:
            try: pk = self.be.aggregate_keys(keys)
            except ValueError: pre = errKeyDeserialize
        else: pre = errKeyDeserialize
        st = self.be.verify_status([pk], [bytes(v.Payload) if len(v.Payload) == 96 else bytes(96)], [self.message])[0]
        if pre is not None or st == bls.VB_BAD_KEY_ENCODING: return errKeyDeserialize
        if any(k in self.BallotBox for k in keys): return errAlreadyReceived
        if len(v.Payload) != 96 or st == bls.VB_BAD_SIG_ENCODING: return errSigDeserialize
        if st != bls.VB_OK: return errVoteSig
        if len(set(keys)) != len(keys): return errDuplicateKey
        for k in keys: self.BallotBox[k] = (keys, bytes(v.Payload))
        member = all(k in self.index for k in keys)
        bm = bytearray(self.blen)
        if member:
            for k in keys: i = self.index[k]; bm[i >> 3] |= 1 << (i & 7)
        else: self.unbitted.update(keys)
        self.box.AddVote(bytes(bm), bytes(v.Payload))
        return None if member else errKeyNotFound
    def AggregateVotes(self):
        """(aggregate signature, bitmap) of the collected ballots: the device box's running sum and bitmap (quorum.go:164-196)."""
        sig, bm = self.box.Aggregate()
        return (sig if self.BallotBox else bytes(96)), bm
