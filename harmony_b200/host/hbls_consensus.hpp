// harmony_b200/host/hbls_consensus.hpp -- the signature checks of Harmony's FBFT message handlers, batched over libhbls.so
// (SURVEY.md 8f rank 3; the callers behind BASELINE configs[3], the view-change storm).  C++ mirror, same names and error
// strings as the reference; harmony_b200/consensus.py is the Python twin the parity tests drive.
//
//   consensus/consensus_service.go:115-133  signMessage                 consensus/checks.go:20-56     verifyMessageSig
//   consensus/view_change_msg.go:139-190    ParseViewChangeMessage      consensus/checks.go:139-193   onViewChangeSanityCheck
//   consensus/view_change_construct.go:237-375 ProcessViewChangeMsg, :122-151 GetM2Bitmap / GetM3Bitmap, :154-234 VerifyNewViewMsg
//   consensus/view_change.go:445-500        onNewView (M3 quorum, M1 proof)
//   consensus/leader.go:110-345             onPrepare / onCommit (VoteCollector)    staking/slash/double-sign.go:139-262 (slash::VerifyBallots)
//
// The reference makes one cgo call per VerifyHash under consensus.mutex.  Here the booleans of a whole batch of VIEWCHANGE
// messages come from TWO device calls (hbls_verify_batch_status over the 2 N independent triples, hbls_verify_headers over the
// embedded PREPARED proofs); the reference's bookkeeping then runs over them in arrival order, so each message gets the error the
// sequential code returns.  Messages of different lengths share a batch: hash-to-G2 reads min(len, 48) bytes as a little-endian
// integer (SURVEY A.3), so NIL (1 byte), the view id (8) and an M1 payload (>= 128) are zero-padded / cut to 48 bytes.
// Out of scope (callbacks / opaque bytes): protobuf marshalling, RLP, block verification.
#pragma once
#include <functional>
#include <map>
#include "hbls_host.hpp"

namespace harmony {
namespace hash {       // == crypto/hash/hash.go:9-17 (golang.org/x/crypto/sha3.NewLegacyKeccak256)
inline void keccak_f1600(uint64_t a[25]) {
    static const uint64_t RC[24] = {0x0000000000000001ull, 0x0000000000008082ull, 0x800000000000808aull, 0x8000000080008000ull, 0x000000000000808bull,
        0x0000000080000001ull, 0x8000000080008081ull, 0x8000000000008009ull, 0x000000000000008aull, 0x0000000000000088ull, 0x0000000080008009ull,
        0x000000008000000aull, 0x000000008000808bull, 0x800000000000008bull, 0x8000000000008089ull, 0x8000000000008003ull, 0x8000000000008002ull,
        0x8000000000000080ull, 0x000000000000800aull, 0x800000008000000aull, 0x8000000080008081ull, 0x8000000000008080ull, 0x0000000080000001ull,
        0x8000000080008008ull};
    static const int ROT[25] = {0, 1, 62, 28, 27, 36, 44, 6, 55, 20, 3, 10, 43, 25, 39, 41, 45, 15, 21, 8, 18, 2, 61, 56, 14};      // index x + 5 y
    auto rol = [](uint64_t v, int n) { return n ? (v << n) | (v >> (64 - n)) : v; };
    for (int r = 0; r < 24; r++) {
        uint64_t c[5], b[25];
        for (int x = 0; x < 5; x++) c[x] = a[x] ^ a[x + 5] ^ a[x + 10] ^ a[x + 15] ^ a[x + 20];
        for (int x = 0; x < 5; x++) { const uint64_t d = c[(x + 4) % 5] ^ rol(c[(x + 1) % 5], 1); for (int y = 0; y < 5; y++) a[x + 5 * y] ^= d; }
        for (int x = 0; x < 5; x++) for (int y = 0; y < 5; y++) b[y + 5 * ((2 * x + 3 * y) % 5)] = rol(a[x + 5 * y], ROT[x + 5 * y]);
        for (int x = 0; x < 5; x++) for (int y = 0; y < 5; y++) a[x + 5 * y] = b[x + 5 * y] ^ (~b[(x + 1) % 5 + 5 * y] & b[(x + 2) % 5 + 5 * y]);
        a[0] ^= RC[r];
    }
}
inline std::vector<uint8_t> Keccak256(const uint8_t* data, size_t n) {
    const size_t rate = 136;
    std::vector<uint8_t> p(data, data + n);
    p.push_back(0x01); while (p.size() % rate) p.push_back(0); p.back() |= 0x80;
    uint64_t a[25] = {0};
    for (size_t off = 0; off < p.size(); off += rate) {
        for (size_t i = 0; i < rate / 8; i++) { uint64_t w = 0; for (int k = 7; k >= 0; k--) w = (w << 8) | p[off + 8 * i + k]; a[i] ^= w; }
        keccak_f1600(a);
    }
    std::vector<uint8_t> out(32);
    for (int i = 0; i < 4; i++) for (int k = 0; k < 8; k++) out[8 * i + k] = (uint8_t)(a[i] >> (8 * k));
    return out;
}
inline std::vector<uint8_t> Keccak256(const std::vector<uint8_t>& d) { return Keccak256(d.data(), d.size()); }
}  // namespace hash

namespace consensus {
using Bytes = std::vector<uint8_t>;
inline const Bytes& NIL() { static const Bytes nil{0x01}; return nil; }                       // consensus/config.go:49-52
constexpr size_t ValidPayloadLength = 32 + bls::BLSSignatureSizeInBytes;                     // view_change_construct.go:25-26
// error values, spelled as in the reference ("" = nil)
constexpr const char* errDupM1 = "received M1 (prepared) message already";
constexpr const char* errDupM2 = "received M2 (NIL) message already";
constexpr const char* errDupM3 = "received M3 (ViewID) message already";
constexpr const char* errVerifyM1 = "failed to verfiy signature for M1 message";
constexpr const char* errVerifyM2 = "failed to verfiy signature for M2 message";
constexpr const char* errM1Payload = "failed to verify multi signature for M1 prepared payload";
constexpr const char* errNoQuorum = "no quorum on M1 (prepared) payload";
constexpr const char* errViewIDSig = "[onViewChangeSanityCheck] Failed to Verify viewID Signature";
constexpr const char* errSigDeserialize = "err blsSignatureDeserialize";
constexpr const char* errKeyDeserialize = "err blsPublicKeyDeserialize";
constexpr const char* errMsgSig = "failed to verify the signature";
constexpr const char* errMultiSigDeserialize = "unable to deserialize multi-signature from payload";
constexpr const char* errSetMask = "mask.SetMask failed";
constexpr const char* errM3Nil = "[VerifyNewViewMsg] M3AggSig or M3Bitmap is nil";
constexpr const char* errM3Verify = "[VerifyNewViewMsg] Unable to Verify Aggregated Signature of M3 (ViewID) payload";
constexpr const char* errM2Verify = "[VerifyNewViewMsg] Unable to Verify Aggregated Signature of M2 (NIL) payload";
constexpr const char* errNewViewQuorum = "[onNewView] Quorum Not achieved";
constexpr const char* errNewViewM1 = "[onNewView] Failed to Verify Signature for M1 (prepare) message";
constexpr const char* errPayloadLength = "payload not have enough length";

inline Bytes le64(uint64_t v) { Bytes b(8); for (int i = 0; i < 8; i++) b[i] = (uint8_t)(v >> (8 * i)); return b; }
// what hash-to-G2 reads of a message: its first 48 bytes as a little-endian integer == zero-padded to 48 bytes
inline void put48(Bytes& blob, const Bytes& m) { const size_t o = blob.size(); blob.resize(o + 48, 0); std::memcpy(&blob[o], m.data(), m.size() < 48 ? m.size() : 48); }

// consensus/consensus_service.go:115-119
inline Bytes signMessage(const Bytes& message, const bls_core::SecretKey* priKey) {
    std::unique_ptr<bls_core::Sign> s(priKey->SignHash(hash::Keccak256(message)));
    return s ? s->Serialize() : Bytes();
}
// consensus/checks.go:20-39 on the marshalled message (Signature field cleared by the caller)
inline std::string verifyMessageSig(const bls_core::PublicKey* signerPubKey, const Bytes& message, const Bytes& signature) {
    bls_core::Sign msgSig;
    if (!msgSig.Deserialize(signature)) return errSigDeserialize;
    if (!msgSig.VerifyHash(signerPubKey, hash::Keccak256(message))) return errMsgSig;
    return "";
}
// one device call for independent (key, message, signature) triples: statuses HBLS_VB_*; malformed lengths are reported as the
// matching decode failure
inline std::vector<uint8_t> verifyStatus(const std::vector<Bytes>& pks, const std::vector<Bytes>& sigs, const std::vector<Bytes>& msgs) {
    const size_t k = pks.size();
    std::vector<uint8_t> st(k, HBLS_VB_BAD_SIG);
    if (!k) return st;
    Bytes pb(48 * k, 0), sb(96 * k, 0), mb; mb.reserve(48 * k);
    for (size_t i = 0; i < k; i++) {
        if (pks[i].size() == 48) std::memcpy(&pb[48 * i], pks[i].data(), 48);
        if (sigs[i].size() == 96) std::memcpy(&sb[96 * i], sigs[i].data(), 96);
        put48(mb, msgs[i]);
    }
    if (hbls_verify_batch_status(k, pb.data(), sb.data(), mb.data(), 48, st.data()) != 0) throw std::runtime_error("hbls_verify_batch_status failed");
    for (size_t i = 0; i < k; i++) { if (pks[i].size() != 48) st[i] = HBLS_VB_BAD_KEY_ENCODING; else if (sigs[i].size() != 96) st[i] = HBLS_VB_BAD_SIG_ENCODING; }
    return st;
}
// senderKeySanityChecks (checks.go:41-56) for a queue of received messages
inline std::vector<std::string> verifyMessageSigBatch(const std::vector<Bytes>& senderKeys, const std::vector<Bytes>& messages, const std::vector<Bytes>& signatures) {
    std::vector<Bytes> digests; for (auto& m : messages) digests.push_back(hash::Keccak256(m));
    auto st = verifyStatus(senderKeys, signatures, digests);
    std::vector<std::string> out;
    for (uint8_t s : st) out.push_back(s == HBLS_VB_OK ? "" : s == HBLS_VB_BAD_KEY_ENCODING ? errKeyDeserialize : s == HBLS_VB_BAD_SIG_ENCODING ? errSigDeserialize : errMsgSig);
    return out;
}

// the fields of FBFTMessage (consensus/fbft_log.go) the view-change checks read; keys and signatures as wire bytes
struct FBFTMessage {
    uint64_t ViewID = 0, BlockNum = 0;
    Bytes SenderPubkey, LeaderPubkey, Payload, Block, ViewchangeSig, ViewidSig;
    bool hasM2 = false, hasM3 = false;              // NEWVIEW: len(M2Aggsigs) > 0 / len(M3Aggsigs) > 0
    Bytes M2AggSig, M2Bitmap, M3AggSig, M3Bitmap;
};

class viewChange {     // consensus/view_change_construct.go:31-51
public:
    using SigTable = std::map<uint64_t, std::map<std::string, Bytes>>;
    SigTable bhpSigs, nilSigs, viewIDSigs;
    std::map<uint64_t, Bytes> bhpBitmap, nilBitmap, viewIDBitmap;
    Bytes m1Payload;
    std::function<std::string(const Bytes&)> verifyBlock = [](const Bytes&) { return std::string(); };
    std::function<bool(const Bytes&)> isQuorumAchievedByMask;        // empty: uniform vote, 2n/3 + 1 slots (one-node-one-vote.go:57-72)

    std::string Init(const std::vector<bls::PublicKeyWrapper>& members) {
        members_ = members; index_.clear();
        for (size_t i = 0; i < members.size(); i++) index_[members[i].Hex()] = i;
        blen_ = (members.size() + 7) >> 3; quorum_ = (size_t)quorum::TwoThirdsSignersCount((int64_t)members.size());
        Reset();
        return com_.Load(members);
    }
    void Reset() { bhpSigs.clear(); nilSigs.clear(); viewIDSigs.clear(); bhpBitmap.clear(); nilBitmap.clear(); viewIDBitmap.clear(); m1Payload.clear(); }
    bool IsM1PayloadEmpty() const { return m1Payload.empty(); }

    // onViewChangeSanityCheck's signature check + ProcessViewChangeMsg for every message, in arrival order: "" or the error
    std::vector<std::string> ProcessViewChangeMsgs(const std::vector<FBFTMessage>& msgs) {
        const size_t n = msgs.size();
        std::vector<std::string> out(n);
        if (!n) return out;
        std::vector<Bytes> pks, sigs, ms; std::vector<bool> m1(n);
        for (size_t i = 0; i < n; i++) {
            const FBFTMessage& m = msgs[i];
            m1[i] = m.Payload.size() >= ValidPayloadLength && !m.Block.empty();
            pks.push_back(m.SenderPubkey); sigs.push_back(m.ViewchangeSig); ms.push_back(m1[i] ? m.Payload : NIL());
            pks.push_back(m.SenderPubkey); sigs.push_back(m.ViewidSig); ms.push_back(le64(m.ViewID));
        }
        const auto st = verifyStatus(pks, sigs, ms);                                     // device call 1
        std::vector<size_t> idx; Bytes hs, hb, hp; std::vector<bool> shortbm;
        for (size_t i = 0; i < n; i++) if (m1[i]) {
            const Bytes& p = msgs[i].Payload;
            const bool sh = p.size() - 128 != blen_;                                     // mask.SetMask: "mismatching bitmap lengths"
            idx.push_back(i); shortbm.push_back(sh);
            hs.insert(hs.end(), p.begin() + 32, p.begin() + 128);
            if (sh) hb.resize(hb.size() + blen_, 0); else hb.insert(hb.end(), p.begin() + 128, p.end());
            put48(hp, Bytes(p.begin(), p.begin() + 32));
        }
        std::vector<uint8_t> hst(idx.size());
        if (!idx.empty() && hbls_verify_headers(com_.handle(), idx.size(), hs.data(), hb.data(), blen_, hp.data(), 48,       // device call 2
                                                isQuorumAchievedByMask ? 0 : quorum_, hst.data()) != 0) throw std::runtime_error("hbls_verify_headers failed");
        size_t k = 0;
        for (size_t i = 0; i < n; i++) {
            const size_t kk = m1[i] ? k++ : 0;
            out[i] = processOne(msgs[i], m1[i], st[2 * i], st[2 * i + 1], m1[i] ? hst[kk] : 0, m1[i] ? (bool)shortbm[kk] : false,
                                m1[i] ? Bytes(hb.begin() + kk * blen_, hb.begin() + (kk + 1) * blen_) : Bytes());
        }
        return out;
    }
    std::string ProcessViewChangeMsg(const FBFTMessage& m) { return ProcessViewChangeMsgs({m})[0]; }

    // view_change_construct.go:122-151: (aggregate signature, bitmap), empty when nobody signed.  The bytes do not depend on the
    // order the reference's map iteration sums in (SURVEY A.6)
    bool GetM2Bitmap(uint64_t viewID, Bytes& sig, Bytes& bitmap) { return aggregate(nilSigs, nilBitmap, viewID, sig, bitmap); }
    bool GetM3Bitmap(uint64_t viewID, Bytes& sig, Bytes& bitmap) { return aggregate(viewIDSigs, viewIDBitmap, viewID, sig, bitmap); }

    // a validator receiving NEWVIEW: ParseNewViewMessage's decodes, VerifyNewViewMsg, the M3 quorum and the M1 proof of onNewView:
    // up to three aggregate checks over 8 / 1 / 32-byte messages in ONE hbls_verify_headers call (quorum gate off)
    std::string OnNewViewChecks(const FBFTMessage& m) {
        const size_t n = members_.size();
        auto maskOf = [&](const Bytes& bm) { return bm.size() == blen_ ? bm : Bytes(blen_, 0); };     // the parser ignores SetMask's error
        const Bytes m3 = m.hasM3 ? maskOf(m.M3Bitmap) : Bytes(), m2 = m.hasM2 ? maskOf(m.M2Bitmap) : Bytes();
        const bool needM1 = m.hasM3 && (!m.hasM2 || quorum::CountSlotBits(m3, n) > quorum::CountSlotBits(m2, n));
        struct Item { char kind; Bytes bitmap, sig, msg; };
        std::vector<Item> items;
        if (m.hasM3) items.push_back({'3', m3, m.M3AggSig, le64(m.ViewID)});
        if (m.hasM2) items.push_back({'2', m2, m.M2AggSig, NIL()});
        std::string m1err;
        if (needM1) {
            if (32 + 96 > m.Payload.size()) m1err = errPayloadLength;
            else {
                if (m.Payload.size() - 128 != blen_) m1err = errSetMask;
                items.push_back({'1', m1err.empty() ? Bytes(m.Payload.begin() + 128, m.Payload.end()) : Bytes(blen_, 0),
                                 Bytes(m.Payload.begin() + 32, m.Payload.begin() + 128), Bytes(m.Payload.begin(), m.Payload.begin() + 32)});
            }
        }
        for (auto& it : items) if (it.sig.size() != 96) return it.kind == '1' ? errMultiSigDeserialize : errSigDeserialize;
        std::map<char, uint8_t> st;
        if (!items.empty()) {
            Bytes hs, hb, hp; for (auto& it : items) { hs.insert(hs.end(), it.sig.begin(), it.sig.end()); hb.insert(hb.end(), it.bitmap.begin(), it.bitmap.end()); put48(hp, it.msg); }
            std::vector<uint8_t> res(items.size());
            if (hbls_verify_headers(com_.handle(), items.size(), hs.data(), hb.data(), blen_, hp.data(), 48, 0, res.data()) != 0) throw std::runtime_error("hbls_verify_headers failed");
            for (size_t i = 0; i < items.size(); i++) st[items[i].kind] = res[i];
        }
        if ((m.hasM3 && st['3'] == HBLS_HDR_BAD_ENCODING) || (m.hasM2 && st['2'] == HBLS_HDR_BAD_ENCODING)) return errSigDeserialize;
        if (!m.hasM3 || m.M3Bitmap.empty()) return errM3Nil;
        if (st['3'] != HBLS_HDR_OK) return errM3Verify;
        if (m.hasM2 && st['2'] != HBLS_HDR_OK) return errM2Verify;
        if (m.Payload.size() >= ValidPayloadLength && !m.Block.empty()) { const std::string e = verifyBlock(m.Block); if (!e.empty()) return e; }
        if (!(isQuorumAchievedByMask ? isQuorumAchievedByMask(m3) : (size_t)quorum::CountSlotBits(m3, n) >= quorum_)) return errNewViewQuorum;
        if (needM1) {
            if (m1err == errPayloadLength) return m1err;
            if (st['1'] == HBLS_HDR_BAD_ENCODING) return errMultiSigDeserialize;
            if (!m1err.empty()) return m1err;
            if (st['1'] != HBLS_HDR_OK) return errNewViewM1;
        }
        return "";
    }
private:
    std::vector<bls::PublicKeyWrapper> members_; std::unordered_map<std::string, size_t> index_;
    bls::Committee com_; size_t blen_ = 0, quorum_ = 0;

    void setKey(std::map<uint64_t, Bytes>& table, uint64_t viewID, const std::string& senderHex) {        // Mask.SetKey(key, true)
        Bytes& bm = table[viewID]; if (bm.empty()) bm.assign(blen_, 0);
        auto it = index_.find(senderHex); if (it != index_.end()) bm[it->second >> 3] |= (uint8_t)(1u << (it->second & 7));
    }
    static bool has(const SigTable& t, uint64_t viewID, const std::string& k) { auto it = t.find(viewID); return it != t.end() && it->second.count(k); }
    bool aggregate(const SigTable& sigs, const std::map<uint64_t, Bytes>& bitmaps, uint64_t viewID, Bytes& sig, Bytes& bitmap) {
        auto it = sigs.find(viewID); sig.clear(); bitmap.clear();
        if (it == sigs.end() || it->second.empty()) return false;
        Bytes blob; for (auto& kv : it->second) blob.insert(blob.end(), kv.second.begin(), kv.second.end());
        sig.resize(96);
        if (hbls_aggregate_sigs(blob.data(), it->second.size(), sig.data()) != 0) { sig.clear(); return false; }
        bitmap = bitmaps.at(viewID); return true;
    }
    std::string processOne(const FBFTMessage& m, bool m1, uint8_t stVc, uint8_t stVid, uint8_t hdr, bool shortBitmap, const Bytes& bitmap) {
        // ParseViewChangeMessage (view_change_msg.go:159-179): sender key, ViewchangeSig, ViewidSig must decode
        if (stVc == HBLS_VB_BAD_KEY_ENCODING || stVid == HBLS_VB_BAD_KEY_ENCODING) return errKeyDeserialize;
        if (stVc == HBLS_VB_BAD_SIG_ENCODING || stVid == HBLS_VB_BAD_SIG_ENCODING) return errSigDeserialize;
        if (stVid != HBLS_VB_OK) return errViewIDSig;                                                    // checks.go:184-191
        const std::string sender = bls_core::hex(m.SenderPubkey.data(), m.SenderPubkey.size());
        if (has(viewIDSigs, m.ViewID, sender)) return errDupM3;
        if (m1) {
            const std::string e = verifyBlock(m.Block); if (!e.empty()) return e;
            if (has(bhpSigs, m.ViewID, sender)) return errDupM1;
            if (stVc != HBLS_VB_OK) return errVerifyM1;
            if (hdr == HBLS_HDR_BAD_ENCODING) return errMultiSigDeserialize;                             // internal/chain/sig.go:39-43
            if (shortBitmap) return errSetMask;                                                          // sig.go:44-48
            if (isQuorumAchievedByMask ? !isQuorumAchievedByMask(bitmap) : hdr == HBLS_HDR_NO_QUORUM) return errNoQuorum;
            if (hdr != HBLS_HDR_OK) return errM1Payload;
            bhpSigs[m.ViewID][sender] = m.ViewchangeSig; setKey(bhpBitmap, m.ViewID, sender);
            viewIDSigs[m.ViewID][sender] = m.ViewidSig; setKey(viewIDBitmap, m.ViewID, sender);
            if (IsM1PayloadEmpty()) m1Payload = m.Payload;
            return "";
        }
        if (has(nilSigs, m.ViewID, sender)) return errDupM2;
        if (stVc != HBLS_VB_OK) return errVerifyM2;
        nilSigs[m.ViewID][sender] = m.ViewchangeSig; setKey(nilBitmap, m.ViewID, sender);
        viewIDSigs[m.ViewID][sender] = m.ViewidSig; setKey(viewIDBitmap, m.ViewID, sender);
        return "";
    }
};

// ------------------------------------------------------------------ the leader's vote collection (consensus/leader.go:110-345; SURVEY 8a R9)
constexpr const char* errAlreadyReceived = "already received message from the validator";      // leader.go:127-136,233-241
constexpr const char* errVoteSig = "received invalid BLS signature";                            // leader.go:171-180,287-290
constexpr const char* errDuplicateKey = "duplicate key found in votes";                          // quorum.go:361-363
constexpr const char* errKeyNotFound = "key not found";                                          // crypto/bls/mask.go:226-233

// sum of a multi-key sender's keys (leader.go:161-169, double-sign.go:241-249): BytesToBLSPublicKey's LRU + PublicKey.Add
inline bool aggregateKeys(const std::vector<Bytes>& keys, Bytes& out) {
    bls_core::PublicKey acc;
    for (auto& k : keys) { auto pk = bls::BytesToBLSPublicKey(k); if (!pk) return false; acc.Add(pk.get()); }
    out = acc.Serialize(); return true;
}

struct Vote { std::vector<Bytes> SenderPubkeys; Bytes Payload; };      // PREPARE / COMMIT as the leader reads it: sender key(s) + signature

// onPrepare / onCommit over a QUEUE of votes for one phase of one block: every vote against the same message in ONE device call (H(m)
// hashed once), then the reference's bookkeeping (already-received test, AddNewVote -> submitVote, SetKeysAtomic, quorum transition)
// in arrival order
class VoteCollector {
public:
    struct Ballot { std::vector<Bytes> SignerPubKeys; Bytes Signature; };
    std::map<Bytes, Ballot> BallotBox;          // votepower.Round.BallotBox: one entry per signer key
    Bytes bitmap;
    void Init(const std::vector<bls::PublicKeyWrapper>& members, const Bytes& message) {
        index_.clear(); for (size_t i = 0; i < members.size(); i++) index_[Bytes(members[i].Bytes.begin(), members[i].Bytes.end())] = i;
        message_ = message; bitmap.assign((members.size() + 7) >> 3, 0); BallotBox.clear();
        quorum_ = (size_t)quorum::TwoThirdsSignersCount((int64_t)members.size());
    }
    size_t SignersCount() const { return BallotBox.size(); }                       // quorum.go:340-352
    bool IsQuorumAchieved() const { return SignersCount() >= quorum_; }            // one-node-one-vote.go:46-54
    // errors[i] == "" when vote i was counted; quorumAt = index of the vote that first reached the quorum in this call, or -1
    std::vector<std::string> onVotes(const std::vector<Vote>& votes, long* quorumAt = nullptr) {
        const size_t n = votes.size();
        std::vector<std::string> out(n); if (quorumAt) *quorumAt = -1;
        if (!n) return out;
        std::vector<Bytes> pks(n), sigs(n), msgs(n, message_); std::vector<bool> keyErr(n, false);
        for (size_t i = 0; i < n; i++) {
            const Vote& v = votes[i];
            if (v.SenderPubkeys.size() == 1) pks[i] = v.SenderPubkeys[0];
            else if (v.SenderPubkeys.empty() || !aggregateKeys(v.SenderPubkeys, pks[i])) { keyErr[i] = true; pks[i] = Bytes(48, 0); }
            sigs[i] = v.Payload;
        }
        const auto st = verifyStatus(pks, sigs, msgs);
        for (size_t i = 0; i < n; i++) {
            const bool was = IsQuorumAchieved();
            out[i] = one(votes[i], st[i], keyErr[i]);
            if (out[i].empty() && !was && IsQuorumAchieved() && quorumAt && *quorumAt < 0) *quorumAt = (long)i;
        }
        return out;
    }
    // consensus/quorum/quorum.go:164-196: one signature per ballot (a multi-key ballot sits under each of its keys), one device call
    bool AggregateVotes(Bytes& sig) const {
        Bytes blob; std::map<Bytes, bool> seen; size_t cnt = 0;
        for (auto& kv : BallotBox) {
            bool dup = false; for (auto& k : kv.second.SignerPubKeys) if (seen.count(k)) { dup = true; break; }
            if (dup) continue;
            for (auto& k : kv.second.SignerPubKeys) seen[k] = true;
            blob.insert(blob.end(), kv.second.Signature.begin(), kv.second.Signature.end()); cnt++;
        }
        sig.assign(96, 0);
        return cnt == 0 || hbls_aggregate_sigs(blob.data(), cnt, sig.data()) == 0;
    }
private:
    std::map<Bytes, size_t> index_; Bytes message_; size_t quorum_ = 0;
    std::string one(const Vote& v, uint8_t st, bool keyErr) {
        if (keyErr || st == HBLS_VB_BAD_KEY_ENCODING) return errKeyDeserialize;             // the message parser decodes the sender keys
        for (auto& k : v.SenderPubkeys) if (BallotBox.count(k)) return errAlreadyReceived;
        if (st == HBLS_VB_BAD_SIG_ENCODING) return errSigDeserialize;
        if (st != HBLS_VB_OK) return errVoteSig;
        for (size_t a = 0; a < v.SenderPubkeys.size(); a++) for (size_t b = a + 1; b < v.SenderPubkeys.size(); b++)
            if (v.SenderPubkeys[a] == v.SenderPubkeys[b]) return errDuplicateKey;             // submitVote (quorum.go:354-377)
        for (auto& k : v.SenderPubkeys) BallotBox[k] = Ballot{v.SenderPubkeys, v.Payload};
        for (auto& k : v.SenderPubkeys) if (!index_.count(k)) return errKeyNotFound;          // SetKeysAtomic, after the ballots were recorded
        for (auto& k : v.SenderPubkeys) { const size_t i = index_[k]; bitmap[i >> 3] |= (uint8_t)(1u << (i & 7)); }
        return "";
    }
};

// VoteCollector's interface and results, collected into a device ballot box (hbls_ballot_box_submit_votes; consensus.py:
// BallotBoxCollector is the Python twin).  Sender keys are mapped to committee slots on the host; a run of votes that each name
// distinct committee members goes to the device in ONE call -- keys summed from the committee table (no key decoded), H(m) once, the
// already-received / Deserialize / VerifyHash rules in arrival order, accepted signatures folded into the box without a second decode.
// A vote with a repeated key, a non-member key or a key held by a ballot without a bit cuts the queue there and takes VoteCollector's
// path (key sum, status triple); honest queues never hold one.  The reference records a non-member's ballot (decider.AddNewVote)
// before bitmap.SetKeysAtomic fails (leader.go:185-196), so its signature counts in AggregateVotes without a bit: it enters the box
// with an empty bitmap, and its keys are kept here so that a later vote by one of them is "already received".
class BallotBoxCollector {
public:
    using Ballot = VoteCollector::Ballot;
    std::map<Bytes, Ballot> BallotBox;          // votepower.Round.BallotBox: one entry per signer key
    Bytes bitmap;                               // the box's bitmap, as the device returned it with the last queue
    std::string Init(const std::vector<bls::PublicKeyWrapper>& members, const Bytes& message) {
        index_.clear(); for (size_t i = 0; i < members.size(); i++) index_[Bytes(members[i].Bytes.begin(), members[i].Bytes.end())] = i;
        message_.clear(); put48(message_, message);                  // what hash-to-G2 reads of the message (VoteCollector: verifyStatus)
        blen_ = (members.size() + 7) >> 3; bitmap.assign(blen_, 0); BallotBox.clear(); unbitted_.clear();
        quorum_ = (size_t)quorum::TwoThirdsSignersCount((int64_t)members.size());
        const std::string e = com_.Load(members);
        return e.empty() ? box_.Create(com_) : e;
    }
    size_t SignersCount() const { return BallotBox.size(); }
    bool IsQuorumAchieved() const { return SignersCount() >= quorum_; }
    // errors[i] == "" when vote i was counted; quorumAt = index of the vote that first reached the quorum in this call, or -1
    std::vector<std::string> onVotes(const std::vector<Vote>& votes, long* quorumAt = nullptr) {
        const size_t n = votes.size();
        std::vector<std::string> out(n); if (quorumAt) *quorumAt = -1;
        size_t i = 0;
        while (i < n) {
            size_t j = i; std::vector<std::vector<size_t>> slots;
            for (std::vector<size_t> s; j < n && slotsOf(votes[j], s); j++) slots.push_back(s);
            if (j > i) device(votes, i, slots, out);
            if (j < n) { out[j] = irregular(votes[j]); j++; }
            i = j;
        }
        // the quorum transition, vote by vote: a vote changes the count only when its ballot is recorded
        auto recorded = [](const std::string& e) { return e.empty() || e == errKeyNotFound; };
        size_t count = SignersCount();
        for (size_t t = 0; t < n; t++) if (recorded(out[t])) count -= votes[t].SenderPubkeys.size();
        for (size_t t = 0; t < n; t++) {
            const bool was = count >= quorum_;
            if (recorded(out[t])) count += votes[t].SenderPubkeys.size();
            if (out[t].empty() && !was && count >= quorum_ && quorumAt && *quorumAt < 0) *quorumAt = (long)t;
        }
        return out;
    }
    // quorum.go:164-196 from the box: its running sum (all zero when nothing was collected, as VoteCollector) and its bitmap
    bool AggregateVotes(Bytes& sig) const { Bytes bm; return AggregateVotes(sig, bm); }
    bool AggregateVotes(Bytes& sig, Bytes& bm) const {
        if (!box_.Aggregate(sig, bm)) return false;
        if (BallotBox.empty()) sig.assign(96, 0);
        return true;
    }
private:
    std::map<Bytes, size_t> index_; std::set<Bytes> unbitted_; Bytes message_; size_t blen_ = 0, quorum_ = 0;
    bls::Committee com_; bls::BallotBox box_;

    // the vote's committee slots when the device can judge it alone
    bool slotsOf(const Vote& v, std::vector<size_t>& s) const {
        s.clear();
        if (v.SenderPubkeys.empty()) return false;
        std::set<Bytes> seen;
        for (auto& k : v.SenderPubkeys) {
            auto it = index_.find(k);
            if (it == index_.end() || unbitted_.count(k) || !seen.insert(k).second) return false;
            s.push_back(it->second);
        }
        return true;
    }
    void device(const std::vector<Vote>& votes, size_t i0, const std::vector<std::vector<size_t>>& slots, std::vector<std::string>& out) {
        const size_t k = slots.size();
        Bytes bms(k * blen_, 0), sigs(96 * k, 0xff);                  // 0xff...: x >= p, stands in for a payload of the wrong length
        for (size_t t = 0; t < k; t++) {
            for (size_t x : slots[t]) bms[t * blen_ + (x >> 3)] |= (uint8_t)(1u << (x & 7));
            const Bytes& p = votes[i0 + t].Payload;
            if (p.size() == 96) std::memcpy(&sigs[96 * t], p.data(), 96);
        }
        std::vector<uint8_t> st;
        const std::string e = box_.SubmitVotes(bms, sigs, message_, st);
        if (!e.empty()) throw std::runtime_error(e);
        for (size_t t = 0; t < k; t++) {
            const Vote& v = votes[i0 + t];
            if (st[t] == HBLS_BALLOT_ACCEPTED) {
                for (auto& key : v.SenderPubkeys) BallotBox[key] = Ballot{v.SenderPubkeys, v.Payload};
                for (size_t x : slots[t]) bitmap[x >> 3] |= (uint8_t)(1u << (x & 7));
                out[i0 + t] = "";
            } else out[i0 + t] = st[t] == HBLS_BALLOT_COLLECTED ? errAlreadyReceived : st[t] == HBLS_BALLOT_BAD_SIG_ENCODING ? errSigDeserialize : errVoteSig;
        }
    }
    // VoteCollector's path for one vote
    std::string irregular(const Vote& v) {
        Bytes pk(48, 0); bool keyErr = false;
        if (v.SenderPubkeys.size() == 1) pk = v.SenderPubkeys[0];
        else if (v.SenderPubkeys.empty() || !aggregateKeys(v.SenderPubkeys, pk)) { keyErr = true; pk = Bytes(48, 0); }
        const uint8_t st = verifyStatus({pk}, {v.Payload}, {message_})[0];
        if (keyErr || st == HBLS_VB_BAD_KEY_ENCODING) return errKeyDeserialize;
        for (auto& k : v.SenderPubkeys) if (BallotBox.count(k)) return errAlreadyReceived;
        if (st == HBLS_VB_BAD_SIG_ENCODING) return errSigDeserialize;
        if (st != HBLS_VB_OK) return errVoteSig;
        for (size_t a = 0; a < v.SenderPubkeys.size(); a++) for (size_t b = a + 1; b < v.SenderPubkeys.size(); b++)
            if (v.SenderPubkeys[a] == v.SenderPubkeys[b]) return errDuplicateKey;
        for (auto& k : v.SenderPubkeys) BallotBox[k] = Ballot{v.SenderPubkeys, v.Payload};
        bool member = true; for (auto& k : v.SenderPubkeys) member &= index_.count(k) != 0;
        Bytes bm(blen_, 0);
        if (member) for (auto& k : v.SenderPubkeys) { const size_t x = index_.at(k); bm[x >> 3] |= (uint8_t)(1u << (x & 7)); }
        else for (auto& k : v.SenderPubkeys) unbitted_.insert(k);
        if (box_.AddVote(bm, v.Payload) < 0) throw std::runtime_error("hbls_ballot_box_add_vote failed");
        for (size_t x = 0; x < blen_; x++) bitmap[x] |= bm[x];
        return member ? "" : errKeyNotFound;
    }
};
}  // namespace consensus

namespace slash {      // == staking/slash/double-sign.go:139-168,215-262, the ballot checks that need no chain state
using consensus::Bytes;
constexpr const char* errSignerKeyNotRightSize = "bls keys from slash candidate not right side";
constexpr const char* errSlashBlockNoConflict = "cannot slash for signing on non-conflicting blocks";
constexpr const char* errNoMatchingDoubleSignKeys = "no matching double sign keys";
constexpr const char* errFailVerifySlash = "could not verify bls key signature on slash";
struct Vote { std::vector<Bytes> SignerPubKeys; std::array<uint8_t, 32> BlockHeaderHash{}; Bytes Signature; };
struct Evidence { uint64_t Epoch = 0, Height = 0, ViewID = 0; uint32_t ShardID = 0; Vote FirstVote, SecondVote; };
struct Record { slash::Evidence Evidence; };
// per record "" or the first error slash.Verify would return from its ballot checks; the 2 R signature checks in ONE device call
inline std::vector<std::string> VerifyBallots(const std::vector<Record>& records) {
    std::vector<std::string> out(records.size());
    std::vector<Bytes> pks, sigs, msgs; std::vector<std::pair<size_t, std::string>> owner;      // (record, error known before the device call)
    for (size_t r = 0; r < records.size(); r++) {
        const Vote &first = records[r].Evidence.FirstVote, &second = records[r].Evidence.SecondVote;
        bool sized = true; for (auto* v : {&first, &second}) for (auto& k : v->SignerPubKeys) sized &= k.size() == bls::PublicKeySizeInBytes;
        if (!sized) { out[r] = errSignerKeyNotRightSize; continue; }
        if (first.BlockHeaderHash == second.BlockHeaderHash) { out[r] = errSlashBlockNoConflict; continue; }
        bool match = false; for (auto& a : first.SignerPubKeys) for (auto& b : second.SignerPubKeys) match |= a == b;
        if (!match) { out[r] = errNoMatchingDoubleSignKeys; continue; }
        for (auto* v : {&first, &second}) {
            // slash verification only happens in the staking era: 48-byte commit payload (double-sign.go:250-252)
            Bytes apk(48, 0); std::string pre;
            bls_core::Sign probe;
            if (v->Signature.size() != 96) pre = consensus::errSigDeserialize;
            else if (!consensus::aggregateKeys(v->SignerPubKeys, apk)) { pre = probe.Deserialize(v->Signature) ? consensus::errKeyDeserialize : consensus::errSigDeserialize; apk.assign(48, 0); }
            pks.push_back(apk); sigs.push_back(v->Signature);
            msgs.push_back(signature::ConstructCommitPayload(true, v->BlockHeaderHash, records[r].Evidence.Height, records[r].Evidence.ViewID));
            owner.push_back({r, pre});
        }
    }
    const auto st = consensus::verifyStatus(pks, sigs, msgs);
    for (size_t k = 0; k < owner.size(); k++) {
        const size_t r = owner[k].first;
        if (!out[r].empty()) continue;                             // the first ballot already failed
        if (!owner[k].second.empty()) out[r] = owner[k].second;
        else if (st[k] == HBLS_VB_BAD_SIG_ENCODING) out[r] = consensus::errSigDeserialize;
        else if (st[k] != HBLS_VB_OK) out[r] = errFailVerifySlash;
    }
    return out;
}
}  // namespace slash
}  // namespace harmony
