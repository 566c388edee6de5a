// harmony_b200/host/hbls_host.hpp -- C++ host-side mirror of the Go packages that sit on the BLS hot path.
//
// The reference's host code is Go (no Go toolchain in this image), so the layer above the C ABI is written in
// C++ with the reference's names, argument meaning and error behaviour:
//   github.com/harmony-one/bls/ffi/go/bls : SecretKey / PublicKey / Sign            (SURVEY.md 8b)
//   crypto/bls/bls.go, mask.go            : SerializedPublicKey, PublicKeyWrapper, BytesToBLSPublicKey (+LRU 1024),
//                                           AggregateSig, Mask, SeparateSigAndMask
//   multibls/multibls.go                  : PrivateKeys / PublicKeys (Dedup, Contains, GetPublicKeys)
//   consensus/signature/signature.go      : ConstructCommitPayload
//   internal/chain/sig.go                 : ParseCommitSigAndBitmap, DecodeSigBitmap
//   consensus/quorum (uniform vote)       : TwoThirdsSignersCount, IsQuorumAchievedByMask, AggregateVotes
//   internal/chain/engine.go:606-642      : verifySignature(+Cached) over a device-resident committee
// Everything that touches a group element goes through include/hbls.h into the CUDA kernels.
#pragma once
#include <array>
#include <cstdint>
#include <cstring>
#include <list>
#include <map>
#include <memory>
#include <optional>
#include <set>
#include <stdexcept>
#include <string>
#include <unordered_map>
#include <vector>
#include "../../include/hbls.h"
#include "hbls_keyfile.hpp"

namespace harmony {
namespace bls_core {   // == github.com/harmony-one/bls/ffi/go/bls

constexpr int BLS12_381 = HBLS_BLS12_381;
inline int Init(int curve) { return blsInit(curve, HBLS_COMPILED_TIME_VAR); }

inline std::string hex(const uint8_t* p, size_t n) {
    static const char* d = "0123456789abcdef"; std::string s(2 * n, '0');
    for (size_t i = 0; i < n; i++) { s[2 * i] = d[p[i] >> 4]; s[2 * i + 1] = d[p[i] & 15]; }
    return s;
}
inline bool unhex(const std::string& s, std::vector<uint8_t>& out) {
    if (s.size() % 2) return false;
    out.resize(s.size() / 2);
    auto v = [](char c) -> int { return c >= '0' && c <= '9' ? c - '0' : c >= 'a' && c <= 'f' ? c - 'a' + 10 : c >= 'A' && c <= 'F' ? c - 'A' + 10 : -1; };
    for (size_t i = 0; i < out.size(); i++) { int a = v(s[2 * i]), b = v(s[2 * i + 1]); if (a < 0 || b < 0) return false; out[i] = (uint8_t)(a * 16 + b); }
    return true;
}

struct PublicKey;
struct Sign;

// plain value types: copyable, zero value = identity, no device handles (mask.go:50 copies *pubKey into the LRU)
struct PublicKey {
    blsPublicKey v{};
    std::vector<uint8_t> Serialize() const { std::vector<uint8_t> b(48); size_t n = blsPublicKeySerialize(b.data(), 48, &v); b.resize(n); return b; }
    bool Deserialize(const uint8_t* buf, size_t n) { return blsPublicKeyDeserialize(&v, buf, n) != 0; }          // Go: error != nil when false
    bool Deserialize(const std::vector<uint8_t>& b) { return Deserialize(b.data(), b.size()); }
    std::string SerializeToHexStr() const { auto b = Serialize(); return hex(b.data(), b.size()); }
    bool DeserializeHexStr(const std::string& s) { std::vector<uint8_t> b; return unhex(s, b) && Deserialize(b); }
    void Add(const PublicKey* rhs) { blsPublicKeyAdd(&v, &rhs->v); }
    void Sub(const PublicKey* rhs) { blsPublicKeySub(&v, &rhs->v); }
    bool IsEqual(const PublicKey* rhs) const { return blsPublicKeyIsEqual(&v, &rhs->v) == 1; }
    std::array<uint8_t, 20> GetAddress() const { std::array<uint8_t, 20> a{}; hbls_get_address(&v, a.data()); return a; }      // internal/utils/utils.go:77
};

struct Sign {
    blsSignature v{};
    std::vector<uint8_t> Serialize() const { std::vector<uint8_t> b(96); size_t n = blsSignatureSerialize(b.data(), 96, &v); b.resize(n); return b; }
    bool Deserialize(const uint8_t* buf, size_t n) { return blsSignatureDeserialize(&v, buf, n) != 0; }
    bool Deserialize(const std::vector<uint8_t>& b) { return Deserialize(b.data(), b.size()); }
    std::string SerializeToHexStr() const { auto b = Serialize(); return hex(b.data(), b.size()); }
    bool DeserializeHexStr(const std::string& s) { std::vector<uint8_t> b; return unhex(s, b) && Deserialize(b); }
    void Add(const Sign* rhs) { blsSignatureAdd(&v, &rhs->v); }
    bool VerifyHash(const PublicKey* pub, const std::vector<uint8_t>& h) const { return blsVerifyHash(&v, &pub->v, h.data(), h.size()) == 1; }
    bool Verify(const PublicKey* pub, const std::string& m) const { return blsVerify(&v, &pub->v, m.data(), m.size()) == 1; }
    bool IsEqual(const Sign* rhs) const { return blsSignatureIsEqual(&v, &rhs->v) == 1; }
};

struct SecretKey {
    blsSecretKey v{};
    void SetByCSPRNG() { if (blsSecretKeySetByCSPRNG(&v) != 0) throw std::runtime_error("err blsSecretKeySetByCSPRNG"); }
    PublicKey* GetPublicKey() const { auto* p = new PublicKey; blsGetPublicKey(&p->v, &v); return p; }
    // nil on failure, like the Go wrapper (callers test != nil: consensus/construct.go:101)
    Sign* SignHash(const std::vector<uint8_t>& h) const { auto* s = new Sign; if (blsSignHash(&s->v, &v, h.data(), h.size()) != 0) { delete s; return nullptr; } return s; }
    Sign* SignMsg(const std::string& m) const { auto* s = new Sign; blsSign(&s->v, &v, m.data(), m.size()); return s; }
    std::vector<uint8_t> Serialize() const { std::vector<uint8_t> b(32); blsSecretKeySerialize(b.data(), 32, &v); return b; }
    bool Deserialize(const std::vector<uint8_t>& b) { return blsSecretKeyDeserialize(&v, b.data(), b.size()) != 0; }
    std::string SerializeToHexStr() const { auto b = Serialize(); return hex(b.data(), b.size()); }
    bool DeserializeHexStr(const std::string& s) { std::vector<uint8_t> b; return unhex(s, b) && Deserialize(b); }
    bool IsEqual(const SecretKey* rhs) const { return blsSecretKeyIsEqual(&v, &rhs->v) == 1; }
};

}  // namespace bls_core

namespace bls {        // == github.com/harmony-one/harmony/crypto/bls

constexpr size_t PublicKeySizeInBytes = 48;
constexpr size_t BLSSignatureSizeInBytes = 96;
using SerializedPublicKey = std::array<uint8_t, PublicKeySizeInBytes>;
using SerializedSignature = std::array<uint8_t, BLSSignatureSizeInBytes>;

inline std::string Hex(const SerializedPublicKey& k) { return bls_core::hex(k.data(), k.size()); }
inline bool IsEmpty(const SerializedPublicKey& k) { for (auto b : k) if (b) return false; return true; }

struct PublicKeyWrapper {          // bls.go:30-33
    SerializedPublicKey Bytes{};
    std::shared_ptr<bls_core::PublicKey> Object;
    std::string Hex() const { return bls::Hex(Bytes); }
};
struct PrivateKeyWrapper {         // bls.go:24-27
    std::shared_ptr<bls_core::SecretKey> Pri;
    std::shared_ptr<PublicKeyWrapper> Pub;
};

// bls.go:109-118; false == the Go error "key size (BLS) size mismatch"
inline bool FromLibBLSPublicKey(SerializedPublicKey& pk, const bls_core::PublicKey* key) {
    auto b = key->Serialize();
    if (b.size() != pk.size()) return false;
    std::memcpy(pk.data(), b.data(), pk.size()); return true;
}
inline PrivateKeyWrapper WrapperFromPrivateKey(std::shared_ptr<bls_core::SecretKey> pri) {   // bls.go:41-52
    std::shared_ptr<bls_core::PublicKey> pub(pri->GetPublicKey());
    auto w = std::make_shared<PublicKeyWrapper>(); FromLibBLSPublicKey(w->Bytes, pub.get()); w->Object = pub;
    return PrivateKeyWrapper{pri, w};
}
inline std::shared_ptr<bls_core::SecretKey> RandPrivateKey() { auto s = std::make_shared<bls_core::SecretKey>(); s->SetByCSPRNG(); return s; }

// mask.go:35-55: LRU(1024) keyed by the raw bytes; returns nullptr + err string like the Go (nil, error)
class PubKeyCache {
    size_t cap_; std::list<std::pair<std::string, bls_core::PublicKey>> order_;
    std::unordered_map<std::string, decltype(order_)::iterator> idx_;
public:
    explicit PubKeyCache(size_t cap = 1024) : cap_(cap) {}
    bool Get(const std::string& k, bls_core::PublicKey& out) {
        auto it = idx_.find(k); if (it == idx_.end()) return false;
        order_.splice(order_.begin(), order_, it->second); out = it->second->second; return true;
    }
    void Add(const std::string& k, const bls_core::PublicKey& v) {
        auto it = idx_.find(k);
        if (it != idx_.end()) { it->second->second = v; order_.splice(order_.begin(), order_, it->second); return; }
        order_.emplace_front(k, v); idx_[k] = order_.begin();
        if (order_.size() > cap_) { idx_.erase(order_.back().first); order_.pop_back(); }
    }
    size_t Len() const { return order_.size(); }
};
inline PubKeyCache& BLSPubKeyCache() { static PubKeyCache c(1024); return c; }
inline std::shared_ptr<bls_core::PublicKey> BytesToBLSPublicKey(const std::vector<uint8_t>& bytes, std::string* err = nullptr) {
    if (bytes.empty()) { if (err) *err = "BytesToBLSPublicKey: empty input"; return nullptr; }
    std::string k(bytes.begin(), bytes.end());
    auto pk = std::make_shared<bls_core::PublicKey>();
    if (BLSPubKeyCache().Get(k, *pk)) return pk;
    if (!pk->Deserialize(bytes)) { if (err) *err = "err blsPublicKeyDeserialize"; return nullptr; }
    BLSPubKeyCache().Add(k, *pk);
    return pk;
}

// mask.go:58-64
inline std::shared_ptr<bls_core::Sign> AggregateSig(const std::vector<bls_core::Sign*>& sigs) {
    auto agg = std::make_shared<bls_core::Sign>();
    for (auto* s : sigs) agg->Add(s);
    return agg;
}
// bls.go:120-136
inline bool SeparateSigAndMask(const std::vector<uint8_t>& commitSigs, std::vector<uint8_t>& aggSig, std::vector<uint8_t>& bitmap) {
    if (commitSigs.size() < BLSSignatureSizeInBytes) return false;          // "no mask data found in commit sigs"
    aggSig.assign(commitSigs.begin(), commitSigs.begin() + 96); bitmap.assign(commitSigs.begin() + 96, commitSigs.end());
    return true;
}

// mask.go:67-242.  Methods return "" on success or the Go error string.
class Mask {
public:
    std::vector<uint8_t> Bitmap;
    std::vector<PublicKeyWrapper*> Publics;
    std::map<SerializedPublicKey, int> PublicsIndex;
    std::shared_ptr<bls_core::PublicKey> AggregatePublic;

    explicit Mask(std::vector<PublicKeyWrapper>& publics) {
        for (size_t i = 0; i < publics.size(); i++) { Publics.push_back(&publics[i]); PublicsIndex[publics[i].Bytes] = (int)i; }
        Bitmap.assign(Len(), 0); AggregatePublic = std::make_shared<bls_core::PublicKey>();
    }
    void Clear() { Bitmap.assign(Len(), 0); AggregatePublic = std::make_shared<bls_core::PublicKey>(); }
    std::vector<uint8_t> GetMask() const { return Bitmap; }
    int Len() const { return (int)((Publics.size() + 7) >> 3); }
    std::string SetMask(const std::vector<uint8_t>& mask) {
        if ((size_t)Len() != mask.size())
            return "mismatching bitmap lengths expectedBitmapLength " + std::to_string(Len()) + " providedBitmapLength " + std::to_string(mask.size());
        for (size_t i = 0; i < Publics.size(); i++) {
            size_t byt = i >> 3; uint8_t msk = (uint8_t)(1u << (i & 7));
            if ((Bitmap[byt] & msk) == 0 && (mask[byt] & msk) != 0) { Bitmap[byt] ^= msk; AggregatePublic->Add(Publics[i]->Object.get()); }
            if ((Bitmap[byt] & msk) != 0 && (mask[byt] & msk) == 0) { Bitmap[byt] ^= msk; AggregatePublic->Sub(Publics[i]->Object.get()); }
        }
        return "";
    }
    std::string SetBit(int i, bool enable) {
        if (i >= (int)Publics.size()) return "index out of range";
        size_t byt = (size_t)i >> 3; uint8_t msk = (uint8_t)(1u << (i & 7));
        if ((Bitmap[byt] & msk) == 0 && enable) { Bitmap[byt] ^= msk; AggregatePublic->Add(Publics[i]->Object.get()); }
        if ((Bitmap[byt] & msk) != 0 && !enable) { Bitmap[byt] ^= msk; AggregatePublic->Sub(Publics[i]->Object.get()); }
        return "";
    }
    std::vector<bls_core::PublicKey*> GetPubKeyFromMask(bool flag) const {
        std::vector<bls_core::PublicKey*> out;
        for (size_t i = 0; i < Publics.size(); i++) if (((Bitmap[i >> 3] >> (i & 7)) & 1) == (flag ? 1 : 0)) out.push_back(Publics[i]->Object.get());
        return out;
    }
    std::string GetSignedPubKeysFromBitmap(const std::vector<uint8_t>& bitmap, std::vector<PublicKeyWrapper*>& out) const {
        if ((size_t)Len() != bitmap.size())
            return "mismatching bitmap lengths expectedBitmapLength " + std::to_string(Len()) + " providedBitmapLength " + std::to_string(bitmap.size());
        for (size_t i = 0; i < Publics.size(); i++) if ((bitmap[i >> 3] >> (i & 7)) & 1) out.push_back(Publics[i]);
        return "";
    }
    std::string IndexEnabled(int i, bool& on) const { if (i >= (int)Publics.size()) return "index out of range"; on = (Bitmap[(size_t)i >> 3] >> (i & 7)) & 1; return ""; }
    std::string KeyEnabled(const SerializedPublicKey& k, bool& on) const { auto it = PublicsIndex.find(k); if (it == PublicsIndex.end()) return "key not found"; return IndexEnabled(it->second, on); }
    std::string SetKey(const SerializedPublicKey& k, bool enable) { auto it = PublicsIndex.find(k); if (it == PublicsIndex.end()) return "key not found"; return SetBit(it->second, enable); }
    std::string SetKeysAtomic(const std::vector<PublicKeyWrapper*>& publics, bool enable) {
        std::vector<int> idx;
        for (auto* k : publics) { auto it = PublicsIndex.find(k->Bytes); if (it == PublicsIndex.end()) return "key not found"; idx.push_back(it->second); }
        for (int i : idx) { auto e = SetBit(i, enable); if (!e.empty()) return e; }
        return "";
    }
    int CountEnabled() const { int hw = 0; for (size_t i = 0; i < Publics.size(); i++) hw += (Bitmap[i >> 3] >> (i & 7)) & 1; return hw; }
    int CountTotal() const { return (int)Publics.size(); }
};
inline std::unique_ptr<Mask> NewMask(std::vector<PublicKeyWrapper>& publics) { return std::make_unique<Mask>(publics); }
inline bool AggregateMasks(const std::vector<uint8_t>& a, const std::vector<uint8_t>& b, std::vector<uint8_t>& out) {
    if (a.size() != b.size()) return false;
    out.resize(a.size()); for (size_t i = 0; i < a.size(); i++) out[i] = a[i] | b[i];
    return true;
}
struct CompletePolicy { bool Check(const Mask& m) const { return m.CountEnabled() == m.CountTotal(); } };
struct ThresholdPolicy { int thold; bool Check(const Mask& m) const { return m.CountEnabled() >= thold; } };

// ---- device-resident committee + the BASELINE.json entry points (thin wrappers, SURVEY.md fact 3)
class Committee {
    hbls_committee* h_ = nullptr; size_t n_ = 0;
public:
    Committee() = default;
    Committee(const Committee&) = delete; Committee& operator=(const Committee&) = delete;
    ~Committee() { if (h_) hbls_committee_destroy(h_); }
    // returns "" or an error; bad_index = first undecodable key
    std::string Load(const std::vector<PublicKeyWrapper>& pubKeys, size_t* bad_index = nullptr) {
        std::vector<uint8_t> blob(pubKeys.size() * 48);
        for (size_t i = 0; i < pubKeys.size(); i++) std::memcpy(&blob[48 * i], pubKeys[i].Bytes.data(), 48);
        if (h_) { hbls_committee_destroy(h_); h_ = nullptr; }
        int rc = hbls_committee_create(&h_, blob.data(), pubKeys.size(), bad_index);
        if (rc == HBLS_ERR_DECODE) return "err blsPublicKeyDeserialize";
        if (rc != 0) return "hbls_committee_create failed";
        n_ = pubKeys.size(); return "";
    }
    size_t Size() const { return n_; }
    size_t BitmapLen() const { return (n_ + 7) >> 3; }
    const hbls_committee* handle() const { return h_; }
};
// running vote aggregate over a device-resident committee (hbls_ballot_box_*): the collected bitmap and the G2 sum of the collected
// signatures; each signature is decoded once, when its vote arrives (quorum.go:164-196 AggregateVotes re-decodes every ballot)
class BallotBox {
    hbls_ballot_box* h_ = nullptr; size_t blen_ = 0;
public:
    BallotBox() = default;
    BallotBox(const BallotBox&) = delete; BallotBox& operator=(const BallotBox&) = delete;
    ~BallotBox() { if (h_) hbls_ballot_box_destroy(h_); }
    std::string Create(const Committee& c) {
        if (h_) { hbls_ballot_box_destroy(h_); h_ = nullptr; }
        if (hbls_ballot_box_create(&h_, c.handle()) != 0) return "hbls_ballot_box_create failed";
        blen_ = c.BitmapLen(); return "";
    }
    size_t BitmapLen() const { return blen_; }
    // one ballot: 0 added, 1 skipped (a signer is already collected), HBLS_ERR_DECODE for an undecodable signature, < 0 error
    int AddVote(const std::vector<uint8_t>& signerBitmap, const std::vector<uint8_t>& sig96) {
        if (signerBitmap.size() != blen_ || sig96.size() != BLSSignatureSizeInBytes) return HBLS_ERR_ARG;
        return hbls_ballot_box_add_vote(h_, signerBitmap.data(), blen_, sig96.data());
    }
    // a leader's queue of k votes on msg (bitmaps: k * BitmapLen() bytes, sigs: 96 k): status[j] = HBLS_BALLOT_*; "" or the error
    std::string SubmitVotes(const std::vector<uint8_t>& bitmaps, const std::vector<uint8_t>& sigs, const std::vector<uint8_t>& msg, std::vector<uint8_t>& status) {
        const size_t k = sigs.size() / 96;
        if (sigs.size() != 96 * k || bitmaps.size() != k * blen_) return "vote queue: bitmap / signature sizes do not match";
        status.assign(k, 0);
        const int rc = hbls_ballot_box_submit_votes(h_, k, bitmaps.data(), blen_, sigs.data(), msg.data(), msg.size(), status.data());
        return rc == 0 ? "" : rc == HBLS_ERR_ARG ? "hbls_ballot_box_submit_votes: bad argument" : "hbls_ballot_box_submit_votes failed";
    }
    // aggregate signature of the collected ballots and their bitmap (construct.go:158-175)
    bool Aggregate(std::vector<uint8_t>& sig96, std::vector<uint8_t>& bitmap) const {
        sig96.assign(96, 0); bitmap.assign(blen_, 0);
        return hbls_ballot_box_aggregate(h_, sig96.data(), bitmap.data(), blen_) == 0;
    }
};
// batch entry points test large batches in random-linear-combination groups first (exact fallback); exactOnly forces the per-round algorithm
inline void SetBatchMode(bool exactOnly) { hbls_set_batch_mode(exactOnly ? 0 : 1); }
// == NewMask(pubKeys).SetMask(bitmap) ; aggSig.Deserialize ; aggSig.VerifyHash(mask.AggregatePublic, msg)
inline int FastAggregateVerify(const Committee& c, const std::vector<uint8_t>& bitmap, const SerializedSignature& sig, const std::vector<uint8_t>& msg) {
    return hbls_aggregate_verify(c.handle(), bitmap.data(), bitmap.size(), sig.data(), msg.data(), msg.size());
}
inline int VerifyAggregateSig(const Committee& c, const std::vector<uint8_t>& bitmap, const SerializedSignature& sig, const std::vector<uint8_t>& msg) {
    return FastAggregateVerify(c, bitmap, sig, msg);
}

}  // namespace bls

namespace multibls {   // == multibls/multibls.go
struct PublicKeys : std::vector<bls::PublicKeyWrapper> {
    std::string SerializeToHexStr() const { std::string s; for (auto& k : *this) s += k.Hex() + ";"; return s; }
    bool Contains(const bls_core::PublicKey* pk) const { for (auto& k : *this) if (k.Object->IsEqual(pk)) return true; return false; }
};
struct PrivateKeys : std::vector<bls::PrivateKeyWrapper> {
    PublicKeys GetPublicKeys() const { PublicKeys out; for (auto& k : *this) out.push_back(*k.Pub); return out; }
    PrivateKeys Dedup() const {
        std::set<bls::SerializedPublicKey> seen; PrivateKeys out;
        for (auto& k : *this) { if (seen.count(k.Pub->Bytes)) continue; seen.insert(k.Pub->Bytes); out.push_back(k); }
        return out;
    }
};
inline PrivateKeys GetPrivateKeys(const std::vector<std::shared_ptr<bls_core::SecretKey>>& secretKeys) {
    PrivateKeys keys; for (auto& s : secretKeys) keys.push_back(bls::WrapperFromPrivateKey(s)); return keys;
}
}  // namespace multibls

namespace signature {  // == consensus/signature/signature.go:12-24
inline std::vector<uint8_t> ConstructCommitPayload(bool isStaking, const std::array<uint8_t, 32>& blockHash, uint64_t blockNum, uint64_t viewID) {
    std::vector<uint8_t> p(8);
    for (int i = 0; i < 8; i++) p[i] = (uint8_t)(blockNum >> (8 * i));
    p.insert(p.end(), blockHash.begin(), blockHash.end());
    if (!isStaking) return p;
    for (int i = 0; i < 8; i++) p.push_back((uint8_t)(viewID >> (8 * i)));
    return p;
}
}  // namespace signature

namespace chain {      // == internal/chain/sig.go, engine.go:606-642
inline bool ParseCommitSigAndBitmap(const std::vector<uint8_t>& payload, bls::SerializedSignature& sig, std::vector<uint8_t>& bitmap) {
    if (payload.size() < bls::BLSSignatureSizeInBytes) return false;        // "payload not have enough length"
    std::memcpy(sig.data(), payload.data(), 96); bitmap.assign(payload.begin() + 96, payload.end()); return true;
}
// sig.go:37-49; "" or the Go error string
inline std::string DecodeSigBitmap(const bls::SerializedSignature& sigBytes, const std::vector<uint8_t>& bitmap, std::vector<bls::PublicKeyWrapper>& pubKeys,
                                   std::shared_ptr<bls_core::Sign>& aggSig, std::unique_ptr<bls::Mask>& mask) {
    aggSig = std::make_shared<bls_core::Sign>();
    if (!aggSig->Deserialize(sigBytes.data(), sigBytes.size())) return "unable to deserialize multi-signature from payload";
    mask = bls::NewMask(pubKeys);
    if (!mask->SetMask(bitmap).empty()) return "mask.SetMask failed";
    return "";
}
}  // namespace chain

namespace quorum {     // == consensus/quorum, uniform (one-node-one-vote) policy + ballot aggregation
inline int64_t TwoThirdsSignersCount(int64_t participants) { return participants * 2 / 3 + 1; }       // quorum.go:409-411
inline int64_t CountOneBits(const std::vector<uint8_t>& bm) { int64_t c = 0; for (uint8_t b : bm) c += __builtin_popcount(b); return c; }
// Set bits among the committee's n slots only.  The reference counts mask.Bitmap AFTER SetMask, which never sets a bit i >= n
// (crypto/bls/mask.go:121-133), so the padding bits of the last byte of a RAW header bitmap must not count: with n = 250 an
// attacker could otherwise add 6 phantom votes and pass the 167 threshold with 161 real signers.
inline int64_t CountSlotBits(const std::vector<uint8_t>& bm, size_t n) {
    int64_t c = 0;
    for (size_t i = 0; i < (n >> 3) && i < bm.size(); i++) c += __builtin_popcount(bm[i]);
    if ((n & 7) && (n >> 3) < bm.size()) c += __builtin_popcount(bm[n >> 3] & ((1u << (n & 7)) - 1u));
    return c;
}
inline bool IsQuorumAchievedByMask(const bls::Mask* mask, int64_t participants) {                      // one-node-one-vote.go:57-72
    if (!mask) return false;
    return CountOneBits(mask->Bitmap) >= TwoThirdsSignersCount(participants);                          // Mask.Bitmap never holds padding bits
}
struct Ballot { std::vector<bls::SerializedPublicKey> SignerPubKeys; std::vector<uint8_t> Signature; };
// quorum.go:164-196: skip ballots sharing a signer with an already collected ballot, re-decode each stored signature, fold Add.
// The decode + sum runs as ONE device call (hbls_aggregate_sigs) instead of n cgo round trips.
inline std::shared_ptr<bls_core::Sign> AggregateVotes(const std::vector<Ballot>& ballots) {
    std::set<bls::SerializedPublicKey> collected; std::vector<uint8_t> blob; size_t n = 0;
    for (auto& b : ballots) {
        bool dup = false; for (auto& k : b.SignerPubKeys) if (collected.count(k)) { dup = true; break; }
        if (dup) continue;
        for (auto& k : b.SignerPubKeys) collected.insert(k);
        if (b.Signature.size() != 96) continue;
        blob.insert(blob.end(), b.Signature.begin(), b.Signature.end()); n++;
    }
    uint8_t out[96];
    auto agg = std::make_shared<bls_core::Sign>();
    if (hbls_aggregate_sigs(blob.data(), n, out) != 0) return agg;
    agg->Deserialize(out, 96);
    return agg;
}
}  // namespace quorum

namespace chain {
inline const char* headerStatusError(uint8_t st) {          // the Go error strings of engine.go:619-642 / sig.go:37-49
    switch (st) {
    case HBLS_HDR_OK: return "";
    case HBLS_HDR_BAD_ENCODING: return "deserialize signature and bitmap: unable to deserialize multi-signature from payload";
    case HBLS_HDR_NO_QUORUM: return "not enough signature collected";
    default: return "Unable to verify aggregated signature for block";
    }
}
// engine.go:619-642 over a device-resident committee, with the 100-entry verified-signature cache of engine.go:606-617
class SignatureVerifier {
    std::list<std::string> order_; std::set<std::string> seen_; size_t cap_;
public:
    explicit SignatureVerifier(size_t cap = 100) : cap_(cap) {}
    // "" on success or the Go error string.  Order of checks as in engine.go:630-640: DecodeSigBitmap (signature deserialise,
    // SetMask length) -> IsQuorumAchievedByMask over the committee's slots -> VerifyHash; one device call (hbls_verify_headers, n = 1).
    std::string verifySignature(const bls::Committee& ec, const bls::SerializedSignature& commitSig, const std::vector<uint8_t>& commitBitmap,
                                const std::vector<uint8_t>& commitPayload) {
        if (commitBitmap.size() != ec.BitmapLen()) return "deserialize signature and bitmap: mask.SetMask failed";
        uint8_t st = 0;
        int rc = hbls_verify_headers(ec.handle(), 1, commitSig.data(), commitBitmap.data(), commitBitmap.size(), commitPayload.data(), commitPayload.size(),
                                     (size_t)quorum::TwoThirdsSignersCount((int64_t)ec.Size()), &st);
        if (rc != 0) return "deserialize signature and bitmap";
        return headerStatusError(st);
    }
    std::string verifySignatureCached(const bls::Committee& ec, const std::array<uint8_t, 32>& blockHash, const bls::SerializedSignature& sig,
                                      const std::vector<uint8_t>& bitmap, const std::vector<uint8_t>& payload) {
        std::string key(blockHash.begin(), blockHash.end()); key.append(sig.begin(), sig.end()); key.append(bitmap.begin(), bitmap.end());
        if (seen_.count(key)) return "";
        auto e = verifySignature(ec, sig, bitmap, payload);
        if (!e.empty()) return e;
        seen_.insert(key); order_.push_back(key);
        if (order_.size() > cap_) { seen_.erase(order_.front()); order_.pop_front(); }
        return "";
    }
};

// ---- range form (SURVEY 8f.1): engine.go:81-97 VerifyHeaders / stagedstreamsync/sig_verify.go:23-58 verify one header
// signature per cgo round trip; here the block range of ONE committee epoch goes to the device in one call (hbls_verify_headers).
struct HeaderSig {
    bls::SerializedSignature commitSig; std::vector<uint8_t> commitBitmap; std::vector<uint8_t> commitPayload;   // payload = ConstructCommitPayload(...)
};
struct HeaderBatch {          // what hbls_verify_headers consumes: same-length payloads, well-formed bitmaps
    size_t msgLen = 0; std::vector<size_t> index; std::vector<uint8_t> bitmaps, sigs, msgs;
    size_t rounds() const { return index.size(); }
};
// Pure host step (no device): rejects malformed records (bitmap length: sig.go:43 mask.SetMask error; empty payload) and packs the
// rest by payload length (40 B pre-staking / 48 B staking eras never mix inside one call).  Quorum and signature checks happen in
// hbls_verify_headers, in the reference's order.
inline std::vector<HeaderBatch> AssembleHeaderBatches(size_t committeeSize, const std::vector<HeaderSig>& headers, std::vector<std::string>& errs) {
    const size_t blen = (committeeSize + 7) >> 3;
    errs.assign(headers.size(), "");
    std::vector<HeaderBatch> out;
    for (size_t i = 0; i < headers.size(); i++) {
        const HeaderSig& h = headers[i];
        if (h.commitBitmap.size() != blen) { errs[i] = "deserialize signature and bitmap: mask.SetMask failed"; continue; }
        if (h.commitPayload.empty()) { errs[i] = "invalid commit payload"; continue; }
        HeaderBatch* b = nullptr;
        for (auto& c : out) if (c.msgLen == h.commitPayload.size()) { b = &c; break; }
        if (!b) { out.emplace_back(); b = &out.back(); b->msgLen = h.commitPayload.size(); }
        b->index.push_back(i);
        b->bitmaps.insert(b->bitmaps.end(), h.commitBitmap.begin(), h.commitBitmap.end());
        b->sigs.insert(b->sigs.end(), h.commitSig.begin(), h.commitSig.end());
        b->msgs.insert(b->msgs.end(), h.commitPayload.begin(), h.commitPayload.end());
    }
    return out;
}
// errs[i] == "" iff header i carries a valid quorum signature of the committee (same strings as verifySignature above)
inline std::vector<std::string> VerifyHeaderSignatures(const bls::Committee& ec, const std::vector<HeaderSig>& headers) {
    std::vector<std::string> errs;
    const size_t quorum = (size_t)quorum::TwoThirdsSignersCount((int64_t)ec.Size());
    for (auto& b : AssembleHeaderBatches(ec.Size(), headers, errs)) {
        std::vector<uint8_t> st(b.rounds(), 0);
        int rc = hbls_verify_headers(ec.handle(), b.rounds(), b.sigs.data(), b.bitmaps.data(), ec.BitmapLen(), b.msgs.data(), b.msgLen, quorum, st.data());
        for (size_t k = 0; k < b.rounds(); k++) errs[b.index[k]] = rc != 0 ? "deserialize signature and bitmap" : headerStatusError(st[k]);
    }
    return errs;
}
}  // namespace chain
namespace blsgen {     // == internal/blsgen/lib.go (key files; codec in hbls_keyfile.hpp)
// LoadBLSKeyWithPassPhrase (lib.go:51-71) on the file's content: nullptr + err on a wrong passphrase / damaged file / bad key
inline std::shared_ptr<bls_core::SecretKey> LoadBLSKeyWithPassPhrase(const std::string& fileName, const std::string& fileContent, const std::string& passphrase, std::string* err = nullptr) {
    std::string skHex;
    if (!LoadBLSKeyHexWithPassPhrase(fileContent, passphrase, skHex, err)) return nullptr;
    auto sk = std::make_shared<bls_core::SecretKey>();
    if (!sk->DeserializeHexStr(skHex)) { if (err) *err = "could not deserialize byte content of " + fileName + " as BLS secret key"; return nullptr; }
    return sk;
}
// GenBLSKeyWithPassPhrase's file (lib.go:20-34): name = hex(pk) + ".key", content = encrypt(hex(sk), passphrase)
inline std::pair<std::string, std::string> KeyFileFor(const bls_core::SecretKey& sk, const std::string& passphrase, const uint8_t nonce[12]) {
    std::unique_ptr<bls_core::PublicKey> pk(sk.GetPublicKey());
    return {pk->SerializeToHexStr() + ".key", encrypt(sk.SerializeToHexStr(), passphrase, nonce)};
}
}  // namespace blsgen

}  // namespace harmony
