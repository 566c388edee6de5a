// harmony_b200/host/hbls_host_test.cpp -- the reference's own host-level tests restated on the C++ mirror
// (hbls_host.hpp) over libhbls.so.  Needs a GPU (every group operation is a kernel).  Exit code 0 = all passed.
//   crypto/bls/mask_test.go            TestNewMask, TestSetMask/SetBit/SetKey/SetKeysAtomic, TestCountEnabled, policies
//   consensus/quorum/quorom_test.go    TestSubmitVote (:73-125, AggregateVotes == manual Add chain),
//                                      TestAddNewVoteInvalidAggregateSig (:381-501), TestInvalidAggregateSig (:503-552)
//   consensus/signature/signature_test.go, internal/chain/sig.go + engine.go:619-642
//   consensus message signatures (consensus_service.go:115-119, checks.go:20-56) incl. the reference's signature vector, and a small
//   view-change storm + NEWVIEW (view_change_construct.go:154-375, view_change.go:445-500) through hbls_consensus.hpp
#include <cstdio>
#include <cstdlib>
#include "hbls_host.hpp"
#include "hbls_consensus.hpp"

using namespace harmony;
static int g_fail = 0;
#define CHECK(c) do { if (!(c)) { fprintf(stderr, "CHECK FAILED %s:%d: %s\n", __FILE__, __LINE__, #c); g_fail++; } } while (0)

static std::vector<bls::PrivateKeyWrapper> make_keys(int n) {
    std::vector<bls::PrivateKeyWrapper> v;
    for (int i = 0; i < n; i++) v.push_back(bls::WrapperFromPrivateKey(bls::RandPrivateKey()));
    return v;
}

static void test_mask() {
    auto keys = make_keys(9);
    std::vector<bls::PublicKeyWrapper> pubs; for (auto& k : keys) pubs.push_back(*k.Pub);
    auto m = bls::NewMask(pubs);
    CHECK(m->Len() == 2 && m->CountTotal() == 9 && m->CountEnabled() == 0);
    CHECK(!m->SetMask({0x01}).empty());                                   // mismatching bitmap lengths
    CHECK(m->SetBit(0, true).empty()); CHECK(m->SetKey(pubs[8].Bytes, true).empty());
    CHECK(m->GetMask() == std::vector<uint8_t>({0x01, 0x01}) && m->CountEnabled() == 2);
    bls_core::PublicKey exp; exp.Add(pubs[0].Object.get()); exp.Add(pubs[8].Object.get());
    CHECK(m->AggregatePublic->IsEqual(&exp));
    CHECK(m->SetBit(9, true) == "index out of range");
    bls::SerializedPublicKey zero{}; CHECK(m->SetKey(zero, true) == "key not found");
    CHECK(m->SetKeysAtomic({&pubs[1], &pubs[2]}, true).empty());
    bool on = false; CHECK(m->IndexEnabled(1, on).empty() && on); CHECK(m->KeyEnabled(pubs[2].Bytes, on).empty() && on);
    CHECK(m->IndexEnabled(3, on).empty() && !on);
    m->SetBit(0, false); m->SetBit(8, false); m->SetKeysAtomic({&pubs[1], &pubs[2]}, false);
    bls_core::PublicKey id; CHECK(m->AggregatePublic->IsEqual(&id) && m->CountEnabled() == 0);
    CHECK(m->AggregatePublic->Serialize() == std::vector<uint8_t>(48, 0));
    CHECK(!bls::ThresholdPolicy{1}.Check(*m) && !bls::CompletePolicy{}.Check(*m));
    CHECK(m->SetMask({0xff, 0x01}).empty() && bls::CompletePolicy{}.Check(*m));
    CHECK(m->GetPubKeyFromMask(true).size() == 9 && m->GetPubKeyFromMask(false).empty());
    std::vector<uint8_t> o; CHECK(bls::AggregateMasks({1, 2}, {0x10, 2}, o) && o == std::vector<uint8_t>({0x11, 2}));
}

static void test_quorum_votes() {
    auto keys = make_keys(8);
    std::vector<bls::PublicKeyWrapper> pubs; for (auto& k : keys) pubs.push_back(*k.Pub);
    std::vector<uint8_t> hash(32); for (int i = 0; i < 32; i++) hash[i] = (uint8_t)(i * 7 + 1);
    std::vector<std::unique_ptr<bls_core::Sign>> sigs;
    for (auto& k : keys) { sigs.emplace_back(k.Pri->SignHash(hash)); CHECK(sigs.back() != nullptr); }
    // TestSubmitVote: AggregateVotes == manual Add chain (serialised equality)
    std::vector<quorum::Ballot> ballots;
    for (int i = 0; i < 3; i++) ballots.push_back({{pubs[i].Bytes}, sigs[i]->Serialize()});
    ballots.push_back({{pubs[1].Bytes}, sigs[1]->Serialize()});           // duplicate signer ballot is skipped
    auto agg = quorum::AggregateVotes(ballots);
    bls_core::Sign manual; for (int i = 0; i < 3; i++) manual.Add(sigs[i].get());
    CHECK(agg->SerializeToHexStr() == manual.SerializeToHexStr());
    // 4-of-8 aggregate verifies against the 4-signer mask (quorom_test.go:465-472)
    auto a4 = bls::AggregateSig({sigs[0].get(), sigs[1].get(), sigs[2].get(), sigs[3].get()});
    auto mask = bls::NewMask(pubs); CHECK(mask->SetMask({0x0f}).empty());
    CHECK(a4->VerifyHash(mask->AggregatePublic.get(), hash));
    CHECK(!quorum::IsQuorumAchievedByMask(mask.get(), 8));                // 4 < 8*2/3+1 = 6
    CHECK(mask->SetMask({0x3f}).empty() && quorum::IsQuorumAchievedByMask(mask.get(), 8));
    CHECK(!a4->VerifyHash(mask->AggregatePublic.get(), hash));
    // TestInvalidAggregateSig: duplicated signer fails against the de-duplicated key, correct set verifies
    auto dup = bls::AggregateSig({sigs[0].get(), sigs[1].get(), sigs[1].get()});
    bls_core::PublicKey apk; apk.Add(pubs[0].Object.get()); apk.Add(pubs[1].Object.get());
    CHECK(!dup->VerifyHash(&apk, hash));
    auto okk = bls::AggregateSig({sigs[0].get(), sigs[1].get()});
    CHECK(okk->VerifyHash(&apk, hash));
    // engine.go:619-642 through the device-resident committee; sig.go helpers
    bls::Committee com; CHECK(com.Load(pubs).empty());
    auto a6 = bls::AggregateSig({sigs[0].get(), sigs[1].get(), sigs[2].get(), sigs[3].get(), sigs[4].get(), sigs[5].get()});
    std::vector<uint8_t> payload = a6->Serialize(); payload.push_back(0x3f);
    bls::SerializedSignature s96; std::vector<uint8_t> bitmap;
    CHECK(chain::ParseCommitSigAndBitmap(payload, s96, bitmap) && bitmap == std::vector<uint8_t>({0x3f}));
    chain::SignatureVerifier eng;
    std::array<uint8_t, 32> bh; std::copy(hash.begin(), hash.end(), bh.begin());
    CHECK(eng.verifySignatureCached(com, bh, s96, bitmap, hash).empty());
    CHECK(eng.verifySignatureCached(com, bh, s96, bitmap, hash).empty());                       // cache hit
    CHECK(eng.verifySignature(com, s96, {0x0f}, hash) == "not enough signature collected");
    CHECK(eng.verifySignature(com, s96, {0x7e}, hash) == "Unable to verify aggregated signature for block");
    CHECK(!eng.verifySignature(com, s96, {0x3f, 0x00}, hash).empty());
    std::shared_ptr<bls_core::Sign> dsig; std::unique_ptr<bls::Mask> dmask;
    CHECK(chain::DecodeSigBitmap(s96, bitmap, pubs, dsig, dmask).empty() && dsig->VerifyHash(dmask->AggregatePublic.get(), hash));
    CHECK(chain::DecodeSigBitmap(s96, {0x3f, 0x00}, pubs, dsig, dmask) == "mask.SetMask failed");
    CHECK(bls::FastAggregateVerify(com, bitmap, s96, hash) == 1 && bls::VerifyAggregateSig(com, {0x1f}, s96, hash) == 0);
    // padding bits are not votes: 6-key committee (1-byte bitmap, quorum 5).  4 real signers + the two padding bits give a raw
    // popcount of 6, and the aggregate of the 4 verifies -- the reference counts mask.Bitmap after SetMask (4 < 5) and rejects.
    {
        std::vector<bls::PublicKeyWrapper> six(pubs.begin(), pubs.begin() + 6);
        bls::Committee c6; CHECK(c6.Load(six).empty());
        bls::SerializedSignature s4; auto b4 = a4->Serialize(); std::copy(b4.begin(), b4.end(), s4.begin());
        CHECK(bls::FastAggregateVerify(c6, {0xcf}, s4, hash) == 1);                               // the device ignores the padding bits
        CHECK(eng.verifySignature(c6, s4, {0xcf}, hash) == "not enough signature collected");
        CHECK(eng.verifySignature(c6, s4, {0x0f}, hash) == "not enough signature collected");
        // header range: valid / below quorum (padding attack) / wrong payload / undecodable signature / valid
        bls::SerializedSignature s6; auto b6 = a6->Serialize(); std::copy(b6.begin(), b6.end(), s6.begin());
        std::vector<chain::HeaderSig> hs(5);
        for (auto& x : hs) { x.commitSig = s6; x.commitBitmap = {0x3f}; x.commitPayload = hash; }
        hs[1].commitSig = s4; hs[1].commitBitmap = {0xcf};
        hs[2].commitPayload[3] ^= 1;
        hs[3].commitSig.fill(0xff);
        auto errs = chain::VerifyHeaderSignatures(c6, hs);
        CHECK(errs[0].empty() && errs[4].empty());
        CHECK(errs[1] == "not enough signature collected");
        CHECK(errs[2] == "Unable to verify aggregated signature for block");
        CHECK(errs[3] == "deserialize signature and bitmap: unable to deserialize multi-signature from payload");
    }
    // GetAddress (internal/utils/utils.go:77): 20 bytes, deterministic, differs between keys
    CHECK(pubs[0].Object->GetAddress() == pubs[0].Object->GetAddress() && pubs[0].Object->GetAddress() != pubs[1].Object->GetAddress());
}

static void test_codecs_multibls_payload() {
    // core/tx_pool_test.go:52-53 golden pair
    bls_core::SecretKey sk; CHECK(sk.DeserializeHexStr("c6d7603520311f7a4e6aac0b26701fc433b75b38df504cd416ef2b900cd66205"));
    std::unique_ptr<bls_core::PublicKey> pk(sk.GetPublicKey());
    CHECK(pk->SerializeToHexStr() == "30b2c38b1316da91e068ac3bd8751c0901ef6c02a1d58bc712104918302c6ed03d5894671d0c816dad2b4d303320f202");
    std::string err; auto viaCache = bls::BytesToBLSPublicKey(pk->Serialize(), &err);
    CHECK(viaCache && viaCache->IsEqual(pk.get()) && bls::BLSPubKeyCache().Len() >= 1);
    CHECK(bls::BytesToBLSPublicKey({}, &err) == nullptr && err == "BytesToBLSPublicKey: empty input");
    CHECK(bls::BytesToBLSPublicKey(std::vector<uint8_t>(48, 0xff), &err) == nullptr);
    auto s1 = bls::RandPrivateKey(), s2 = bls::RandPrivateKey();
    auto mk = multibls::GetPrivateKeys({s1, s2, s1});
    CHECK(mk.size() == 3 && mk.Dedup().size() == 2);
    auto pubs = mk.GetPublicKeys(); CHECK(pubs.Contains(mk[1].Pub->Object.get()));
    std::unique_ptr<bls_core::PublicKey> other(bls::RandPrivateKey()->GetPublicKey()); CHECK(!pubs.Contains(other.get()));
    CHECK(pubs.SerializeToHexStr() == mk[0].Pub->Hex() + ";" + mk[1].Pub->Hex() + ";" + mk[2].Pub->Hex() + ";");
    std::array<uint8_t, 32> h; for (int i = 0; i < 32; i++) h[i] = (uint8_t)i;
    auto p = signature::ConstructCommitPayload(true, h, 0x0102030405060708ull, 0x1112131415161718ull);
    CHECK(p.size() == 48 && p[0] == 8 && p[7] == 1 && p[8] == 0 && p[39] == 31 && p[40] == 0x18 && p[47] == 0x11);
    CHECK(signature::ConstructCommitPayload(false, h, 1, 2).size() == 40);
    std::vector<uint8_t> a, b; CHECK(!bls::SeparateSigAndMask(std::vector<uint8_t>(95), a, b));
    CHECK(bls::SeparateSigAndMask(std::vector<uint8_t>(100, 7), a, b) && a.size() == 96 && b.size() == 4);
    // string Sign/Verify round trip (consensus/quorum/quorom_test.go:97-121 style)
    std::unique_ptr<bls_core::Sign> sg(s1->SignMsg("test")); std::unique_ptr<bls_core::PublicKey> p1(s1->GetPublicKey());
    CHECK(sg->Verify(p1.get(), "test") && !sg->Verify(p1.get(), "tesT"));
    // SignHash returns nil when the message maps to no point (t = 0)
    CHECK(s1->SignHash(std::vector<uint8_t>(8, 0)) == nullptr);
}

static consensus::Bytes sign_bytes(const bls::PrivateKeyWrapper& k, const consensus::Bytes& m) {
    std::unique_ptr<bls_core::Sign> s(k.Pri->SignHash(m)); return s ? s->Serialize() : consensus::Bytes();
}
static void test_consensus_messages() {
    using namespace consensus;
    // the reference's only (sk, message) -> signature vector is signMessage("harmony-one") (staking/types/validator.go:30,525-527;
    // rosetta/services/construction_create_test.go:460-467)
    bls_core::SecretKey sk; CHECK(sk.DeserializeHexStr("c6d7603520311f7a4e6aac0b26701fc433b75b38df504cd416ef2b900cd66205"));
    const std::string m0 = "harmony-one"; const Bytes msg(m0.begin(), m0.end());
    const Bytes sig = signMessage(msg, &sk);
    CHECK(bls_core::hex(sig.data(), sig.size()) == "68f800b6adf657b674903e04708060912b893b7c7b500788808247550ab3e186e56a44ebf3ca488f8ed1a42f6cef3a04bd5d2b2b7eb5a767848d3135b362e668ce6bba42c7b9d5666d8e3a83be707b5708e722c58939fe9b07c170f3b7062414");
    std::unique_ptr<bls_core::PublicKey> pk(sk.GetPublicKey());
    CHECK(verifyMessageSig(pk.get(), msg, sig).empty());
    Bytes other = msg; other[0] ^= 1;
    CHECK(verifyMessageSig(pk.get(), other, sig) == errMsgSig && verifyMessageSig(pk.get(), msg, Bytes(96, 0xff)) == errSigDeserialize);
    auto errs = verifyMessageSigBatch({pk->Serialize(), pk->Serialize(), Bytes(48, 0xff), pk->Serialize(), pk->Serialize()}, {msg, other, msg, msg, msg},
                                      {sig, sig, sig, Bytes(96, 0xff), Bytes(50, 1)});
    CHECK(errs[0].empty() && errs[1] == errMsgSig && errs[2] == errKeyDeserialize && errs[3] == errSigDeserialize && errs[4] == errSigDeserialize);

    // view-change storm on a 7-validator committee (quorum 5)
    auto keys = make_keys(7);
    std::vector<bls::PublicKeyWrapper> pubs; for (auto& k : keys) pubs.push_back(*k.Pub);
    const uint64_t viewID = 41;
    Bytes bh(32); for (int i = 0; i < 32; i++) bh[i] = (uint8_t)(3 * i + 5);
    auto proof = [&](int signers, uint8_t bitmap) {
        std::vector<std::unique_ptr<bls_core::Sign>> ss; std::vector<bls_core::Sign*> ptr;
        for (int i = 0; i < signers; i++) { ss.emplace_back(keys[i].Pri->SignHash(bh)); ptr.push_back(ss.back().get()); }
        Bytes p = bh; auto a = bls::AggregateSig(ptr)->Serialize(); p.insert(p.end(), a.begin(), a.end()); p.push_back(bitmap); return p;
    };
    const Bytes payload = proof(5, 0x1f), low = proof(4, 0x0f);
    auto vcmsg = [&](int i, bool m1, const Bytes& pl) {
        FBFTMessage m; m.ViewID = viewID; m.BlockNum = 9; m.SenderPubkey = Bytes(pubs[i].Bytes.begin(), pubs[i].Bytes.end()); m.LeaderPubkey = m.SenderPubkey;
        if (m1) { m.Payload = pl; m.Block = {0xc0}; m.ViewchangeSig = sign_bytes(keys[i], pl); } else m.ViewchangeSig = sign_bytes(keys[i], NIL());
        m.ViewidSig = sign_bytes(keys[i], le64(viewID)); return m;
    };
    std::vector<FBFTMessage> storm = {vcmsg(0, true, payload), vcmsg(1, true, payload), vcmsg(2, true, payload), vcmsg(3, false, {}), vcmsg(4, false, {}),
                                      vcmsg(5, false, {}), vcmsg(6, true, low), vcmsg(0, true, payload), vcmsg(5, false, {})};
    storm[5].ViewchangeSig = sign_bytes(keys[5], Bytes{0x02});                         // signed 0x02, not NIL
    storm[8].ViewidSig = sign_bytes(keys[5], le64(viewID + 1));                        // signed another view
    viewChange vc; CHECK(vc.Init(pubs).empty());
    const uint64_t l0 = hbls_kernel_launch_count();
    auto out = vc.ProcessViewChangeMsgs(storm);
    CHECK(hbls_kernel_launch_count() > l0);
    for (int i = 0; i < 5; i++) CHECK(out[i].empty());
    CHECK(out[5] == errVerifyM2 && out[6] == errNoQuorum && out[7] == errDupM3 && out[8] == errViewIDSig);
    CHECK(vc.m1Payload == payload && vc.bhpBitmap[viewID] == Bytes{0x07} && vc.nilBitmap[viewID] == Bytes{0x18} && vc.viewIDBitmap[viewID] == Bytes{0x1f});
    // a decider with its own quorum rule (staked vote) accepts the 4-of-7 proof
    viewChange vc2; CHECK(vc2.Init(pubs).empty()); vc2.isQuorumAchievedByMask = [](const Bytes& bm) { return quorum::CountSlotBits(bm, 7) >= 4; };
    CHECK(vc2.ProcessViewChangeMsg(storm[6]).empty());
    // NEWVIEW from what the storm collected
    Bytes m2s, m2b, m3s, m3b; CHECK(vc.GetM2Bitmap(viewID, m2s, m2b) && vc.GetM3Bitmap(viewID, m3s, m3b) && m2b == Bytes{0x18} && m3b == Bytes{0x1f});
    CHECK(!vc.GetM2Bitmap(viewID + 1, m2s, m2b)); CHECK(vc.GetM2Bitmap(viewID, m2s, m2b));
    { bls_core::Sign manual; for (int i = 0; i < 5; i++) { bls_core::Sign s; CHECK(s.Deserialize(storm[i].ViewidSig)); manual.Add(&s); } CHECK(manual.Serialize() == m3s); }
    // both aggregates in one batch call, and the batch entry itself on sets with an empty one and an undecodable signature
    { Bytes s2, b2, s3, b3; const uint64_t l1 = hbls_kernel_launch_count();
      CHECK(vc.GetM2M3Bitmaps(viewID, s2, b2, s3, b3) == std::make_pair(true, true) && s2 == m2s && b2 == m2b && s3 == m3s && b3 == m3b);
      const uint64_t one_call = hbls_kernel_launch_count() - l1;
      CHECK(vc.GetM2M3Bitmaps(viewID + 1, s2, b2, s3, b3) == std::make_pair(false, false) && s2.empty() && b3.empty());
      CHECK(hbls_kernel_launch_count() - l1 == one_call);                            // nobody signed: no device call
      std::vector<Bytes> aggs;
      const auto st = bls::AggregateSigBatch({{storm[0].ViewidSig, storm[1].ViewidSig}, {}, {storm[0].ViewidSig, Bytes(96, 0xff)}}, aggs);
      bls_core::Sign ident; const Bytes id96 = ident.Serialize();
      CHECK(st == (std::vector<uint8_t>{HBLS_AGG_OK, HBLS_AGG_OK, HBLS_AGG_BAD_SIG_ENCODING}) && aggs.size() == 3 && aggs[1] == id96 && aggs[2] == id96);
      bls_core::Sign two; for (int i = 0; i < 2; i++) { bls_core::Sign s; CHECK(s.Deserialize(storm[i].ViewidSig)); two.Add(&s); }
      CHECK(aggs[0] == two.Serialize()); }
    FBFTMessage nv; nv.ViewID = viewID; nv.BlockNum = 9; nv.SenderPubkey = storm[0].SenderPubkey; nv.Payload = payload; nv.Block = {0xc0};
    nv.hasM2 = nv.hasM3 = true; nv.M2AggSig = m2s; nv.M2Bitmap = m2b; nv.M3AggSig = m3s; nv.M3Bitmap = m3b;
    viewChange validator; CHECK(validator.Init(pubs).empty());
    CHECK(validator.OnNewViewChecks(nv).empty());
    { auto bad = nv; bad.M3AggSig = m2s; CHECK(validator.OnNewViewChecks(bad) == errM3Verify); }
    { auto bad = nv; bad.M2AggSig = m3s; CHECK(validator.OnNewViewChecks(bad) == errM2Verify); }
    { auto bad = nv; bad.hasM3 = false; CHECK(validator.OnNewViewChecks(bad) == errM3Nil); }
    { auto bad = nv; bad.Payload[3] ^= 1; CHECK(validator.OnNewViewChecks(bad) == errNewViewM1); }
    { auto bad = nv; bad.Payload.resize(100); CHECK(validator.OnNewViewChecks(bad) == errPayloadLength); }
    { auto bad = nv; bad.M3AggSig.assign(96, 0xff); CHECK(validator.OnNewViewChecks(bad) == errSigDeserialize); }
    { auto bad = nv; bad.M3Bitmap = {0x0f}; CHECK(validator.OnNewViewChecks(bad) == errM3Verify); }                  // aggregate of 5 against 4 keys
}

static void test_leader_votes_and_slash() {
    using namespace consensus;
    // leader's COMMIT collection on a 7-validator committee (quorum 5): single-key votes, one 2-key vote, one fault of each kind
    auto keys = make_keys(8);
    std::vector<bls::PublicKeyWrapper> pubs; for (int i = 0; i < 7; i++) pubs.push_back(*keys[i].Pub);
    auto kb = [&](int i) { return Bytes(keys[i].Pub->Bytes.begin(), keys[i].Pub->Bytes.end()); };
    std::array<uint8_t, 32> bh; for (int i = 0; i < 32; i++) bh[i] = (uint8_t)(11 * i + 3);
    const Bytes payload = signature::ConstructCommitPayload(true, bh, 77, 78);
    auto vote1 = [&](int i) { return Vote{{kb(i)}, sign_bytes(keys[i], payload)}; };
    // keys 1 and 2 belong to one validator: ONE signature that verifies against pk1 + pk2 (the sum of the two signatures)
    std::unique_ptr<bls_core::Sign> s1(keys[1].Pri->SignHash(payload)), s2(keys[2].Pri->SignHash(payload));
    Vote multi{{kb(1), kb(2)}, bls::AggregateSig({s1.get(), s2.get()})->Serialize()};
    std::vector<Vote> votes = {vote1(0), multi, vote1(3), vote1(4), vote1(0), vote1(5), vote1(6), vote1(7)};
    votes[2].Payload = sign_bytes(keys[4], payload);             // somebody else's signature
    votes[5].Payload.assign(96, 0xff);                           // does not decode
    VoteCollector col; col.Init(pubs, payload);
    long q = -2; auto out = col.onVotes(votes, &q);
    CHECK(out[0].empty() && out[1].empty() && out[2] == errVoteSig && out[3].empty() && out[4] == errAlreadyReceived && out[5] == errSigDeserialize);
    CHECK(out[6].empty() && out[7] == errKeyNotFound);            // key 7 signs correctly but is not in the committee
    CHECK(q == 6 && col.SignersCount() == 6 && col.bitmap == Bytes{0x57});      // keys 0,1,2,4,6 + the recorded outsider ballot (reference quirk)
    { VoteCollector c2; c2.Init(pubs, payload); votes.pop_back(); c2.onVotes(votes); votes.push_back(vote1(3)); long q2 = -2; auto o2 = c2.onVotes({votes.back()}, &q2);
      CHECK(o2[0].empty() && q2 == -1 && c2.bitmap == Bytes{0x5f});
      Bytes agg; CHECK(c2.AggregateVotes(agg));
      bls::Committee com; CHECK(com.Load(pubs).empty());
      bls::SerializedSignature a96; std::copy(agg.begin(), agg.end(), a96.begin());
      CHECK(bls::FastAggregateVerify(com, c2.bitmap, a96, payload) == 1); }

    // double-sign evidence (staking/slash/double-sign.go): validator with keys 0 and 1 signs two blocks at one height / view
    std::array<uint8_t, 32> h1 = bh, h2 = bh; h2[0] ^= 1;
    auto ballot = [&](std::vector<int> idx, const std::array<uint8_t, 32>& h, const std::array<uint8_t, 32>& signedh) {
        slash::Vote v; v.BlockHeaderHash = h; std::vector<std::unique_ptr<bls_core::Sign>> ss; std::vector<bls_core::Sign*> ptr;
        const Bytes pl = signature::ConstructCommitPayload(true, signedh, 37, 38);
        for (int i : idx) { v.SignerPubKeys.push_back(kb(i)); ss.emplace_back(keys[i].Pri->SignHash(pl)); ptr.push_back(ss.back().get()); }
        v.Signature = bls::AggregateSig(ptr)->Serialize(); return v;
    };
    auto rec = [&](slash::Vote a, slash::Vote b) { slash::Record r; r.Evidence.Height = 37; r.Evidence.ViewID = 38; r.Evidence.FirstVote = a; r.Evidence.SecondVote = b; return r; };
    std::vector<slash::Record> recs = {rec(ballot({0, 1}, h1, h1), ballot({0, 1}, h2, h2)), rec(ballot({0}, h1, h1), ballot({0, 2}, h2, h2)),
                                       rec(ballot({0, 1}, h1, h1), ballot({0, 1}, h1, h1)), rec(ballot({0, 1}, h1, h1), ballot({2, 3}, h2, h2)),
                                       rec(ballot({0, 1}, h1, h1), ballot({0, 1}, h2, h1)), rec(ballot({0, 1}, h1, h1), ballot({0, 1}, h2, h2)),
                                       rec(ballot({0, 1}, h1, h1), ballot({0, 1}, h2, h2))};
    recs[5].Evidence.FirstVote.Signature.assign(96, 0xff);
    recs[6].Evidence.SecondVote.SignerPubKeys[1].assign(48, 0xff);
    auto se = slash::VerifyBallots(recs);
    CHECK(se[0].empty() && se[1].empty() && se[2] == slash::errSlashBlockNoConflict && se[3] == slash::errNoMatchingDoubleSignKeys);
    CHECK(se[4] == slash::errFailVerifySlash && se[5] == errSigDeserialize && se[6] == errKeyDeserialize);
}

int main() {
    if (bls_core::Init(bls_core::BLS12_381) != 0) { fprintf(stderr, "bls.Init failed: CUDA device required (no CPU fallback)\n"); return 2; }
    test_mask(); test_quorum_votes(); test_codecs_multibls_payload(); test_consensus_messages(); test_leader_votes_and_slash();
    if (g_fail) { fprintf(stderr, "%d check(s) failed\n", g_fail); return 1; }
    printf("hbls_host_test: all checks passed\n");
    return 0;
}
