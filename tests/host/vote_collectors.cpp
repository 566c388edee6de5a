// tests/host/vote_collectors.cpp -- TEST HARNESS ONLY: the C++ consensus::BallotBoxCollector against consensus::VoteCollector
// (harmony_b200/host/hbls_consensus.hpp), both over the CPU oracle (tests/host/oracle_abi.cpp).  Seeded queues of one-key and multi-key
// votes with every fault the handlers distinguish -- undecodable, short, wrong and someone else's signatures, repeated keys, non-member
// keys, an empty key list, signers repeated within and across ticks -- in one tick or cut into many: the same errors, quorum index,
// ballots, bitmap and AggregateVotes bytes; a queue of distinct members is one box call and nothing else.
#include <cstdio>
#include <random>
#include "../../harmony_b200/host/hbls_consensus.hpp"

extern "C" {
int ho_get_public_key(const uint8_t sk[32], uint8_t pk48[48]);
int ho_sign_hash(const uint8_t sk[32], const uint8_t* msg, size_t len, uint8_t sig96[96]);
int ho_sig_add(const uint8_t a[96], const uint8_t b[96], uint8_t out[96]);
}
extern size_t oracle_abi_calls[3];
using namespace harmony;
using consensus::Bytes;
static int g_fail = 0;
#define CHECK(c) do { if (!(c)) { fprintf(stderr, "CHECK FAILED %s:%d: %s\n", __FILE__, __LINE__, #c); g_fail++; } } while (0)

struct Keys {
    std::vector<Bytes> pk, sig;                  // member i < n, outsiders after; sig[i] = key i's signature of the message
    std::vector<bls::PublicKeyWrapper> members;
    Keys(size_t n, size_t extra, const Bytes& msg) {
        for (size_t i = 0; i < n + extra; i++) {
            uint8_t sk[32] = {0}; uint64_t x = 0x9e3779b97f4a7c15ull * (i + 1);
            for (int b = 0; b < 24; b++) { x ^= x >> 29; x *= 0xbf58476d1ce4e5b9ull; sk[b] = (uint8_t)(x >> 32); }      // < 2^192 < r
            Bytes p(48), s(96);
            ho_get_public_key(sk, p.data()); ho_sign_hash(sk, msg.data(), msg.size(), s.data());
            pk.push_back(p); sig.push_back(s);
            if (i < n) { bls::PublicKeyWrapper w; std::memcpy(w.Bytes.data(), p.data(), 48); members.push_back(w); }
        }
    }
    Bytes signOf(const std::vector<size_t>& idx) const {           // signature of the key sum = sum of the signatures
        Bytes acc = sig[idx[0]];
        for (size_t t = 1; t < idx.size(); t++) { Bytes o(96); ho_sig_add(acc.data(), sig[idx[t]].data(), o.data()); acc = o; }
        return acc;
    }
    consensus::Vote vote(const std::vector<size_t>& idx, const std::vector<size_t>& signers) const {
        consensus::Vote v; for (size_t i : idx) v.SenderPubkeys.push_back(pk[i]);
        v.Payload = signOf(signers); return v;
    }
};

static std::vector<consensus::Vote> queue(const Keys& K, size_t n, std::mt19937& rng, size_t len) {
    std::vector<consensus::Vote> out;
    auto pick = [&](size_t m) { std::vector<size_t> all(n); for (size_t i = 0; i < n; i++) all[i] = i; std::shuffle(all.begin(), all.end(), rng); all.resize(m); return all; };
    for (size_t t = 0; t < len; t++) {
        const size_t r = rng() % 20;
        auto idx = pick(rng() % 3 ? 1 : 2 + rng() % 3);
        consensus::Vote v = K.vote(idx, idx);
        if (r == 1) v.Payload.assign(96, 0xff);                                           // does not decode
        else if (r == 2) v = K.vote(idx, {(idx[0] + 1) % n});                              // someone else's signature
        else if (r == 3) v.Payload.resize(95);                                             // short payload
        else if (r == 4) v = K.vote({idx[0], idx[0]}, {idx[0], idx[0]});                   // repeated key
        else if (r == 5) { const size_t o = n + rng() % (K.pk.size() - n); v = rng() % 2 ? K.vote({idx[0], o}, {idx[0], o}) : K.vote({o}, {o}); }   // non-member
        else if (r == 6) v.SenderPubkeys.clear();
        else if (r == 7 && idx.size() > 1) v = K.vote(idx, {idx.begin(), idx.end() - 1});  // multi-key signature missing a key
        out.push_back(v);
    }
    return out;
}

int main() {
    const size_t n = 21;
    Bytes msg(40); for (size_t i = 0; i < 40; i++) msg[i] = (uint8_t)(3 * i + 1);
    Keys K(n, 3, msg);
    std::set<std::string> seen;                     // every outcome the handlers distinguish occurs in the seeded queues
    for (unsigned seed = 0; seed < 8; seed++) {
        std::mt19937 rng(seed);
        consensus::VoteCollector ref; ref.Init(K.members, msg);
        consensus::BallotBoxCollector col; CHECK(col.Init(K.members, msg).empty());
        std::vector<std::vector<consensus::Vote>> ticks;
        auto q = queue(K, n, rng, 36);
        if (seed % 2 == 0) ticks.push_back(q);
        else for (size_t pos = 0; pos < q.size();) { const size_t step = 1 + rng() % 8; ticks.emplace_back(q.begin() + pos, q.begin() + std::min(q.size(), pos + step)); pos += step; }
        ticks.push_back(queue(K, n, rng, 12));
        for (auto& tick : ticks) {
            long qa = -2, qb = -2;
            const auto ea = ref.onVotes(tick, &qa), eb = col.onVotes(tick, &qb);
            CHECK(ea == eb); CHECK(qa == qb);
            seen.insert(ea.begin(), ea.end());
            CHECK(ref.SignersCount() == col.SignersCount() && ref.IsQuorumAchieved() == col.IsQuorumAchieved());
        }
        CHECK(ref.BallotBox.size() == col.BallotBox.size());
        for (auto& kv : ref.BallotBox) {
            auto it = col.BallotBox.find(kv.first);
            CHECK(it != col.BallotBox.end() && it->second.SignerPubKeys == kv.second.SignerPubKeys && it->second.Signature == kv.second.Signature);
        }
        Bytes sa, sb, bm;
        CHECK(ref.AggregateVotes(sa) && col.AggregateVotes(sb, bm));
        CHECK(sa == sb && bm == ref.bitmap && col.bitmap == ref.bitmap);
    }
    CHECK(seen == std::set<std::string>({"", consensus::errKeyDeserialize, consensus::errAlreadyReceived, consensus::errSigDeserialize,
                                         consensus::errVoteSig, consensus::errDuplicateKey, consensus::errKeyNotFound}));
    // an honest queue: one box call, the key sums and status triples of VoteCollector's path are never needed
    {
        consensus::BallotBoxCollector col; CHECK(col.Init(K.members, msg).empty());
        std::vector<consensus::Vote> q;
        for (size_t i = 0; i < 8; i++) q.push_back(K.vote({i}, {i}));
        q.push_back(K.vote({8, 9, 10}, {8, 9, 10})); q.push_back(K.vote({3}, {3})); q.push_back(K.vote({11, 12, 13, 14, 15}, {11, 12, 13, 14, 15}));
        const size_t cached = bls::BLSPubKeyCache().Len();
        const size_t c0[3] = {oracle_abi_calls[0], oracle_abi_calls[1], oracle_abi_calls[2]};
        long qa = -2;
        const auto e = col.onVotes(q, &qa);
        CHECK(oracle_abi_calls[0] == c0[0] + 1 && oracle_abi_calls[1] == c0[1] && oracle_abi_calls[2] == c0[2]);
        CHECK(e == std::vector<std::string>({"", "", "", "", "", "", "", "", "", consensus::errAlreadyReceived, ""}));
        CHECK(qa == 10 && col.SignersCount() == 16 && col.IsQuorumAchieved());                   // 2 * 21 / 3 + 1 = 15
        CHECK(bls::BLSPubKeyCache().Len() == cached);                                            // no key was decoded
    }
    if (g_fail) { fprintf(stderr, "%d check(s) failed\n", g_fail); return 1; }
    printf("vote_collectors: all checks passed\n"); return 0;
}
