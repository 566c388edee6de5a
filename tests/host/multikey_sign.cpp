// tests/host/multikey_sign.cpp -- GPU: the multi-key signing of the C++ mirror (multibls::PrivateKeys::SignHashAggregate /
// SignHashEach, harmony_b200/host/hbls_host.hpp) against the loops it replaces, written out with one SignHash per key:
//   consensus/construct.go:97-114   sig := Sign{}; for each key { if s := SignHash(msg); s != nil { sig.Add(s) } }; sig.Serialize()
//   leader.go:57-75, view_change_construct.go:402-483, view_change_msg.go:78-92   SignHash(msg) per key, each serialized
// Links libhbls.so.  Exit code 0 and "all checks passed" = every check held.
#include <cstdio>
#include <string>
#include "../../harmony_b200/host/hbls_host.hpp"

using namespace harmony;
static int g_fail = 0;
#define CHECK(c) do { if (!(c)) { fprintf(stderr, "CHECK FAILED %s:%d: %s\n", __FILE__, __LINE__, #c); g_fail++; } } while (0)

// the loop of construct.go:99-114, one device call per SignHash / Add / Serialize
static std::vector<uint8_t> loop_aggregate(const multibls::PrivateKeys& keys, const std::vector<uint8_t>& msg) {
    bls_core::Sign sig;
    for (auto& k : keys) {
        std::unique_ptr<bls_core::Sign> s(k.Pri->SignHash(msg));
        if (s) sig.Add(s.get());
    }
    return sig.Serialize();
}

static std::vector<uint8_t> bytes_of(const std::string& s) { return std::vector<uint8_t>(s.begin(), s.end()); }

int main() {
    if (bls_core::Init(bls_core::BLS12_381) != 0) { fprintf(stderr, "blsInit failed\n"); return 2; }
    std::vector<std::shared_ptr<bls_core::SecretKey>> secrets;
    for (int i = 0; i < 10; i++) secrets.push_back(bls::RandPrivateKey());
    const multibls::PrivateKeys keys = multibls::GetPrivateKeys(secrets);

    std::array<uint8_t, 32> block_hash{}; for (int i = 0; i < 32; i++) block_hash[i] = (uint8_t)(7 * i + 1);
    const std::vector<uint8_t> commit = signature::ConstructCommitPayload(true, block_hash, 1234567, 89);      // 48 bytes
    const std::vector<uint8_t> prepare(block_hash.begin(), block_hash.end());                                  // 32 bytes
    std::vector<uint8_t> m1(prepare); for (int i = 0; i < 40; i++) m1.push_back((uint8_t)(i * 13));            // hash || payload: 72 bytes
    const std::vector<uint8_t> nil = bytes_of("NIL");                                                          // unused message form
    std::vector<uint8_t> view_id(8); for (int i = 0; i < 8; i++) view_id[i] = (uint8_t)(90 >> (8 * i));
    const std::vector<uint8_t> unmappable(48, 0);

    // the validator's vote: prepare (32 bytes), commit (48 bytes), and a message that maps to no point (identity, like the loop)
    for (const std::vector<uint8_t>& msg : {prepare, commit, m1, unmappable}) {
        const auto got = keys.SignHashAggregate(msg), want = loop_aggregate(keys, msg);
        CHECK(got.size() == 96 && got == want);
    }
    CHECK(keys.SignHashAggregate(unmappable) == std::vector<uint8_t>(96, 0));
    multibls::PrivateKeys one, none; one.push_back(keys[0]);
    CHECK(one.SignHashAggregate(commit) == loop_aggregate(one, commit));
    CHECK(none.SignHashAggregate(commit) == std::vector<uint8_t>(96, 0));

    // the per-key loops: view change (M1 or NIL, then the view id) and the leader's own votes
    const std::vector<std::vector<uint8_t>> msgs = {m1, view_id, nil, unmappable, prepare};
    const auto each = keys.SignHashEach(msgs);
    CHECK(each.size() == msgs.size());
    for (size_t j = 0; j < msgs.size(); j++) {
        CHECK(each[j].size() == keys.size());
        for (size_t i = 0; i < keys.size() && each[j].size() == keys.size(); i++) {
            std::unique_ptr<bls_core::Sign> s(keys[i].Pri->SignHash(msgs[j]));
            if (s) CHECK(each[j][i] == s->Serialize());
            else CHECK(each[j][i].empty());
        }
    }
    CHECK(each[3][0].empty() && !each[0][0].empty());
    // a per-key signature verifies under its key, and their sum is the aggregate
    bls_core::Sign sum;
    for (size_t i = 0; i < keys.size(); i++) {
        bls_core::Sign s; CHECK(s.Deserialize(each[4][i]));
        CHECK(s.VerifyHash(keys[i].Pub->Object.get(), prepare));
        sum.Add(&s);
    }
    CHECK(sum.Serialize() == keys.SignHashAggregate(prepare));

    if (g_fail) { printf("%d checks failed\n", g_fail); return 1; }
    printf("all checks passed\n");
    return 0;
}
