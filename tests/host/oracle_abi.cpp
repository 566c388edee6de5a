// tests/host/oracle_abi.cpp -- TEST HARNESS ONLY: the subset of include/hbls.h that the C++ vote collectors of
// harmony_b200/host/hbls_consensus.hpp call, restated over the CPU oracle (oracle/libhbls_oracle.so), so that their host logic runs
// without a GPU.  Linked into tests/host/vote_collectors.cpp in place of libhbls.so; never part of the product.
// Keys and signatures are kept in their serialized form inside the herumi-shaped structs (all-zero = the identity encoding).
#include <cstring>
#include <set>
#include <vector>
#include "../../include/hbls.h"

extern "C" {
int ho_pk_deserialize_check(const uint8_t pk48[48]);
int ho_sig_deserialize_check(const uint8_t sig96[96]);
int ho_pk_add(const uint8_t a[48], const uint8_t b[48], int sub, uint8_t out[48]);
int ho_verify_hash(const uint8_t sig96[96], const uint8_t pk48[48], const uint8_t* msg, size_t len);
int ho_aggregate_sigs(size_t n, const uint8_t* sigs96, uint8_t out96[96]);
void* ho_committee_new(size_t n, const uint8_t* pks48);
void ho_committee_free(void* h);
int ho_committee_aggregate_verify(void* h, const uint8_t* bitmap, size_t blen, const uint8_t sig96[96], const uint8_t* msg, size_t len);
}

struct hbls_committee { void* h = nullptr; size_t n = 0; };
struct hbls_ballot_box { const hbls_committee* c = nullptr; std::vector<uint8_t> collected; std::vector<uint8_t> sigs; };

// calls made, for the test's "one box call" check: [0] hbls_ballot_box_submit_votes, [1] hbls_verify_batch_status, [2] hbls_ballot_box_add_vote
size_t oracle_abi_calls[3] = {0, 0, 0};

static bool overlaps(const uint8_t* bm, const std::vector<uint8_t>& col, size_t n) {
    for (size_t i = 0; i < n; i++) if ((bm[i >> 3] >> (i & 7)) & (col[i >> 3] >> (i & 7)) & 1) return true;
    return false;
}
static void join(const uint8_t* bm, std::vector<uint8_t>& col, size_t n) {
    for (size_t i = 0; i < n; i++) if ((bm[i >> 3] >> (i & 7)) & 1) col[i >> 3] |= (uint8_t)(1u << (i & 7));
}

extern "C" {
size_t blsPublicKeySerialize(void* buf, size_t maxBufSize, const blsPublicKey* pub) {
    if (maxBufSize < 48) return 0;
    std::memcpy(buf, pub->d, 48); return 48;
}
size_t blsPublicKeyDeserialize(blsPublicKey* pub, const void* buf, size_t bufSize) {
    if (bufSize != 48 || ho_pk_deserialize_check((const uint8_t*)buf) != 1) return 0;
    std::memset(pub, 0, sizeof *pub); std::memcpy(pub->d, buf, 48); return 48;
}
void blsPublicKeyAdd(blsPublicKey* pub, const blsPublicKey* rhs) {
    uint8_t out[48];
    if (ho_pk_add((const uint8_t*)pub->d, (const uint8_t*)rhs->d, 0, out) == 0) std::memcpy(pub->d, out, 48);
}
int hbls_verify_batch_status(size_t k, const uint8_t* pk48, const uint8_t* sig96, const uint8_t* msgs, size_t msg_len, uint8_t* status) {
    oracle_abi_calls[1]++;
    for (size_t j = 0; j < k; j++) {
        const uint8_t *pk = pk48 + 48 * j, *sg = sig96 + 96 * j;
        if (ho_pk_deserialize_check(pk) != 1) status[j] = HBLS_VB_BAD_KEY_ENCODING;
        else if (ho_sig_deserialize_check(sg) != 1) status[j] = HBLS_VB_BAD_SIG_ENCODING;
        else status[j] = ho_verify_hash(sg, pk, msgs + msg_len * j, msg_len) == 1 ? HBLS_VB_OK : HBLS_VB_BAD_SIG;
    }
    return 0;
}
int hbls_aggregate_sigs(const uint8_t* sig96, size_t n, uint8_t out96[96]) {
    return ho_aggregate_sigs(n, sig96, out96) == 0 ? 0 : HBLS_ERR_DECODE;
}
int hbls_committee_create(hbls_committee** out, const uint8_t* pk48, size_t n, size_t* bad_index) {
    for (size_t i = 0; i < n; i++) if (ho_pk_deserialize_check(pk48 + 48 * i) != 1) { if (bad_index) *bad_index = i; return HBLS_ERR_DECODE; }
    *out = new hbls_committee{ho_committee_new(n, pk48), n};
    return 0;
}
void hbls_committee_destroy(hbls_committee* c) { if (c) { ho_committee_free(c->h); delete c; } }
int hbls_ballot_box_create(hbls_ballot_box** out, const hbls_committee* c) {
    *out = new hbls_ballot_box{c, std::vector<uint8_t>((c->n + 7) >> 3, 0), {}};
    return 0;
}
void hbls_ballot_box_destroy(hbls_ballot_box* b) { delete b; }
int hbls_ballot_box_add_vote(hbls_ballot_box* b, const uint8_t* signer_bitmap, size_t blen, const uint8_t sig96[96]) {
    oracle_abi_calls[2]++;
    if (blen != b->collected.size()) return HBLS_ERR_ARG;
    if (overlaps(signer_bitmap, b->collected, b->c->n)) return 1;
    if (ho_sig_deserialize_check(sig96) != 1) return HBLS_ERR_DECODE;
    join(signer_bitmap, b->collected, b->c->n); b->sigs.insert(b->sigs.end(), sig96, sig96 + 96);
    return 0;
}
// the ballot rules of leader.go:227-290 in arrival order: already collected, Sign.Deserialize, VerifyHash over the signers' key sum
int hbls_ballot_box_submit_votes(hbls_ballot_box* b, size_t k, const uint8_t* signer_bitmaps, size_t blen, const uint8_t* sigs96,
                                 const void* msg, size_t msg_len, uint8_t* status) {
    oracle_abi_calls[0]++;
    if (!b || !status || blen != b->collected.size() || msg_len > 64) return HBLS_ERR_ARG;
    for (size_t j = 0; j < k; j++) {
        const uint8_t *bm = signer_bitmaps + j * blen, *sg = sigs96 + 96 * j;
        if (overlaps(bm, b->collected, b->c->n)) status[j] = HBLS_BALLOT_COLLECTED;
        else if (ho_sig_deserialize_check(sg) != 1) status[j] = HBLS_BALLOT_BAD_SIG_ENCODING;
        else if (ho_committee_aggregate_verify(b->c->h, bm, blen, sg, (const uint8_t*)msg, msg_len) != 1) status[j] = HBLS_BALLOT_BAD_SIG;
        else { status[j] = HBLS_BALLOT_ACCEPTED; join(bm, b->collected, b->c->n); b->sigs.insert(b->sigs.end(), sg, sg + 96); }
    }
    return 0;
}
int hbls_ballot_box_aggregate(const hbls_ballot_box* b, uint8_t out_sig96[96], uint8_t* bitmap_out, size_t blen) {
    if (b->sigs.empty()) std::memset(out_sig96, 0, 96);
    else if (ho_aggregate_sigs(b->sigs.size() / 96, b->sigs.data(), out_sig96) != 0) return HBLS_ERR_DECODE;
    if (bitmap_out) std::memcpy(bitmap_out, b->collected.data(), blen);
    return 0;
}
}
