// harmony_b200/host/hbls_concurrency_test.cpp -- herumi-API calls from many std::threads at once, through include/hbls.h only.
// Every result is compared with the same call made alone (one thread, before the threads start): GetPublicKey and SignHash struct
// bytes, Serialize / Deserialize round trips, Add then Sub, IsEqual, and VerifyHash of valid triples, wrong messages and other
// threads' signatures.  Prints "all checks passed" and exits 0; needs a CUDA device (built and run by tests/test_concurrent_calls.py).
#include "../../include/hbls.h"
#include <atomic>
#include <cstdio>
#include <cstring>
#include <thread>
#include <vector>

static std::atomic<int> failures{0};
#define CHECK(cond, ...) do { if (!(cond)) { if (failures++ < 20) { std::printf("FAIL line %d: ", __LINE__); std::printf(__VA_ARGS__); std::printf("\n"); } } } while (0)

static uint64_t mix64(uint64_t x) { x += 0x9e3779b97f4a7c15ull; x = (x ^ (x >> 30)) * 0xbf58476d1ce4e5b9ull; x = (x ^ (x >> 27)) * 0x94d049bb133111ebull; return x ^ (x >> 31); }

struct Item {
    blsSecretKey sk; uint8_t msg[32];
    blsPublicKey pk; blsSignature sig; uint8_t pk48[48], sig96[96];        // the lone-call results
};

int main() {
    if (blsInit(HBLS_BLS12_381, HBLS_COMPILED_TIME_VAR) != 0) { std::printf("blsInit failed\n"); return 2; }
    const int T = 32, K = 6;
    std::vector<Item> items(T * K);
    for (int i = 0; i < T * K; i++) {
        Item& it = items[i];
        for (int w = 0; w < 4; w++) it.sk.d[w] = mix64(1000 + 4 * i + w);
        it.sk.d[3] &= 0x3fffffffffffffffull;                                   // < 2^254 < r
        for (int b = 0; b < 32; b++) it.msg[b] = (uint8_t)mix64((i % 3 == 0 ? 7 : 100 + i) * 64 + b);   // every third message shared
        blsGetPublicKey(&it.pk, &it.sk);
        CHECK(blsSignHash(&it.sig, &it.sk, it.msg, 32) == 0, "lone SignHash %d", i);
        CHECK(blsPublicKeySerialize(it.pk48, 48, &it.pk) == 48 && blsSignatureSerialize(it.sig96, 96, &it.sig) == 96, "lone Serialize %d", i);
    }
    uint64_t t0, r0, m0; hbls_coalesce_stats(&t0, &r0, &m0);
    std::vector<std::thread> th;
    for (int t = 0; t < T; t++)
        th.emplace_back([&, t] {
            for (int k = 0; k < K; k++) {
                const Item& it = items[t * K + k];
                const Item& other = items[((t + 1) % T) * K + k];
                blsPublicKey pk; blsGetPublicKey(&pk, &it.sk);
                CHECK(std::memcmp(&pk, &it.pk, sizeof pk) == 0, "GetPublicKey %d/%d differs from the lone call", t, k);
                blsSignature sig;
                CHECK(blsSignHash(&sig, &it.sk, it.msg, 32) == 0 && std::memcmp(&sig, &it.sig, sizeof sig) == 0, "SignHash %d/%d", t, k);
                CHECK(blsVerifyHash(&it.sig, &it.pk, it.msg, 32) == 1, "VerifyHash valid %d/%d", t, k);
                uint8_t bad[32]; std::memcpy(bad, it.msg, 32); bad[5] ^= 1;
                CHECK(blsVerifyHash(&it.sig, &it.pk, bad, 32) == 0, "VerifyHash wrong message %d/%d", t, k);
                CHECK(blsVerifyHash(&other.sig, &it.pk, it.msg, 32) == 0, "VerifyHash other signature %d/%d", t, k);
                uint8_t ser[96];
                CHECK(blsPublicKeySerialize(ser, 48, &pk) == 48 && std::memcmp(ser, it.pk48, 48) == 0, "PublicKeySerialize %d/%d", t, k);
                CHECK(blsSignatureSerialize(ser, 96, &sig) == 96 && std::memcmp(ser, it.sig96, 96) == 0, "SignatureSerialize %d/%d", t, k);
                blsPublicKey pk2; blsSignature sig2;
                CHECK(blsPublicKeyDeserialize(&pk2, it.pk48, 48) == 48 && blsPublicKeyIsEqual(&pk2, &it.pk) == 1, "PublicKeyDeserialize %d/%d", t, k);
                CHECK(blsSignatureDeserialize(&sig2, it.sig96, 96) == 96 && blsSignatureIsEqual(&sig2, &it.sig) == 1, "SignatureDeserialize %d/%d", t, k);
                uint8_t junk[96]; std::memset(junk, 0xff, 96);
                CHECK(blsSignatureDeserialize(&sig2, junk, 96) == 0, "undecodable signature accepted %d/%d", t, k);
                blsPublicKeyAdd(&pk2, &other.pk);
                CHECK(blsPublicKeyIsEqual(&pk2, &it.pk) == 0, "Add left the key unchanged %d/%d", t, k);
                blsPublicKeySub(&pk2, &other.pk);
                CHECK(blsPublicKeyIsEqual(&pk2, &it.pk) == 1, "Add then Sub %d/%d", t, k);
                blsSignature s3 = it.sig; blsSignatureAdd(&s3, &other.sig);
                CHECK(blsSignatureIsEqual(&s3, &it.sig) == 0, "SignatureAdd %d/%d", t, k);
            }
        });
    for (auto& x : th) x.join();
    uint64_t t1, r1, m1; hbls_coalesce_stats(&t1, &r1, &m1);
    std::printf("%llu requests in %llu turns, largest turn %llu\n", (unsigned long long)(r1 - r0), (unsigned long long)(t1 - t0), (unsigned long long)m1);
    CHECK(r1 - r0 == (uint64_t)T * K * 18,"%llu requests counted", (unsigned long long)(r1 - r0));
    char msg[160]; CHECK(hbls_last_error(msg, sizeof msg) == 0, "CUDA error: %s", msg);
    if (failures) { std::printf("%d checks failed\n", failures.load()); return 1; }
    std::printf("all checks passed\n");
    return 0;
}
