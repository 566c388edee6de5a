// harmony_b200/csrc/chacha20.hpp -- the host's coefficient stream: ChaCha20 block function (RFC 8439 section 2.3), keyed from
// /dev/urandom at init (hbls.cu), state words 12, 13 = the call counter, 14 = the stream's nonce word, 15 = the block.  Host code only;
// the device draws of captured calls use kernels.cuh chacha20_block_dev under another nonce word.
#pragma once
#include <cstdint>
#include <cstring>

inline void chacha20_block(const uint32_t key[8], uint64_t counter, uint32_t out[16], uint32_t block = 0) {
    uint32_t st[16] = {0x61707865u, 0x3320646eu, 0x79622d32u, 0x6b206574u, key[0], key[1], key[2], key[3], key[4], key[5], key[6], key[7],
                       (uint32_t)counter, (uint32_t)(counter >> 32), 0x68626c73u /* "hbls" */, block};
    uint32_t x[16]; memcpy(x, st, sizeof x);
    auto rotl = [](uint32_t v, int c) { return (v << c) | (v >> (32 - c)); };
    auto qr = [&](int a, int b, int c, int d) {
        x[a] += x[b]; x[d] ^= x[a]; x[d] = rotl(x[d], 16); x[c] += x[d]; x[b] ^= x[c]; x[b] = rotl(x[b], 12);
        x[a] += x[b]; x[d] ^= x[a]; x[d] = rotl(x[d], 8);  x[c] += x[d]; x[b] ^= x[c]; x[b] = rotl(x[b], 7);
    };
    for (int r = 0; r < 10; r++) { qr(0, 4, 8, 12); qr(1, 5, 9, 13); qr(2, 6, 10, 14); qr(3, 7, 11, 15); qr(0, 5, 10, 15); qr(1, 6, 11, 12); qr(2, 7, 8, 13); qr(3, 4, 9, 14); }
    for (int i = 0; i < 16; i++) out[i] = x[i] + st[i];
}
