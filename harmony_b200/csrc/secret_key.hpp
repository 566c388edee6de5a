// harmony_b200/csrc/secret_key.hpp -- host-side handling of secret-key bytes (hbls.cu; also compiled into the CPU tests).
// Every function here runs the same instruction sequence whatever the key: no branch, table index or variable-latency
// instruction (no `/` or `%`: on x86-64 a 128-bit division is a __udivti3 call whose run time depends on its operands)
// decides on key bits.
#pragma once
#include <stdint.h>
#include <string.h>

namespace hb_secret {

// r (BLS12-381 group order), little-endian u64
static const uint64_t R_ORDER[4] = {0xffffffff00000001ull, 0x53bda402fffe5bfeull, 0x3339d80809a1d805ull, 0x73eda753299d7d48ull};
static const uint64_t Z_ABS = 0xd201000000010000ull;          // |z|, the BLS parameter

// v <- v / Z, returns v mod Z: restoring division, one quotient bit per step over all 256 bits.  The remainder stays below Z < 2^64,
// so 2 rem + bit < 2^65 and the trial subtraction's borrow (bit 127 of the 128-bit difference) is the comparison.
inline uint64_t div_z(uint64_t v[4]) {
    unsigned __int128 rem = 0;
    for (int i = 255; i >= 0; i--) {
        rem = (rem << 1) | ((v[i >> 6] >> (i & 63)) & 1u);
        const unsigned __int128 t = rem - Z_ABS;
        const uint64_t ge = (uint64_t)(t >> 127) ^ 1u;               // 1 when rem >= Z
        rem -= (unsigned __int128)(Z_ABS & (0 - ge));
        v[i >> 6] = (v[i >> 6] & ~(1ull << (i & 63))) | (ge << (i & 63));
    }
    return (uint64_t)rem;
}

// sk (little-endian u64 x 4) -> its four base-Z digits (sk = d0 + d1 Z + d2 Z^2 + d3 Z^3, d3 < 2^64).  Returns false for sk >= Z^3 2^64,
// which only a hand-filled struct holds (every key below r < Z^4 fits); that case is public and may take another path.
inline bool sk_digits_base_z(const uint64_t sk[4], uint64_t dig[4]) {
    uint64_t v[4] = {sk[0], sk[1], sk[2], sk[3]};
    for (int k = 0; k < 3; k++) dig[k] = div_z(v);
    dig[3] = v[0];
    const bool fits = (v[1] | v[2] | v[3]) == 0;
    for (int i = 0; i < 4; i++) v[i] = 0;
    __asm__ __volatile__("" : : "r"(v) : "memory");
    return fits;
}

// k < r: the borrow out of k - r
inline bool scalar_lt_r(const uint64_t k[4]) {
    uint64_t borrow = 0;
    for (int i = 0; i < 4; i++) {
        const unsigned __int128 d = (unsigned __int128)k[i] - R_ORDER[i] - borrow;
        borrow = (uint64_t)(d >> 64) & 1u;
    }
    return borrow != 0;
}

// v <- v - r when v >= r: the subtraction always runs and a mask made from its borrow selects the result
inline void sub_r_if_ge(uint64_t v[4]) {
    uint64_t t[4], borrow = 0;
    for (int i = 0; i < 4; i++) {
        const unsigned __int128 d = (unsigned __int128)v[i] - R_ORDER[i] - borrow;
        t[i] = (uint64_t)d; borrow = (uint64_t)(d >> 64) & 1u;
    }
    const uint64_t keep = 0 - borrow;                               // all ones when v < r
    for (int i = 0; i < 4; i++) v[i] = (v[i] & keep) | (t[i] & ~keep);
    t[0] = t[1] = t[2] = t[3] = 0;
    __asm__ __volatile__("" : : "r"(t) : "memory");
}

// sum = (sk_0 + ... + sk_{k-1}) mod r over k little-endian 32-byte keys.  Each key is first reduced by two conditional subtractions
// (2^256 < 3r), so a hand-filled struct >= r adds what its own ladder signs with: sk H = (sk mod r) H.  acc + key < 2r < 2^256
// never carries out of 256 bits, and one more conditional subtraction brings it back below r.
inline void sk_sum_mod_r(const uint8_t* sk32, size_t k, uint64_t sum[4]) {
    uint64_t acc[4] = {0, 0, 0, 0}, v[4];
    for (size_t j = 0; j < k; j++) {
        memcpy(v, sk32 + 32 * j, 32);
        sub_r_if_ge(v); sub_r_if_ge(v);
        uint64_t carry = 0;
        for (int i = 0; i < 4; i++) {
            const unsigned __int128 s = (unsigned __int128)acc[i] + v[i] + carry;
            acc[i] = (uint64_t)s; carry = (uint64_t)(s >> 64);
        }
        sub_r_if_ge(acc);
    }
    for (int i = 0; i < 4; i++) { sum[i] = acc[i]; acc[i] = 0; v[i] = 0; }
    __asm__ __volatile__("" : : "r"(acc), "r"(v) : "memory");
}

// 32-byte equality without an early exit
inline bool eq32(const void* a, const void* b) {
    const uint8_t* x = static_cast<const uint8_t*>(a); const uint8_t* y = static_cast<const uint8_t*>(b);
    uint32_t d = 0;
    for (int i = 0; i < 32; i++) d |= (uint32_t)(x[i] ^ y[i]);
    return d == 0;
}

// zeroes n bytes; the barrier makes the compiler keep the stores although the buffer is not read again
inline void wipe(void* p, size_t n) {
    if (!n) return;
    memset(p, 0, n);
    __asm__ __volatile__("" : : "r"(p) : "memory");
}

}  // namespace hb_secret
