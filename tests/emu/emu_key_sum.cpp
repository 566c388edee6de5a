// tests/emu/emu_key_sum.cpp -- TEST HARNESS ONLY: exports the key sum of harmony_b200/csrc/secret_key.hpp (hb_secret::sk_sum_mod_r,
// the aggregate key of hbls_sign_hash_keys) and the base-|z| digits the library takes of it.  Never linked into libhbls.so.
#include <cstddef>
#include <cstdint>
#include "../../harmony_b200/csrc/secret_key.hpp"

// sum = (sum of the k little-endian 32-byte keys) mod r; dig = its four base-|z| digits.  Returns sk_digits_base_z's verdict on the sum.
extern "C" int emu_key_sum(const uint8_t* sk32, size_t k, uint64_t* sum, uint64_t* dig) {
    hb_secret::sk_sum_mod_r(sk32, k, sum);
    return hb_secret::sk_digits_base_z(sum, dig) ? 1 : 0;
}
