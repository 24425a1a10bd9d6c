// Order key of a float keypoint response, usable from host and device code.
//
// The Harris-score selection (orb_select<true>) sorts 64-bit records key << 32 | (score:8|y:12|x:12) by their upper word, so
// the key's unsigned order must be the float order: non-negative floats get their sign bit set, negative ones are
// complemented. -0.0f is mapped to the key of +0.0f first (the two compare equal as floats, and equal floats must stay
// ties for the introselect permutation). NaN never occurs (the Harris response of integer sums is finite).
// tests/native/resp_key_host.cpp checks the host build over every float class.
#pragma once
#include <stdint.h>
#if !defined(__CUDACC__)
#include <string.h>
#endif

#if defined(__CUDACC__)
#define SE2_RK_HD __host__ __device__ __forceinline__
#else
#define SE2_RK_HD inline
#endif

namespace se2gpu {

SE2_RK_HD uint32_t float_bits(float v) {
#if defined(__CUDA_ARCH__)
    return __float_as_uint(v);
#else
    uint32_t u;
    memcpy(&u, &v, sizeof u);
    return u;
#endif
}

SE2_RK_HD float bits_float(uint32_t u) {
#if defined(__CUDA_ARCH__)
    return __uint_as_float(u);
#else
    float v;
    memcpy(&v, &u, sizeof v);
    return v;
#endif
}

SE2_RK_HD uint32_t resp_key(float v) {
    uint32_t u = float_bits(v);
    if (u == 0x80000000u) u = 0u;                          // -0 -> +0
    return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}

// inverse of resp_key (returns +0.0f for the key of -0.0f)
SE2_RK_HD float resp_from_key(uint32_t k) {
    return bits_float((k & 0x80000000u) ? (k & 0x7FFFFFFFu) : ~k);
}

}  // namespace se2gpu
