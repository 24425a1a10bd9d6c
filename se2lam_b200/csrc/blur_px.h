// Byte <-> float32 conversions of orb_blur without conversion-pipe instructions (I2F / F2I).
//
// Shared by the CUDA kernel (orb.cu: orb_blur) and by a host unit test (tests/native/blur_px_host.cpp), which compiles THIS source
// with PRMT emulated (fastpx::perm) and checks the identities below exhaustively over the value ranges the blur produces.
//   byte -> float   the word 0x4B0000bb is the float 2^23 + b (ulp 1 in [2^23, 2^24)), so one PRMT and one exact
//                   subtraction give (float)b
//   float -> byte   for 0 <= x < 2^22, x + 1.5 * 2^23 lies in [1.5 * 2^23, 2^24) where the ulp is 1: the FADD rounds to the nearest
//                   integer, ties to even (1.5 * 2^23 is even), and the result's bits are 0x4B400000 + rint(x). One unsigned min
//                   against 0x4B4000FF saturates at 255; the low byte is then min(rint(x), 255). The blur's sums lie in [0, 255.5).
#pragma once
#include <cstdint>
#include <cstring>

#include "fast_screen.h"   // SE2_HD, fastpx::perm (PRMT, emulated on the host)

namespace blurpx {

SE2_HD float as_float(unsigned u) {
#if defined(__CUDA_ARCH__)
    return __uint_as_float(u);
#else
    float f;
    std::memcpy(&f, &u, sizeof f);
    return f;
#endif
}
SE2_HD unsigned as_uint(float f) {
#if defined(__CUDA_ARCH__)
    return __float_as_uint(f);
#else
    unsigned u;
    std::memcpy(&u, &f, sizeof u);
    return u;
#endif
}
SE2_HD float add_rn(float a, float b) {
#if defined(__CUDA_ARCH__)
    return __fadd_rn(a, b);
#else
    return a + b;
#endif
}

// (float) of byte k (0..3) of w
SE2_HD float byte_to_float(unsigned w, int k) { return add_rn(as_float(fastpx::perm(w, 0x4B000000u, 0x7540u | (unsigned)k)), -8388608.0f); }

// min(rint(x), 255) in the low byte, for 0 <= x < 2^22 (the other bytes are those of 0x4B400000)
SE2_HD unsigned round_sat_bits(float x) {
    const unsigned b = as_uint(add_rn(x, 12582912.0f));
    return b < 0x4B4000FFu ? b : 0x4B4000FFu;
}

// the low bytes of a, b, c, d as one word (a in byte 0)
SE2_HD unsigned pack_low_bytes(unsigned a, unsigned b, unsigned c, unsigned d) {
    return fastpx::perm(fastpx::perm(a, b, 0x0040u), fastpx::perm(c, d, 0x0040u), 0x5410u);
}

}  // namespace blurpx
