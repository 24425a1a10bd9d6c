// Host check of se2lam_b200/csrc/blur_px.h — the byte <-> float32 conversions orb_blur is compiled from — with PRMT emulated:
//   1. byte_to_float(w, k) is (float) of byte k of w, bit for bit, for all 256 bytes in each of the 4 positions
//   2. for every float32 x in [0, 256] (every bit pattern, so every tie x.5 included): the bits of x + 1.5 * 2^23 are
//      0x4B400000 + lrintf(x), and round_sat_bits(x) carries min(lrintf(x), 255) in its low byte, which is what the saturating
//      round-to-nearest-even of cv::GaussianBlur's u8 output gives
//   3. pack_low_bytes puts the low bytes of its 4 arguments into bytes 0..3
// Prints "OK <checks>" and exits 0, or a diagnostic and exits 1.
#include <cmath>
#include <cstdio>
#include <cstring>

#include "../../se2lam_b200/csrc/blur_px.h"

static unsigned bits(float f) {
    unsigned u;
    std::memcpy(&u, &f, sizeof u);
    return u;
}

int main() {
    long long checks = 0;
    for (int k = 0; k < 4; ++k)
        for (unsigned b = 0; b < 256; ++b) {
            const unsigned w = (0xA5C3E17Fu & ~(0xFFu << (8 * k))) | (b << (8 * k));   // the other bytes are not zero
            const float f = blurpx::byte_to_float(w, k);
            if (bits(f) != bits((float)b)) {
                std::printf("byte_to_float(0x%08x, %d) = %.9g, expected %u\n", w, k, f, b);
                return 1;
            }
            ++checks;
        }
    for (unsigned u = 0; u <= bits(256.0f); ++u) {
        float x;
        std::memcpy(&x, &u, sizeof x);
        const long r = lrintf(x);
        if (bits(blurpx::add_rn(x, 12582912.0f)) != 0x4B400000u + (unsigned)r) {
            std::printf("x = %.9g (0x%08x): x + 1.5*2^23 = 0x%08x, lrintf = %ld\n", x, u, bits(blurpx::add_rn(x, 12582912.0f)), r);
            return 1;
        }
        const unsigned s = blurpx::round_sat_bits(x);
        if ((s >> 8) != 0x4B4000u || (long)(s & 0xFFu) != (r < 255 ? r : 255)) {
            std::printf("round_sat_bits(%.9g) = 0x%08x, lrintf = %ld\n", x, s, r);
            return 1;
        }
        ++checks;
    }
    for (unsigned v = 0; v < 256; ++v) {
        const unsigned p = blurpx::pack_low_bytes(0x4B400000u | v, 0x4B400000u | (255 - v), 0x4B400000u | (v ^ 0x5A), 0x4B400000u | ((v * 7) & 255));
        const unsigned e = v | ((255 - v) << 8) | ((v ^ 0x5A) << 16) | (((v * 7) & 255) << 24);
        if (p != e) {
            std::printf("pack_low_bytes: 0x%08x, expected 0x%08x\n", p, e);
            return 1;
        }
        ++checks;
    }
    std::printf("OK %lld\n", checks);
    return 0;
}
