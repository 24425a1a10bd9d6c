// FAST-9-16 necessary condition on packed ring differences, 4 pixels (one 32-bit patch word) at a time.
//
// Shared by the CUDA kernels (orb.cu: pass A of both instantiations of orb_fast_cells) and by a host unit test
// (tests/native/fast_screen_host.cpp), which compiles THIS source with the packed-SIMD intrinsics emulated, checks it against the
// scalar definition of cv::FAST's quick reject (reference src/ORBextractor.cpp:616-623 -> cv::FAST(cell, th, true) [upstream
// OpenCV fast.cpp]) and simulates the kernel's pass A thread by thread.
//
// A 9-pixel arc of the 16-pixel Bresenham ring always contains one pixel of each opposite pair (k, k+8). For a pixel to be a
// corner at threshold t with a DARKER arc (all 9 ring pixels < v - t) every one of the 4 tested pairs (0,8) (4,12) (2,10) (6,14)
// therefore needs a member with v - p > t; for a BRIGHTER arc a member with p - v > t. On the ring pixels themselves:
//   darker possible   <=>  lo = max over pairs of min(p_k, p_k+8) < v - t
//   brighter possible <=>  hi = min over pairs of max(p_k, p_k+8) > v + t
// Two pixels ride in the two s16 halves of a word, so one VIMNMX(3).S16x2 evaluates two pixels at once, and no ring difference
// is formed: the two comparisons are one 3-input add each against the bias 511 - t.
#pragma once
#include <cstdint>

#if defined(__CUDACC__)
#define SE2_HD __host__ __device__ __forceinline__
#else
#define SE2_HD inline
#endif

namespace fastpx {
// packed-SIMD primitives: the PTX instruction in device code, an emulation of its semantics in host code
// (prmt.b32 default mode, per-halfword signed min/max, wrapping per-halfword add)
SE2_HD int16_t lo16(unsigned a) { return (int16_t)(a & 0xFFFF); }
SE2_HD int16_t hi16(unsigned a) { return (int16_t)(a >> 16); }
SE2_HD unsigned pack16(int lo, int hi) { return ((unsigned)lo & 0xFFFFu) | ((unsigned)hi << 16); }
SE2_HD unsigned perm(unsigned a, unsigned b, unsigned s) {
#if defined(__CUDA_ARCH__)
    return __byte_perm(a, b, s);
#else
    const uint64_t src = ((uint64_t)b << 32) | a;
    unsigned r = 0;
    for (int i = 0; i < 4; ++i) {
        const unsigned sel = (s >> (4 * i)) & 0xF;
        unsigned byte = (unsigned)(src >> (8 * (sel & 7))) & 0xFF;
        if (sel & 8) byte = (byte & 0x80) ? 0xFF : 0x00;
        r |= byte << (8 * i);
    }
    return r;
#endif
}
SE2_HD unsigned maxs2(unsigned a, unsigned b) {
#if defined(__CUDA_ARCH__)
    return __vmaxs2(a, b);
#else
    return pack16(lo16(a) > lo16(b) ? lo16(a) : lo16(b), hi16(a) > hi16(b) ? hi16(a) : hi16(b));
#endif
}
SE2_HD unsigned mins2(unsigned a, unsigned b) {
#if defined(__CUDA_ARCH__)
    return __vmins2(a, b);
#else
    return pack16(lo16(a) < lo16(b) ? lo16(a) : lo16(b), hi16(a) < hi16(b) ? hi16(a) : hi16(b));
#endif
}
SE2_HD unsigned min3s2(unsigned a, unsigned b, unsigned c) {
#if defined(__CUDA_ARCH__)
    return __vimin3_s16x2(a, b, c);
#else
    return mins2(mins2(a, b), c);
#endif
}
SE2_HD unsigned max3s2(unsigned a, unsigned b, unsigned c) {
#if defined(__CUDA_ARCH__)
    return __vimax3_s16x2(a, b, c);
#else
    return maxs2(maxs2(a, b), c);
#endif
}
SE2_HD unsigned add2(unsigned a, unsigned b) {
#if defined(__CUDA_ARCH__)
    return __vadd2(a, b);
#else
    return pack16((lo16(a) + lo16(b)) & 0xFFFF, (hi16(a) + hi16(b)) & 0xFFFF);
#endif
}
}  // namespace fastpx

namespace fastpx {

// threshold constant of screen4: the bias 511 - t in both halfwords, the same for either polarity:
//   v + bias - lo >= 512  <=>  lo < v - t ;   hi + bias - v >= 512  <=>  hi > v + t
// Every sum lies in [256 - t, 766 - t], inside a halfword and positive, so the plain 32-bit adds never carry across halves.
SE2_HD unsigned screen_bias(int t) { return (unsigned)(511 - t) * 0x10001u; }

// The 4 pixels of patch word `zc` (row y, bytes x..x+3). Neighbouring words: zl / zr = the words left / right of zc on row y,
// n3 / s3 = the word above / below at rows y-3 / y+3, n2l n2c n2r / s2l s2c s2r = the three words at rows y-2 / y+2.
// Returns bit j set <=> pixel j may be a FAST corner at the threshold encoded in bias = screen_bias(t) (necessary condition).
SE2_HD unsigned screen4(unsigned n3, unsigned s3, unsigned n2l, unsigned n2c, unsigned n2r, unsigned s2l, unsigned s2c, unsigned s2r,
                        unsigned zl, unsigned zc, unsigned zr, unsigned bias) {
    // 4-byte spans starting at dx = -3, +3 (row y) and dx = -2, +2 (rows y-2, y+2) of the word's first pixel
    const unsigned w_m3 = perm(zl, zc, 0x4321), w_p3 = perm(zc, zr, 0x6543);
    const unsigned nw_ = perm(n2l, n2c, 0x5432), ne_ = perm(n2c, n2r, 0x5432);
    const unsigned sw_ = perm(s2l, s2c, 0x5432), se_ = perm(s2c, s2r, 0x5432);
    unsigned ok[2];
#if defined(__CUDA_ARCH__)
#pragma unroll
#endif
    for (int hlf = 0; hlf < 2; ++hlf) {
        const unsigned sel = hlf ? 0x4341u : 0x4240u;      // pixels (0,2) or (1,3) -> the two s16 halves
        const unsigned v = perm(zc, 0, sel);
        const unsigned p0 = perm(s3, 0, sel), p8 = perm(n3, 0, sel);          // (0,+3) (0,-3)
        const unsigned p4 = perm(w_p3, 0, sel), p12 = perm(w_m3, 0, sel);     // (+3,0) (-3,0)
        const unsigned p2 = perm(se_, 0, sel), p10 = perm(nw_, 0, sel);       // (+2,+2) (-2,-2)
        const unsigned p6 = perm(ne_, 0, sel), p14 = perm(sw_, 0, sel);       // (+2,-2) (-2,+2)
        const unsigned lo = maxs2(max3s2(mins2(p0, p8), mins2(p4, p12), mins2(p2, p10)), mins2(p6, p14));
        const unsigned hi = mins2(min3s2(maxs2(p0, p8), maxs2(p4, p12), maxs2(p2, p10)), maxs2(p6, p14));
        ok[hlf] = ((v + bias - lo) | (hi + bias - v)) & 0x02000200u;         // bit 9 of a half <=> that pixel may be a corner
    }
    // bits 9, 10, 25, 26 = pixels 0, 1, 2, 3
    const unsigned b = ok[0] + (ok[1] << 1);
    return ((b >> 9) | (b >> 23)) & 0xFu;
}
// the form with one constant per polarity (darker T1, brighter U1) that tests/native/fast_screen_host.cpp is written against;
// both constants are the bias, so U1 == T1
SE2_HD unsigned screen_T1(int t) { return screen_bias(t); }
SE2_HD unsigned screen_U1(int t) { return screen_bias(t); }
SE2_HD unsigned screen4(unsigned n3, unsigned s3, unsigned n2l, unsigned n2c, unsigned n2r, unsigned s2l, unsigned s2c, unsigned s2r,
                        unsigned zl, unsigned zc, unsigned zr, unsigned T1, unsigned /*U1*/) {
    return screen4(n3, s3, n2l, n2c, n2r, s2l, s2c, s2r, zl, zc, zr, T1);
}

// bits j of an item of up to 8 pixels (interior x = x0 + j) that lie inside the cell interior [0, cw); needs x0 <= cw - 1 and x0 >= -7
SE2_HD unsigned inside_mask8(int x0, int cw) {
    const int lo = x0 < 0 ? -x0 : 0;
    const int hi = cw - x0 < 8 ? cw - x0 : 8;        // 1 <= hi <= 8
    return (0xFFu << lo) & (0xFFu >> (8 - hi)) & 0xFFu;
}

// ---- pass A work distribution of orb_fast_cells (shared with the host tests, which simulate the CTA's threads:
// tests/native/fast_pass_a8_host.cpp the kernel's 8-pixel items, section 3 of tests/native/fast_screen_host.cpp the earlier
// split of one 4-pixel group per item, which the kernel no longer uses)
// The patch row starts `shift` bytes left of the cell's first apron pixel (0..15 with the 16 B aligned TMA box, 0..3 with the
// 4 B aligned plain loads), so interior pixel x sits at patch byte x + 3 + shift. An item = row y of the cell x one 4-pixel group
// g = 0 .. groups_per_row - 1, i.e. patch word first_group + g, interior x = group_x0(g) .. +3.
SE2_HD int first_group(int shift) { return (shift + 3) >> 2; }
SE2_HD int groups_per_row(int cw, int shift) { return ((shift + 2 + cw) >> 2) - first_group(shift) + 1; }
SE2_HD int group_x0(int g, int shift) { return 4 * (g + first_group(shift)) - 3 - shift; }   // -3 .. cw-1
// A pass A item is 8 pixels: the groups 2i and 2i+1 of row y (patch words first_group + 2i, +1; interior x = group_x0(2i) .. +7),
// so the two screens share the 16 patch words they read. When groups_per_row is odd, the last item of a row has a second group
// past the cell: inside_mask8 drops its pixels, and its reads end at most one word past the patch's last row, inside the score
// plane that follows the patch in shared memory (its right-hand words on rows y-2 .. y+2 fall on the next patch row).
SE2_HD int items_per_row(int cw, int shift) { return (groups_per_row(cw, shift) + 1) >> 1; }
// thread tid visits items tid, tid + nthreads, tid + 2 nthreads, ... (item = y * G + g) without a division per item
struct ItemWalk {
    int y, g, dY, dG, G;
    SE2_HD void init(int tid, int nthreads, int groups) { G = groups; y = tid / G; g = tid - y * G; dY = nthreads / G; dG = nthreads - dY * G; }
    SE2_HD void next() { g += dG; y += dY; if (g >= G) { g -= G; ++y; } }
};

// ---- pass C (strict 3x3 non-maximum suppression) and pass E (emission) of orb_fast_cells
// The u8 score plane has the patch's row pitch pw (a multiple of 4, at least cw + 6) and holds cell pixel (x, y) at byte
// (y + 1) * pw + x + NMS_X0: a zero apron of 1 px around the cell, every other byte of a row zero too. Pixel x's word is then
// word x/4 + 1 of its row, so the 32 pixels of bitmap word k are the whole plane words 8k+1 .. 8k+8.
constexpr int NMS_X0 = 4;
// nms32 on the last word of a row reads up to 32 bytes past the row's end (32 * words_per_row + 8 <= cw + 39 <= pw + 33), so
// past the plane behind its last row: the plane's shared-memory block is this long
SE2_HD int nms_plane_bytes(int pw, int ch) { return pw * (ch + 2) + 32; }
// the bitmap has whole words per cell row: bit x & 31 of word y * nms_words_per_row(cw) + (x >> 5) is pixel (x, y)
SE2_HD int nms_words_per_row(int cw) { return (cw + 31) >> 5; }
// bits of bitmap word k that lie inside the cell
SE2_HD unsigned nms_row_mask(int k, int cw) { const int n = cw - 32 * k; return n >= 32 ? 0xFFFFFFFFu : (1u << n) - 1u; }

// Bitmap word k of cell row y: bit i set <=> score(32k+i, y) > all 8 neighbours (so it is nonzero). u, c, d point at plane word 8k
// of the plane rows y, y+1, y+2 (the cell rows y-1, y, y+1); each supplies the 10 words of pixels 32k-4 .. 32k+35. Scores are
// 0..255, so two pixels ride in the two 16-bit halves of a word: E = bytes (0, 2) and O = bytes (1, 3) of a plane word.
SE2_HD unsigned nms32(const uint32_t* u, const uint32_t* c, const uint32_t* d) {
    unsigned c3e[10], c3o[10];   // 3-row maxima; [0] only needs the odd bytes, [9] only the even ones
    unsigned r[4];               // 8 result bits each at bits 24..31
#if defined(__CUDA_ARCH__)
#pragma unroll
#endif
    for (int j = 0; j < 10; ++j) {
        const unsigned ua = u[j], ca = c[j], da = d[j];
        if (j > 0) c3e[j] = max3s2(perm(ua, 0, 0x4240), perm(ca, 0, 0x4240), perm(da, 0, 0x4240));
        if (j < 9) c3o[j] = max3s2(perm(ua, 0, 0x4341), perm(ca, 0, 0x4341), perm(da, 0, 0x4341));
    }
#if defined(__CUDA_ARCH__)
#pragma unroll
#endif
    for (int g = 0; g < 8; ++g) {   // pixels 4g .. 4g+3 = plane word j = g + 1
        const int j = g + 1;
        const unsigned ua = u[j], ca = c[j], da = d[j];
        const unsigned ce = perm(ca, 0, 0x4240), co = perm(ca, 0, 0x4341);                       // centres of pixels (0,2), (1,3)
        const unsigned ve = maxs2(perm(ua, 0, 0x4240), perm(da, 0, 0x4240));                   // above / below
        const unsigned vo = maxs2(perm(ua, 0, 0x4341), perm(da, 0, 0x4341));
        // pixels (0,2): left = bytes (-1, 1) = halves (hi of O_j-1, lo of O_j), right = bytes (1, 3) = O_j
        // pixels (1,3): left = bytes (0, 2) = E_j, right = bytes (2, 4) = halves (hi of E_j, lo of E_j+1)
        const unsigned ne = max3s2(perm(c3o[j - 1], c3o[j], 0x5432), ve, c3o[j]);
        const unsigned no = max3s2(c3e[j], vo, perm(c3e[j], c3e[j + 1], 0x5432));
        // 255 + centre - max in [0, 510] per half (no borrow across halves): bit 8 of the half <=> centre > max
        const unsigned te = ce + 0x00FF00FFu - ne, to = co + 0x00FF00FFu - no;
        const unsigned bytes = perm(te, to, 0x7351);            // byte i = 1 <=> pixel 4g+i is kept
        if (g & 1) {
            // bytes of pixels 4g-4 .. 4g-1 in the low nibbles, 4g .. 4g+3 in the high ones; the product's byte 3 is the 8 bits
            r[g >> 1] = (r[g >> 1] + (bytes << 4)) * 0x01020408u;
        } else {
            r[g >> 1] = bytes;
        }
    }
    return perm(perm(r[0], r[1], 0x7373), perm(r[2], r[3], 0x7373), 0x5410);
}

// passes C and E: thread tid owns the consecutive bitmap words [w, w1) in raster order, so an exclusive scan of the threads'
// keypoint counts gives every keypoint its raster-order slot; (y, k) of the word is walked, not divided per word
struct WordRun {
    int w, w1, y, k, wpr;
    SE2_HD void init(int tid, int nthreads, int ch, int words_per_row) {
        wpr = words_per_row;
        const int nw = ch * wpr, q = (nw + nthreads - 1) / nthreads;
        w = tid * q < nw ? tid * q : nw;
        w1 = w + q < nw ? w + q : nw;
        y = w / wpr; k = w - y * wpr;
    }
    SE2_HD bool more() const { return w < w1; }
    SE2_HD void next() { ++w; if (++k == wpr) { k = 0; ++y; } }
};

}  // namespace fastpx
