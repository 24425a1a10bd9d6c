// FAST-9-16 necessary condition on packed ring differences, 4 pixels (one 32-bit patch word) at a time.
//
// Shared by the CUDA kernels (orb.cu: pass A of both instantiations of orb_fast_cells) and by a host unit test
// (tests/native/fast_screen_host.cpp), which compiles THIS source with the packed-SIMD intrinsics emulated, checks it against the
// scalar definition of cv::FAST's quick reject (reference src/ORBextractor.cpp:616-623 -> cv::FAST(cell, th, true) [upstream
// OpenCV fast.cpp]) and simulates the kernel's pass A thread by thread.
//
// A 9-pixel arc of the 16-pixel Bresenham ring always contains one pixel of each opposite pair (k, k+8). For a pixel to be a
// corner at threshold t with a DARKER arc (all 9 ring pixels < v - t) every one of the 4 tested pairs (0,8) (4,12) (2,10) (6,14)
// therefore needs a member with v - p > t; for a BRIGHTER arc a member with p - v > t. With e_k = 256 + v - p_k (in [1, 511]):
//   darker possible   <=>  min over pairs of max(e_k, e_k+8) > 256 + t
//   brighter possible <=>  max over pairs of min(e_k, e_k+8) < 256 - t
// Two pixels ride in the two s16 halves of a word, so one VIMNMX(3).S16x2 evaluates two pixels at once.
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

// threshold constants of screen4 (per halfword): D + T1 >= 0 (s16) <=> D > 256 + t ;  U1 + ~B >= 0 <=> B < 256 - t
SE2_HD unsigned screen_T1(int t) { return (unsigned)(0x10000 - (257 + t)) * 0x10001u; }
SE2_HD unsigned screen_U1(int t) { return (unsigned)(256 - t) * 0x10001u; }

// The 4 pixels of patch word `zc` (row y, bytes x..x+3). Neighbouring words: zl / zr = the words left / right of zc on row y,
// n3 / s3 = the word above / below at rows y-3 / y+3, n2l n2c n2r / s2l s2c s2r = the three words at rows y-2 / y+2.
// Returns bit j set <=> pixel j may be a FAST corner at the threshold encoded in T1/U1 (necessary condition).
SE2_HD unsigned screen4(unsigned n3, unsigned s3, unsigned n2l, unsigned n2c, unsigned n2r, unsigned s2l, unsigned s2c, unsigned s2r,
                        unsigned zl, unsigned zc, unsigned zr, unsigned T1, unsigned U1) {
    // 4-byte spans starting at dx = -3, +3 (row y) and dx = -2, +2 (rows y-2, y+2) of the word's first pixel
    const unsigned w_m3 = perm(zl, zc, 0x4321), w_p3 = perm(zc, zr, 0x6543);
    const unsigned nw_ = perm(n2l, n2c, 0x5432), ne_ = perm(n2c, n2r, 0x5432);
    const unsigned sw_ = perm(s2l, s2c, 0x5432), se_ = perm(s2c, s2r, 0x5432);
    unsigned m = 0;
#if defined(__CUDA_ARCH__)
#pragma unroll
#endif
    for (int hlf = 0; hlf < 2; ++hlf) {
        const unsigned sel = hlf ? 0x4342u : 0x4140u;      // pixels (0,1) or (2,3) -> the two s16 halves
        const unsigned cb = perm(zc, 0, sel) + 0x01000100u;                                  // 256 + v
        // e = 256 + v - ring (both halves stay in [1,511], so the plain subtraction never borrows)
        const unsigned e0 = cb - perm(s3, 0, sel), e8 = cb - perm(n3, 0, sel);               // (0,+3) (0,-3)
        const unsigned e4 = cb - perm(w_p3, 0, sel), e12 = cb - perm(w_m3, 0, sel);          // (+3,0) (-3,0)
        const unsigned e2 = cb - perm(se_, 0, sel), e10 = cb - perm(nw_, 0, sel);            // (+2,+2) (-2,-2)
        const unsigned e6 = cb - perm(ne_, 0, sel), e14 = cb - perm(sw_, 0, sel);            // (+2,-2) (-2,+2)
        const unsigned D = mins2(min3s2(maxs2(e0, e8), maxs2(e4, e12), maxs2(e2, e10)), maxs2(e6, e14));
        const unsigned B = maxs2(max3s2(mins2(e0, e8), mins2(e4, e12), mins2(e2, e10)), mins2(e6, e14));
        const unsigned r = maxs2(add2(D, T1), add2(~B, U1));                                 // >= 0 per half <=> may be a corner
        const unsigned ok = ~r & 0x80008000u;
        m |= ((ok >> 15) & 1u) << (2 * hlf) | ((ok >> 31) & 1u) << (2 * hlf + 1);
    }
    return m;
}

// bits j of an item of up to 8 pixels (interior x = x0 + j) that lie inside the cell interior [0, cw); needs x0 <= cw - 1 and x0 >= -7
SE2_HD unsigned inside_mask8(int x0, int cw) {
    const int lo = x0 < 0 ? -x0 : 0;
    const int hi = cw - x0 < 8 ? cw - x0 : 8;        // 1 <= hi <= 8
    return (0xFFu << lo) & (0xFFu >> (8 - hi)) & 0xFFu;
}

// ---- pass A work distribution of orb_fast_cells (shared with the host test, which simulates the CTA's threads)
// The patch row starts `shift` bytes left of the cell's first apron pixel (0..15 with the 16 B aligned TMA box, 0..3 with the
// 4 B aligned plain loads), so interior pixel x sits at patch byte x + 3 + shift. An item = row y of the cell x one 4-pixel group
// g = 0 .. groups_per_row - 1, i.e. patch word first_group + g, interior x = group_x0(g) .. +3.
SE2_HD int first_group(int shift) { return (shift + 3) >> 2; }
SE2_HD int groups_per_row(int cw, int shift) { return ((shift + 2 + cw) >> 2) - first_group(shift) + 1; }
SE2_HD int group_x0(int g, int shift) { return 4 * (g + first_group(shift)) - 3 - shift; }   // -3 .. cw-1
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
