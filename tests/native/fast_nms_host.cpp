// Host check of passes C and E of orb_fast_cells as se2lam_b200/csrc/fast_screen.h defines them (nms32, nms_row_mask, WordRun,
// the score-plane layout), with the packed-SIMD instructions emulated. For every cell width 1..70 and height 1..40, in the TMA
// layout (pitch = the 16 B rounded box width, shift 0..15) and the plain-load layout (pitch rounded up to 4 B, shift 0..3), and for
// random and adversarial score planes (all zero, plateaus of equal scores, maxima at 254, isolated maxima on every cell edge and
// corner), a CTA of 256 threads is simulated: its bitmap equals the scalar strict 3x3 maximum (zero outside the cell), the
// exclusive scan of the threads' counts gives the scalar keypoint count, and the emitted (y, x, score) sequence is the scalar
// raster order. Reads past the plane stay inside nms_plane_bytes and see garbage, which must not leak into the result.
// Prints "OK <checks>" and exits 0, or a diagnostic and exits 1.
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <random>
#include <vector>

#include "../../se2lam_b200/csrc/fast_screen.h"

static const int NTHREADS = 256;   // FAST_THREADS
static const int NPATTERNS = 7;
static long checks = 0;

static void fail(const char* what, int cw, int ch, int pw, int pattern, int a, int b) {
    printf("FAIL %s: cw %d ch %d pw %d pattern %d (%d, %d)\n", what, cw, ch, pw, pattern, a, b);
    exit(1);
}

// the cell's scores S[y * cw + x], 0..254 as pass B stores them (M - 1 with M <= 255)
static void fill(std::vector<int>& S, int cw, int ch, int pattern, std::mt19937& rng) {
    S.assign((size_t)cw * ch, 0);
    for (int y = 0; y < ch; ++y)
        for (int x = 0; x < cw; ++x) {
            int& s = S[(size_t)y * cw + x];
            const unsigned r = rng();
            switch (pattern) {
            case 0: s = (r & 1) ? (int)((r >> 1) % 255) : 0; break;                        // half the pixels scored
            case 1: s = 0; break;                                                            // nothing scored
            case 2: s = ((x / 3 + y / 2) & 1) ? 8 : ((r & 7) == 0 ? 9 : 7); break;           // plateaus, a few single bumps
            case 3: s = (r % 3 == 0) ? 0 : 253 + (int)((r >> 4) & 1); break;                 // 253 / 254 next to each other
            case 4: {                                                                        // isolated maxima on the cell's edges
                const bool edge = x == 0 || y == 0 || x == cw - 1 || y == ch - 1;
                s = edge && ((x + y) % 2 == 0) ? 1 + (int)(r % 254) : 0;
                if ((x == 0 || x == cw - 1) && (y == 0 || y == ch - 1)) s = 254;             // corners
                break;
            }
            case 5: s = (r % 10 == 0) ? 1 + (int)((r >> 8) % 254) : 0; break;               // sparse
            default: s = ((x + y) & 1) ? 0 : 1 + (int)((r >> 8) % 254); break;              // checkerboard of maxima
            }
        }
}

static void check_cell(int cw, int ch, int pw, int pattern, std::mt19937& rng) {
    std::vector<int> S;
    fill(S, cw, ch, pattern, rng);
    const int pww = pw / 4, wpr = fastpx::nms_words_per_row(cw), nw = ch * wpr;
    const int bytes = fastpx::nms_plane_bytes(pw, ch);
    // every word nms32 reads: rows y..y+2 of the plane, words 8k .. 8k+9
    if (((ch + 1) * pww + 8 * (wpr - 1) + 10) * 4 > bytes) fail("read past nms_plane_bytes", cw, ch, pw, pattern, bytes, 0);
    std::vector<uint32_t> mem((bytes + 3) / 4);
    uint8_t* plane = reinterpret_cast<uint8_t*>(mem.data());
    memset(plane, 0, (size_t)pw * (ch + 2));
    for (int i = pw * (ch + 2); i < (int)mem.size() * 4; ++i) plane[i] = (uint8_t)(1 + rng() % 255);   // not cleared by the kernel
    for (int y = 0; y < ch; ++y)
        for (int x = 0; x < cw; ++x) plane[(y + 1) * pw + x + fastpx::NMS_X0] = (uint8_t)S[(size_t)y * cw + x];

    // scalar: strict 3x3 maximum, neighbours outside the cell are 0; raster order
    std::vector<uint32_t> ref_bitmap(nw, 0u);
    std::vector<int> ref_out;   // (y << 20) | (x << 8) | score
    for (int y = 0; y < ch; ++y)
        for (int x = 0; x < cw; ++x) {
            const int s = S[(size_t)y * cw + x];
            bool keep = true;
            for (int dy = -1; dy <= 1; ++dy)
                for (int dx = -1; dx <= 1; ++dx) {
                    if (!dx && !dy) continue;
                    const int xx = x + dx, yy = y + dy;
                    const int n = (xx < 0 || yy < 0 || xx >= cw || yy >= ch) ? 0 : S[(size_t)yy * cw + xx];
                    keep = keep && s > n;
                }
            if (keep) { ref_bitmap[y * wpr + (x >> 5)] |= 1u << (x & 31); ref_out.push_back((y << 20) | (x << 8) | s); }
        }

    // the CTA: pass C per thread, the exclusive scan, pass E per thread
    std::vector<uint32_t> bitmap(nw, 0xDEADBEEFu);
    std::vector<int> cnt(NTHREADS, 0), written(nw, 0);
    for (int t = 0; t < NTHREADS; ++t) {
        fastpx::WordRun r;
        r.init(t, NTHREADS, ch, wpr);
        for (; r.more(); r.next()) {
            if (r.y * wpr + r.k != r.w || r.k >= wpr || r.y >= ch) fail("word walk", cw, ch, pw, pattern, t, r.w);
            const uint32_t* u = mem.data() + r.y * pww + 8 * r.k;
            const unsigned bits = fastpx::nms32(u, u + pww, u + 2 * pww) & fastpx::nms_row_mask(r.k, cw);
            bitmap[r.w] = bits;
            ++written[r.w];
            cnt[t] += __builtin_popcount(bits);
        }
    }
    for (int w = 0; w < nw; ++w) {
        if (written[w] != 1) fail("word not written exactly once", cw, ch, pw, pattern, w, written[w]);
        if (bitmap[w] != ref_bitmap[w]) fail("bitmap word", cw, ch, pw, pattern, w, (int)(bitmap[w] ^ ref_bitmap[w]));
    }
    int total = 0;
    std::vector<int> out(ref_out.size() + 1, -1);
    for (int t = 0; t < NTHREADS; ++t) {
        int pos = total;
        total += cnt[t];
        fastpx::WordRun r;
        r.init(t, NTHREADS, ch, wpr);
        for (; r.more(); r.next()) {
            uint32_t bits = bitmap[r.w];
            const uint8_t* srow = plane + (r.y + 1) * pw + fastpx::NMS_X0 + 32 * r.k;
            while (bits) {
                const int i = __builtin_ctz(bits);
                bits &= bits - 1;
                if (pos >= (int)ref_out.size()) fail("slot past the count", cw, ch, pw, pattern, pos, (int)ref_out.size());
                out[pos++] = (r.y << 20) | ((32 * r.k + i) << 8) | srow[i];
            }
        }
    }
    if (total != (int)ref_out.size()) fail("count", cw, ch, pw, pattern, total, (int)ref_out.size());
    for (size_t i = 0; i < ref_out.size(); ++i)
        if (out[i] != ref_out[i]) fail("emitted keypoint", cw, ch, pw, pattern, (int)i, out[i]);
    ++checks;
}

int main() {
    std::mt19937 rng(12345);
    int n = 0;
    for (int cw = 1; cw <= 70; ++cw)
        for (int ch = 1; ch <= 40; ++ch) {
            for (int shift = 0; shift < 16; ++shift) check_cell(cw, ch, (shift + cw + 6 + 15) & ~15, n++ % NPATTERNS, rng);   // TMA
            for (int shift = 0; shift < 4; ++shift) check_cell(cw, ch, (shift + cw + 6 + 3) & ~3, n++ % NPATTERNS, rng);      // plain
        }
    // every pattern at the tightest pitch of a few sizes, including a TMA box wider than the cell needs
    const int sizes[][2] = {{1, 1}, {26, 26}, {32, 9}, {33, 17}, {64, 40}, {70, 40}, {122, 75}};
    for (const auto& s : sizes)
        for (int pattern = 0; pattern < NPATTERNS; ++pattern)
            for (int pw : {(s[0] + 6 + 3) & ~3, ((s[0] + 6 + 15) & ~15) + 32}) check_cell(s[0], s[1], pw, pattern, rng);
    printf("OK %ld\n", checks);
    return 0;
}
