// Host check of se2lam_b200/csrc/fast_screen.h — the source pass A of orb_fast_cells is compiled from — with the
// packed-SIMD instructions emulated:
//   1. screen4 == the scalar definition of the FAST-9-16 quick reject, per pixel, for random and extreme patches
//   2. the screen never rejects a true FAST corner (scalar 9-contiguous-arc definition, cv::FAST [upstream OpenCV fast.cpp])
//   3. a CTA's pass A simulated warp by warp (ItemWalk, group addressing, inside_mask8, warp scan + shared counter), for the TMA
//      layout (pitch = box width, shift 0..15) and the plain-load layout (pitch rounded up to 4 B, shift 0..3): every interior
//      pixel of a cell is screened exactly once, the candidate set equals the scalar screen, list entries stay below cw*ch
//      slots and decode to their pixel, and no read leaves the patch
// Prints "OK <checks>" and exits 0, or a diagnostic and exits 1.
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <random>
#include <vector>

#include "../../se2lam_b200/csrc/fast_screen.h"

static const int RING[16][2] = {{0, 3}, {1, 3}, {2, 2}, {3, 1}, {3, 0}, {3, -1}, {2, -2}, {1, -3}, {0, -3}, {-1, -3}, {-2, -2}, {-3, -1}, {-3, 0}, {-3, 1}, {-2, 2}, {-1, 3}};

static bool scalar_screen(const uint8_t* p, int pw, int t) {   // p = centre pixel
    const int v = p[0];
    bool dk = true, br = true;
    for (int k = 0; k < 8; k += 2) {   // opposite pairs (0,8) (2,10) (4,12) (6,14)
        const int a = p[RING[k][1] * pw + RING[k][0]], b = p[RING[k + 8][1] * pw + RING[k + 8][0]];
        dk = dk && (v - a > t || v - b > t);
        br = br && (a - v > t || b - v > t);
    }
    return dk || br;
}

static bool scalar_corner(const uint8_t* p, int pw, int t) {
    const int v = p[0];
    int d[32];
    for (int k = 0; k < 16; ++k) d[k] = d[k + 16] = p[RING[k][1] * pw + RING[k][0]] - v;
    for (int s = 0; s < 16; ++s) {
        bool allb = true, alld = true;
        for (int k = 0; k < 9; ++k) { allb = allb && d[s + k] > t; alld = alld && d[s + k] < -t; }
        if (allb || alld) return true;
    }
    return false;
}

static uint32_t ldw(const uint8_t* base, long word) { uint32_t w; memcpy(&w, base + 4 * word, 4); return w; }

#define FAIL(...) do { fprintf(stderr, __VA_ARGS__); fprintf(stderr, "\n"); return 1; } while (0)

int main() {
    std::mt19937 rng(12345);
    long checks = 0;
    // ---- 1 + 2: screen4 on a 7-row x 3-word neighbourhood
    for (int iter = 0; iter < 200000; ++iter) {
        const int pw = 12;
        uint8_t buf[7 * 12];
        const int mode = iter % 5;
        for (auto& b : buf) {
            switch (mode) {
                case 0: b = (uint8_t)(rng() & 255); break;
                case 1: b = (uint8_t)(100 + (rng() % 50)); break;                       // differences near the thresholds
                case 2: b = (rng() & 1) ? 255 : 0; break;                               // extremes: |diff| = 255
                case 3: b = (uint8_t)((rng() % 3) * 21 + 90); break;                    // ties exactly at t = 20 +- 1
                default: b = (uint8_t)(((rng() >> 8) & 1) ? (rng() & 255) : 128); break;
            }
        }
        const int ts[4] = {20, 7, 1, 254};
        const int t = ts[iter % 4];
        const uint8_t* row = buf + 3 * pw;   // centre row, words 0..2; the screened word is word 1 (bytes 4..7)
        const unsigned m = fastpx::screen4(ldw(buf + 0 * pw, 1), ldw(buf + 6 * pw, 1), ldw(buf + 1 * pw, 0), ldw(buf + 1 * pw, 1), ldw(buf + 1 * pw, 2),
                                           ldw(buf + 5 * pw, 0), ldw(buf + 5 * pw, 1), ldw(buf + 5 * pw, 2), ldw(row, 0), ldw(row, 1), ldw(row, 2),
                                           fastpx::screen_T1(t), fastpx::screen_U1(t));
        for (int j = 0; j < 4; ++j) {
            const bool want = scalar_screen(row + 4 + j, pw, t);
            if ((((m >> j) & 1u) != 0) != want) FAIL("screen4 mismatch: iter %d pixel %d t %d got %u want %d", iter, j, t, (m >> j) & 1u, (int)want);
            if (scalar_corner(row + 4 + j, pw, t) && !want) FAIL("screen rejects a true corner: iter %d pixel %d t %d", iter, j, t);
            ++checks;
        }
    }
    // ---- inside_mask8 and the group distribution, exhaustively over the argument range the kernel produces (every alignment shift)
    for (int shift = 0; shift < 16; ++shift)
        for (int cw = 1; cw <= 300; ++cw) {
            std::vector<int> seen(cw, 0);
            for (int g = 0; g < fastpx::groups_per_row(cw, shift); ++g) {
                const int x0 = fastpx::group_x0(g, shift);
                if (x0 > cw - 1 || x0 < -3) FAIL("group %d of a %d px row (shift %d) starts at %d", g, cw, shift, x0);
                const unsigned m = fastpx::inside_mask8(x0, cw) & 0xFu;
                for (int j = 0; j < 4; ++j) { const bool in = x0 + j >= 0 && x0 + j < cw; if ((((m >> j) & 1u) != 0) != in) FAIL("group mask"); if (in) seen[x0 + j]++; }
                ++checks;
            }
            for (int x = 0; x < cw; ++x) if (seen[x] != 1) FAIL("groups cover pixel %d of %d (shift %d) %d times", x, cw, shift, seen[x]);
        }
    // ---- 3: pass A of one CTA (256 threads = 8 warps), simulated warp by warp exactly as the kernel addresses the patch. Warps run
    // their 32-item chunks in any interleaving; here chunk k of every warp runs before chunk k+1 of any.
    const int NT = 256, NW = 8;
    const int sizes[][2] = {{122, 75}, {101, 62}, {103, 61}, {85, 50}, {93, 50}, {75, 41}, {61, 33}, {49, 26}, {1, 1}, {5, 3}, {6, 9},
                            {230, 225}, {250, 249}, {7, 200}, {13, 1}, {229, 17}, {312, 99}, {300, 150}};
    for (int tma = 0; tma < 2; ++tma)
    for (const auto& sz : sizes) {
      for (int shift = 0; shift < (tma ? 16 : 4); ++shift) {   // alignment shift of the patch start
        const int cw = sz[0], ch = sz[1];
        // patch pitch and rows as orb_fast_cells<TMA> derives them; the TMA box is the level's widest x tallest patch, so it may
        // have more columns and rows than this cell needs
        const int pw = tma ? ((shift + cw + 6 + 15) & ~15) + 16 * (int)(rng() % 2) : (shift + cw + 6 + 3) & ~3, pww = pw / 4;
        const int ph = tma ? ch + 6 + (int)(rng() % 3) : ch + 6;
        if ((size_t)pw * ph > 65535 || (tma && (pw > 256 || ph > 256))) continue;   // the library takes such cells to orb_fast_cells<false> / _big
        std::vector<uint8_t> patch((size_t)pw * ph);
        for (int y = 0; y < ph; ++y) for (int x = 0; x < pw; ++x) patch[(size_t)y * pw + x] = (uint8_t)((((x / 5) ^ (y / 4)) & 1) * 60 + 80 + (int)(rng() % 25));
        const uint8_t* p0 = patch.data() + 3 * pw + 3 + shift;
        const int t = 20;
        const unsigned T1 = fastpx::screen_T1(t), U1 = fastpx::screen_U1(t);
        const int g0 = fastpx::first_group(shift), G = fastpx::groups_per_row(cw, shift), nitems = ch * G;
        const long nwords_patch = (long)pww * ph;
        bool read_outside = false;
        auto ld = [&](long word) { if (word < 0 || word >= nwords_patch) { read_outside = true; return 0u; } return ldw(patch.data(), word); };
        std::vector<int> visited((size_t)cw * ch, 0), cand((size_t)cw * ch, 0);
        std::vector<int> list((size_t)cw * ch, -1);
        int ncand = 0;                                  // the kernel's shared counter s_ncand
        std::vector<fastpx::ItemWalk> walk(NT);
        for (int tid = 0; tid < NT; ++tid) walk[tid].init(tid, NT, G);
        for (int it0c = 0; it0c < nitems; it0c += NW * 32)
            for (int wid = 0; wid < NW; ++wid) {
                const int it0 = it0c + wid * 32;
                if (it0 >= nitems) break;               // the warp's loop has ended (it0 < nitems is warp-uniform)
                unsigned m[32];
                int col0[32], y[32];
                for (int lane = 0; lane < 32; ++lane) {
                    fastpx::ItemWalk& it = walk[wid * 32 + lane];
                    m[lane] = 0;
                    col0[lane] = fastpx::group_x0(it.g, shift);
                    y[lane] = it.y;
                    const bool active = it.y < ch;
                    if (active != (it0 + lane < nitems)) FAIL("activity test differs from the item bound (cw %d ch %d tid %d)", cw, ch, wid * 32 + lane);
                    if (active) {
                        if (it.y * G + it.g != it0 + lane) FAIL("ItemWalk left its item sequence (cw %d ch %d tid %d)", cw, ch, wid * 32 + lane);
                        const long c = (long)(it.y + 3) * pww + it.g + g0;
                        m[lane] = fastpx::screen4(ld(c - 3 * pww), ld(c + 3 * pww), ld(c - 2 * pww - 1), ld(c - 2 * pww), ld(c - 2 * pww + 1),
                                                  ld(c + 2 * pww - 1), ld(c + 2 * pww), ld(c + 2 * pww + 1), ld(c - 1), ld(c), ld(c + 1), T1, U1);
                        if (read_outside) FAIL("pass A reads outside the patch (cw %d ch %d shift %d tma %d)", cw, ch, shift, tma);
                        const unsigned in = fastpx::inside_mask8(col0[lane], cw) & 0xFu;
                        for (int j = 0; j < 4; ++j) if ((in >> j) & 1u) visited[(size_t)it.y * cw + col0[lane] + j]++;
                        m[lane] &= in;
                    }
                    it.next();
                }
                // warp scan of the survivor counts, one atomicAdd on the shared counter, then each lane writes its survivors
                int inc[32], run = 0;
                for (int lane = 0; lane < 32; ++lane) { run += __builtin_popcount(m[lane]); inc[lane] = run; }
                if (run == 0) continue;
                const int base0 = ncand;
                ncand += run;
                for (int lane = 0; lane < 32; ++lane) {
                    int base = base0 + inc[lane] - __builtin_popcount(m[lane]);
                    const int e0 = y[lane] * pw + col0[lane];
                    for (unsigned mm = m[lane]; mm; mm &= mm - 1) {
                        const int j = __builtin_ffs((int)mm) - 1;
                        const int off = e0 + j;
                        if (off < 0 || off > 65535 || off % pw != col0[lane] + j ||off / pw != y[lane]) FAIL("bad list entry");
                        if (base >= cw * ch) FAIL("list overflow: slot %d of %d (cw %d ch %d)", base, cw * ch, cw, ch);
                        if (list[base] != -1) FAIL("list slot %d written twice", base);
                        list[base++] = off;
                        cand[(size_t)y[lane] * cw + col0[lane] + j] = 1;
                    }
                }
            }
        int nlisted = 0;
        for (int v : list) nlisted += v >= 0;
        if (nlisted != ncand) FAIL("%d list entries for a counter of %d", nlisted, ncand);
        for (int y = 0; y < ch; ++y)
            for (int x = 0; x < cw; ++x) {
                if (visited[(size_t)y * cw + x] != 1) FAIL("pixel (%d,%d) of a %dx%d cell screened %d times", x, y, cw, ch, visited[(size_t)y * cw + x]);
                const bool want = scalar_screen(p0 + y * pw + x, pw, t);
                if ((cand[(size_t)y * cw + x] != 0) != want) FAIL("candidate set differs at (%d,%d) of a %dx%d cell (tma %d)", x, y, cw, ch, tma);
                ++checks;
            }
      }
    }
    printf("OK %ld\n", checks);
    return 0;
}
