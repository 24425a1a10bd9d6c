// Host simulation of pass A of orb_fast_cells as the kernel splits it: 8-pixel items (two patch words of one cell row, fastpx::
// items_per_row per row, walked with fastpx::ItemWalk), each screened by two fastpx::screen4 calls on 16 shared patch words, masked
// with fastpx::inside_mask8, and compacted into the candidate list by one shared atomicAdd per lane. For the TMA layout (pitch =
// box width, shift 0..15, box rows >= the cell's) and the plain-load layout (pitch rounded up to 4 B, shift 0..3):
//   - every interior pixel of the cell is screened exactly once and the candidate set equals the scalar quick reject
//   - list entries stay below cw*ch slots, no slot is written twice, and each entry decodes to its pixel
//   - reads stay inside the patch, or at most one word past its end (the score plane follows the patch in shared memory)
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
    for (int k = 0; k < 8; k += 2) {
        const int a = p[RING[k][1] * pw + RING[k][0]], b = p[RING[k + 8][1] * pw + RING[k + 8][0]];
        dk = dk && (v - a > t || v - b > t);
        br = br && (a - v > t || b - v > t);
    }
    return dk || br;
}

#define FAIL(...) do { fprintf(stderr, __VA_ARGS__); fprintf(stderr, "\n"); return 1; } while (0)

int main() {
    std::mt19937 rng(4321);
    long checks = 0;
    const int NT = 256, NW = 8;
    const int sizes[][2] = {{122, 75}, {101, 62}, {103, 61}, {85, 50}, {93, 50}, {75, 41}, {61, 33}, {49, 26}, {1, 1}, {2, 2}, {5, 3}, {6, 9},
                            {9, 4}, {230, 225}, {250, 249}, {7, 200}, {13, 1}, {229, 17}, {312, 99}, {300, 150}};
    const int ts[4] = {20, 7, 1, 254};
    for (int tma = 0; tma < 2; ++tma)
    for (const auto& sz : sizes)
    for (int shift = 0; shift < (tma ? 16 : 4); ++shift) {
        const int cw = sz[0], ch = sz[1];
        // patch pitch and rows as orb_fast_cells<TMA> derives them; the TMA box is the level's widest x tallest patch
        const int pw = tma ? ((shift + cw + 6 + 15) & ~15) + 16 * (int)(rng() % 2) : (shift + cw + 6 + 3) & ~3, pww = pw / 4;
        const int ph = tma ? ch + 6 + (int)(rng() % 3) : ch + 6;
        if ((size_t)pw * ph > 65535 || (tma && (pw > 256 || ph > 256))) continue;   // the library takes such cells to orb_fast_cells<false> / _big
        const long nwords_patch = (long)pww * ph;
        std::vector<uint8_t> smem((size_t)pw * ph + 64);   // the patch, then (a stand-in for) the score plane
        for (int y = 0; y < ph; ++y)
            for (int x = 0; x < pw; ++x)
                smem[(size_t)y * pw + x] = (uint8_t)((((x / 5) ^ (y / 4)) & 1) * 60 + 80 + (int)(rng() % 25));
        const uint8_t* p0 = smem.data() + 3 * pw + 3 + shift;
        const int t = ts[(cw + shift) % 4];
        const unsigned bias = fastpx::screen_bias(t);
        const int g0 = fastpx::first_group(shift), G = fastpx::items_per_row(cw, shift), nitems = ch * G;
        long max_word = -1;
        bool read_below = false;
        auto ld = [&](long w) { if (w < 0) { read_below = true; return 0u; } if (w > max_word) max_word = w; uint32_t v; memcpy(&v, smem.data() + 4 * w, 4); return v; };
        std::vector<int> visited((size_t)cw * ch, 0), cand((size_t)cw * ch, 0), list((size_t)cw * ch, -1);
        int ncand = 0;
        std::vector<fastpx::ItemWalk> walk(NT);
        for (int tid = 0; tid < NT; ++tid) walk[tid].init(tid, NT, G);
        for (int it0c = 0; it0c < nitems; it0c += NW * 32)
            for (int wid = 0; wid < NW; ++wid) {
                const int it0 = it0c + wid * 32;
                if (it0 >= nitems) break;
                for (int lane = 0; lane < 32; ++lane) {   // the lanes' atomicAdds land in some order; lane order here
                    fastpx::ItemWalk& it = walk[wid * 32 + lane];
                    unsigned m = 0;
                    const int col0 = fastpx::group_x0(2 * it.g, shift);
                    const bool active = it.y < ch;
                    if (active != (it0 + lane < nitems)) FAIL("activity test differs from the item bound (cw %d ch %d tid %d)", cw, ch, wid * 32 + lane);
                    if (active) {
                        if (it.y * G + it.g != it0 + lane) FAIL("ItemWalk left its item sequence (cw %d ch %d tid %d)", cw, ch, wid * 32 + lane);
                        if (col0 < -3 || col0 > cw - 1) FAIL("item starts at x %d of a %d px row (shift %d)", col0, cw, shift);
                        const long c = (long)(it.y + 3) * pww + 2 * it.g + g0;
                        const unsigned n2a = ld(c - 2 * pww - 1), n2b = ld(c - 2 * pww), n2c = ld(c - 2 * pww + 1), n2d = ld(c - 2 * pww + 2);
                        const unsigned s2a = ld(c + 2 * pww - 1), s2b = ld(c + 2 * pww), s2c = ld(c + 2 * pww + 1), s2d = ld(c + 2 * pww + 2);
                        const unsigned za = ld(c - 1), zb = ld(c), zc = ld(c + 1), zd = ld(c + 2);
                        m = (fastpx::screen4(ld(c - 3 * pww), ld(c + 3 * pww), n2a, n2b, n2c, s2a, s2b, s2c, za, zb, zc, bias) |
                             fastpx::screen4(ld(c - 3 * pww + 1), ld(c + 3 * pww + 1), n2b, n2c, n2d, s2b, s2c, s2d, zb, zc, zd, bias) << 4) &
                            fastpx::inside_mask8(col0, cw);
                        const unsigned in = fastpx::inside_mask8(col0, cw);
                        for (int j = 0; j < 8; ++j) if ((in >> j) & 1u) visited[(size_t)it.y * cw + col0 + j]++;
                    }
                    int slot = ncand;
                    ncand += __builtin_popcount(m);
                    const int e0 = it.y * pw + col0;
                    for (int j = 0; j < 8; ++j) {
                        if (!((m >> j) & 1u)) continue;
                        const int off = e0 + j;
                        if (off < 0 || off > 65535 || off % pw != col0 + j || off / pw != it.y) FAIL("bad list entry");
                        if (slot >= cw * ch) FAIL("list overflow: slot %d of %d (cw %d ch %d)", slot, cw * ch, cw, ch);
                        if (list[slot] != -1) FAIL("list slot %d written twice", slot);
                        list[slot++] = off;
                        cand[(size_t)it.y * cw + col0 + j] = 1;
                    }
                    it.next();
                }
            }
        if (read_below) FAIL("pass A reads before the patch (cw %d ch %d shift %d tma %d)", cw, ch, shift, tma);
        if (max_word > nwords_patch) FAIL("pass A reads word %ld of a %ld-word patch (cw %d ch %d shift %d tma %d)", max_word, nwords_patch, cw, ch, shift, tma);
        for (int y = 0; y < ch; ++y)
            for (int x = 0; x < cw; ++x) {
                if (visited[(size_t)y * cw + x] != 1) FAIL("pixel (%d,%d) of a %dx%d cell screened %d times", x, y, cw, ch, visited[(size_t)y * cw + x]);
                const bool want = scalar_screen(p0 + y * pw + x, pw, t);
                if ((cand[(size_t)y * cw + x] != 0) != want) FAIL("candidate set differs at (%d,%d) of a %dx%d cell (tma %d shift %d)", x, y, cw, ch, tma, shift);
                ++checks;
            }
    }
    printf("OK %ld\n", checks);
    return 0;
}
