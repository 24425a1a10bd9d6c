// Pins the 64-bit instantiation of se2lam_b200/csrc/introselect.h (records resp_key(response) << 32 | id, key = the upper
// word: the Harris-score selection) against this toolchain's std::nth_element with a float response-greater comparator, on
// tie-heavy float lists with negative values and +-0. Exit code 0 = identical permutations everywhere.
#include <algorithm>
#include <cstdio>
#include <random>
#include <vector>

#include "../../se2lam_b200/csrc/introselect.h"
#include "../../se2lam_b200/csrc/resp_key.h"

struct KP { float response; int id; };
struct Greater { bool operator()(const KP& a, const KP& b) const { return a.response > b.response; } };

static bool check(const std::vector<float>& r, int nth) {
    const int n = (int)r.size();
    std::vector<KP> ref(n);
    std::vector<uint64_t> mine(n);
    for (int i = 0; i < n; ++i) { ref[i] = KP{r[i], i}; mine[i] = ((uint64_t)se2gpu::resp_key(r[i]) << 32) | (uint32_t)i; }
    std::nth_element(ref.begin(), ref.begin() + nth, ref.end(), Greater());
    se2gpu::kp_nth_element<se2gpu::KpKey64>(mine.data(), n, nth);
    for (int i = 0; i < n; ++i)
        if ((int)(uint32_t)mine[i] != ref[i].id) {
            fprintf(stderr, "mismatch n=%d nth=%d at %d: mine id %u ref id %d\n", n, nth, i, (uint32_t)mine[i], ref[i].id);
            return false;
        }
    return true;
}

int main() {
    std::mt19937 rng(777);
    long cases = 0;
    for (int rep = 0; rep < 20000; ++rep) {
        const int n = 1 + rng() % 700;
        const int range = 1 + rng() % (rep % 3 == 0 ? 4 : (rep % 3 == 1 ? 40 : 5000));
        std::vector<float> s(n);
        for (auto& x : s) {
            const int q = (int)(rng() % range) - range / 2;
            x = q == 0 ? ((rng() & 1) ? -0.f : 0.f) : (float)q * 1.5e-3f;    // negatives, +-0 and many exact ties
        }
        if (rep % 7 == 0) std::sort(s.begin(), s.end());
        if (rep % 11 == 0) std::sort(s.rbegin(), s.rend());
        if (!check(s, rng() % n)) return 1;
        ++cases;
    }
    for (int n = 4; n < 3000; n += 37) {   // organ pipe: deep recursion, heap-select fallback
        std::vector<float> o(n);
        for (int i = 0; i < n; ++i) o[i] = (float)(std::min(i, n - 1 - i) % 240) - 120.f;
        for (int nth : {0, n / 3, n / 2, n - 1}) { if (!check(o, nth)) return 1; ++cases; }
    }
    printf("introselect64: %ld cases identical to std::nth_element\n", cases);
    return 0;
}
