// Host build of se2lam_b200/csrc/resp_key.h: the key's unsigned order is the float order over every float class
// (+-0, denormals, normals, +-FLT_MAX, +-inf) and across neighbouring floats of both signs; -0 and +0 share a key;
// resp_from_key inverts it. Exit code 0 = all checks passed.
#include <cfloat>
#include <cmath>
#include <cstdio>
#include <cstring>
#include <random>
#include <vector>

#include "../../se2lam_b200/csrc/resp_key.h"

using se2gpu::resp_key;
using se2gpu::resp_from_key;

static float from_bits(uint32_t u) { float f; memcpy(&f, &u, 4); return f; }
static uint32_t to_bits(float f) { uint32_t u; memcpy(&u, &f, 4); return u; }

static long g_checks = 0;
static bool pair_ok(float a, float b) {
    ++g_checks;
    const uint32_t ka = resp_key(a), kb = resp_key(b);
    if ((a < b) != (ka < kb) || (a == b) != (ka == kb) || (a > b) != (ka > kb)) {
        fprintf(stderr, "order differs: %a (key %08x) vs %a (key %08x)\n", a, ka, b, kb);
        return false;
    }
    const float ra = resp_from_key(ka);
    if (!(ra == a) || (a != 0.f && to_bits(ra) != to_bits(a))) { fprintf(stderr, "round trip of %a gives %a\n", a, ra); return false; }
    return true;
}

int main() {
    std::vector<float> v = {0.f, -0.f, FLT_MIN, -FLT_MIN, FLT_MAX, -FLT_MAX, INFINITY, -INFINITY, FLT_TRUE_MIN, -FLT_TRUE_MIN,
                            1.f, -1.f, 0.04f, -0.04f, 3.8477533e-16f, -3.8477533e-16f};
    // neighbours across classes and signs: the first and last denormals, the normal/denormal boundary, 1.0, FLT_MAX
    for (uint32_t base : {0x00000000u, 0x00000001u, 0x007FFFFFu, 0x00800000u, 0x3F800000u, 0x7F7FFFFFu})
        for (int d = -3; d <= 3; ++d) {
            const uint32_t u = base + (uint32_t)d;
            if ((u & 0x7F800000u) == 0x7F800000u && (u & 0x007FFFFFu)) continue;   // NaN
            v.push_back(from_bits(u & 0x7FFFFFFFu)); v.push_back(-from_bits(u & 0x7FFFFFFFu));
        }
    std::mt19937 rng(5);
    for (int i = 0; i < 4000; ++i) {
        uint32_t u = rng();
        if ((u & 0x7F800000u) == 0x7F800000u) continue;
        v.push_back(from_bits(u));
        v.push_back(from_bits(u) * 0.5f);   // nearby magnitudes, same sign
    }
    for (size_t i = 0; i < v.size(); ++i)
        for (size_t j = 0; j < v.size(); j += 1 + (v.size() > 2000) * 7)
            if (!pair_ok(v[i], v[j])) return 1;
    if (resp_key(-0.f) != resp_key(0.f)) { fprintf(stderr, "-0 and +0 keys differ\n"); return 1; }
    // every float in consecutive bit order from -FLT_MAX towards +FLT_MAX, sampled: keys strictly increase
    uint32_t prev = 0;
    bool first = true;
    for (int64_t i = -(int64_t)0x7F7FFFFF; i <= 0x7F7FFFFF; i += 4093) {
        const float f = i < 0 ? -from_bits((uint32_t)(-i)) : from_bits((uint32_t)i);
        const uint32_t k = resp_key(f);
        if (!first && k <= prev) { fprintf(stderr, "key not increasing at %a\n", f); return 1; }
        prev = k; first = false; ++g_checks;
    }
    printf("resp_key: %ld checks order-preserving\n", g_checks);
    return 0;
}
