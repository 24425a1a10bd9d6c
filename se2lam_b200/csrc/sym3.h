// Closed-form inverse of a symmetric 3x3 block, shared by the landmark damping terms of the BA (ba.cu) and the pivot blocks
// of both block LDL^T solvers (ba.cu, ba_band.cu). Internal to libse2gpu.
#pragma once
#include <cuda_runtime.h>

// [a b c; b e f; c f i]^-1 by cofactors over the determinant. pd: the leading principal minors a, a e - b^2 and det are
// positive (CHOLMOD's "not positive definite" test of a pivot block).
struct Sym3Inv {
    double i00, i01, i02, i11, i12, i22;
    bool pd;
};
__device__ __forceinline__ Sym3Inv sym3_inverse(double a, double b, double c, double e, double f, double i) {
    const double c00 = e * i - f * f, c01 = c * f - b * i, c02 = b * f - c * e;
    const double det = a * c00 + b * c01 + c * c02, m2 = a * e - b * b;
    const double id = 1.0 / det;
    return Sym3Inv{c00 * id, c01 * id, c02 * id, (a * i - c * c) * id, (b * c - a * f) * id, m2 * id,
                   (a > 0.0) && (m2 > 0.0) && (det > 0.0) && isfinite(det)};
}
