// Explicitly rounded float arithmetic for kernels that restate the reference's host float expressions operation by
// operation (geom.cu, loc.cu): the compiler cannot contract a multiply and an add the host keeps apart.
#pragma once

namespace se2gpu {

struct F3 { float x, y, z; };

__device__ __forceinline__ float fm(float a, float b) { return __fmul_rn(a, b); }
__device__ __forceinline__ float fa(float a, float b) { return __fadd_rn(a, b); }
__device__ __forceinline__ float fs(float a, float b) { return __fsub_rn(a, b); }
__device__ __forceinline__ float fd(float a, float b) { return __fdiv_rn(a, b); }

// cvu::se3map: Matx33f * Point3f (float sums from 0) + t
__device__ __forceinline__ F3 se3map(const float* T, F3 p) {
    float r[3];
#pragma unroll
    for (int i = 0; i < 3; i++) r[i] = fa(fa(fa(0.f, fm(T[i * 4], p.x)), fm(T[i * 4 + 1], p.y)), fm(T[i * 4 + 2], p.z));
    return {fa(r[0], T[3]), fa(r[1], T[7]), fa(r[2], T[11])};
}

// cvu::camprjc: Matx33f(K) * Point3f (float sums from 0), then (x / z, y / z)
__device__ __forceinline__ void camprjc(const float* K, F3 p, float* u, float* v) {
    float r[3];
#pragma unroll
    for (int i = 0; i < 3; i++) r[i] = fa(fa(fa(0.f, fm(K[i * 3], p.x)), fm(K[i * 3 + 1], p.y)), fm(K[i * 3 + 2], p.z));
    *u = fd(r[0], r[2]);
    *v = fd(r[1], r[2]);
}

}  // namespace se2gpu
