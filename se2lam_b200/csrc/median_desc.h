// The median-descriptor selection of MapPoint::updateMainKFandDescriptor (reference src/MapPoint.cpp:228-272), shared by
// se2gpu_median_descriptor (bow.cu) and the map-point updates (geom.cu): the Hamming distance matrix of N descriptors and
// the rank-counting selection of the element std::sort would put at index int(0.5*(N-1)) of one of its rows.
#pragma once
#include <cstdint>

#include "common.h"

namespace se2gpu {

// dist [N*N] (row-major, zero diagonal) of the descriptors desc + 8*row(i), i < N; thread t of nt fills every nt-th entry
template <class Row>
__device__ __forceinline__ void hamming_matrix(const uint32_t* __restrict__ desc, Row row, int N, unsigned short* dist, int t, int nt) {
    for (int e = t; e < N * N; e += nt) {
        const int i = e / N, j = e - i * N;
        dist[e] = (unsigned short)(i == j ? 0 : hamming256(desc + 8 * (size_t)row(i), desc + 8 * (size_t)row(j)));
    }
}

// the value at index kth of row[0..N) in ascending order
__device__ __forceinline__ int rank_select(const unsigned short* row, int N, int kth) {
    for (int j = 0; j < N; ++j) {
        const int v = row[j];
        int less = 0, leq = 0;
        for (int t = 0; t < N; ++t) { less += row[t] < v; leq += row[t] <= v; }
        if (less <= kth && kth < leq) return v;
    }
    return 0;
}

}  // namespace se2gpu
