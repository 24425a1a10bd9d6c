// Deterministic re-implementation of libstdc++'s std::nth_element (introselect) for packed keypoint records (32-bit
// FAST-score records, 64-bit Harris-response records), usable from host and device code.
//
// Why: cv::KeyPointsFilter::retainBest (called at reference src/ORBextractor.cpp:692 and :708) is
// std::nth_element(begin, begin+n-1, end, response-greater) followed by a std::partition of the tail
// that se2lam immediately truncates away (keysCell.resize / keypoints.resize, :693-694, :709). FAST
// scores are small integers, so ties are everywhere and WHICH tied keypoints survive — and the order
// of the survivors — is whatever permutation libstdc++'s introselect produces. To be bit-exact with
// the reference the device must reproduce that permutation, not just the selected set:
//   median-of-three pivot moved to front, unguarded Hoare partition, depth limit 2*floor(log2 n) with
//   heap-select fallback, insertion sort for ranges of <= 3.
// tests/test_introselect.py pins this file against the real std::nth_element of this toolchain.
#pragma once
#include <stdint.h>

#if defined(__CUDACC__)
#define SE2_HD __host__ __device__ __forceinline__
#else
#define SE2_HD inline
#endif

namespace se2gpu {

// Record types and their keys: comp(a,b) == (key(a) > key(b)), records with equal keys are ties.
//   KpScore32  FAST score mode: 32-bit record score:8|y:12|x:12, key = the score in the top 8 bits
//   KpKey64    Harris score mode: 64-bit record resp_key(response) << 32 | (score:8|y:12|x:12), key = the upper word
struct KpScore32 {
    typedef uint32_t rec;
    static SE2_HD unsigned key(uint32_t r) { return r >> 24; }
};
struct KpKey64 {
    typedef uint64_t rec;
    static SE2_HD unsigned key(uint64_t r) { return (unsigned)(r >> 32); }
};

template <class K = KpScore32>
SE2_HD bool kp_greater(typename K::rec a, typename K::rec b) { return K::key(a) > K::key(b); }

template <class K = KpScore32>
SE2_HD void kp_swap(typename K::rec* v, int i, int j) { typename K::rec t = v[i]; v[i] = v[j]; v[j] = t; }

template <class K = KpScore32>
SE2_HD void kp_adjust_heap(typename K::rec* first, int holeIndex, int len, typename K::rec value) {
    const int topIndex = holeIndex;
    int secondChild = holeIndex;
    while (secondChild < (len - 1) / 2) {
        secondChild = 2 * (secondChild + 1);
        if (kp_greater<K>(first[secondChild], first[secondChild - 1])) secondChild--;
        first[holeIndex] = first[secondChild];
        holeIndex = secondChild;
    }
    if ((len & 1) == 0 && secondChild == (len - 2) / 2) {
        secondChild = 2 * (secondChild + 1);
        first[holeIndex] = first[secondChild - 1];
        holeIndex = secondChild - 1;
    }
    int parent = (holeIndex - 1) / 2;
    while (holeIndex > topIndex && kp_greater<K>(first[parent], value)) {
        first[holeIndex] = first[parent];
        holeIndex = parent;
        parent = (holeIndex - 1) / 2;
    }
    first[holeIndex] = value;
}

// std::__heap_select(first, middle, last)
template <class K = KpScore32>
SE2_HD void kp_heap_select(typename K::rec* v, int first, int middle, int last) {
    typename K::rec* f = v + first;
    const int len = middle - first;
    if (len >= 2) {
        int parent = (len - 2) / 2;
        while (true) {
            typename K::rec value = f[parent];
            kp_adjust_heap<K>(f, parent, len, value);
            if (parent == 0) break;
            parent--;
        }
    }
    for (int i = middle; i < last; ++i)
        if (kp_greater<K>(v[i], v[first])) {
            typename K::rec value = v[i];
            v[i] = v[first];
            kp_adjust_heap<K>(f, 0, len, value);
        }
}

// std::nth_element(v+0, v+nth, v+n, greater-by-key)
template <class K = KpScore32>
SE2_HD void kp_nth_element(typename K::rec* v, int n, int nth) {
    if (n <= 0 || nth >= n) return;
    int first = 0, last = n;
    int depth = 0;
    for (int t = n; t > 1; t >>= 1) ++depth;  // std::__lg(n)
    depth *= 2;
    while (last - first > 3) {
        if (depth == 0) {
            kp_heap_select<K>(v, first, nth + 1, last);
            kp_swap<K>(v, first, nth);
            return;
        }
        --depth;
        // __unguarded_partition_pivot
        const int mid = first + (last - first) / 2;
        {
            const int a = first + 1, b = mid, c = last - 1;
            if (kp_greater<K>(v[a], v[b])) {
                if (kp_greater<K>(v[b], v[c])) kp_swap<K>(v, first, b);
                else if (kp_greater<K>(v[a], v[c])) kp_swap<K>(v, first, c);
                else kp_swap<K>(v, first, a);
            } else if (kp_greater<K>(v[a], v[c])) kp_swap<K>(v, first, a);
            else if (kp_greater<K>(v[b], v[c])) kp_swap<K>(v, first, c);
            else kp_swap<K>(v, first, b);
        }
        int lo = first + 1, hi = last;
        const uint32_t pivot_slot = first;
        while (true) {
            while (kp_greater<K>(v[lo], v[pivot_slot])) ++lo;
            --hi;
            while (kp_greater<K>(v[pivot_slot], v[hi])) --hi;
            if (!(lo < hi)) break;
            kp_swap<K>(v, lo, hi);
            ++lo;
        }
        const int cut = lo;
        if (cut <= nth) first = cut;
        else last = cut;
    }
    // __insertion_sort(first, last)
    if (first == last) return;
    for (int i = first + 1; i != last; ++i) {
        typename K::rec val = v[i];
        if (kp_greater<K>(val, v[first])) {
            for (int k = i; k > first; --k) v[k] = v[k - 1];
            v[first] = val;
        } else {
            int k = i;
            while (kp_greater<K>(val, v[k - 1])) { v[k] = v[k - 1]; --k; }
            v[k] = val;
        }
    }
}

#if defined(__CUDACC__)
// Warp-cooperative std::nth_element with the SAME resulting permutation as kp_nth_element above; all 32 lanes of a
// warp call it with identical arguments. The unguarded Hoare partition is the only O(n) part and its outcome is a
// pure function of the stop positions: with P the pivot score, l_1 < l_2 < ... the positions in (first, last) whose
// score is <= P ("left stops") and r_1 > r_2 > ... the positions in [first, last) whose score is >= P ("right
// stops"), the serial loop swaps (l_k, r_k) for k = 1..m, m = the last k with l_k < r_k, and returns
// cut = min(l_{m+1}, r_m). Here both scans advance 32 elements per ballot, stops are queued in two 64-entry rings
// (`q`, 128 ints of this warp's shared memory) and up to 32 pairs are swapped per round. Stops found in elements that
// an earlier round already swapped lie beyond r_m (resp. before l_m), so they can only produce failing pairs and
// leave m and cut unchanged. Median-of-three, range bookkeeping, the <= 3 element insertion sort and the heap-select
// fallback are serial on lane 0.
template <class K = KpScore32>
__device__ __forceinline__ int kp_partition_warp(typename K::rec* v, int first, int last, unsigned P, int* q) {
    const int lane = threadIdx.x & 31;
    const unsigned lt = (1u << lane) - 1u;
    int* Lq = q; int* Rq = q + 64;
    int lc = first + 1, rc = last, nl = 0, nr = 0, lh = 0, rh = 0;
    int last_r = 0x7fffffff;
    while (true) {
        while (nl < 32 && lc < last) {
            const int p = lc + lane;
            const bool fl = p < last && K::key(v[p]) <= P;
            const unsigned bal = __ballot_sync(0xffffffffu, fl);
            if (fl) Lq[(lh + nl + __popc(bal & lt)) & 63] = p;
            nl += __popc(bal); lc += 32;
        }
        while (nr < 32 && rc > first) {
            const int p = rc - 1 - lane;
            const bool fr = p >= first && K::key(v[p]) >= P;
            const unsigned bal = __ballot_sync(0xffffffffu, fr);
            if (fr) Rq[(rh + nr + __popc(bal & lt)) & 63] = p;
            nr += __popc(bal); rc -= 32;
        }
        __syncwarp();
        const int np = min(min(nl, nr), 32);
        if (np == 0) return nl > 0 ? min(Lq[lh & 63], last_r) : last_r;
        const int l = lane < np ? Lq[(lh + lane) & 63] : 0, r = lane < np ? Rq[(rh + lane) & 63] : 0;
        const unsigned okb = __ballot_sync(0xffffffffu, lane < np && l < r);
        const int cnt = min(__ffs(~okb) - 1 < 0 ? 32 : __ffs(~okb) - 1, np);   // leading pairs with l < r
        if (lane < cnt) { const typename K::rec t = v[l]; v[l] = v[r]; v[r] = t; }
        if (cnt > 0) last_r = __shfl_sync(0xffffffffu, r, cnt - 1);
        __syncwarp();
        if (cnt < np) return min(__shfl_sync(0xffffffffu, l, cnt), last_r);
        lh += np; nl -= np; rh += np; nr -= np;
    }
}

template <class K = KpScore32>
__device__ __forceinline__ void kp_nth_element_warp(typename K::rec* v, int n, int nth, int* q) {
    const int lane = threadIdx.x & 31;
    if (n <= 0 || nth >= n) return;
    int first = 0, last = n;
    int depth = 0;
    for (int t = n; t > 1; t >>= 1) ++depth;
    depth *= 2;
    while (last - first > 3) {
        if (depth == 0) {
            if (lane == 0) { kp_heap_select<K>(v, first, nth + 1, last); kp_swap<K>(v, first, nth); }
            __syncwarp();
            return;
        }
        --depth;
        if (lane == 0) {
            const int a = first + 1, b = first + (last - first) / 2, c = last - 1;
            const unsigned sa = K::key(v[a]), sb = K::key(v[b]), sc = K::key(v[c]);
            int m;
            if (sa > sb) m = (sb > sc) ? b : (sa > sc) ? c : a;
            else m = (sa > sc) ? a : (sb > sc) ? c : b;
            kp_swap<K>(v, first, m);
        }
        __syncwarp();
        const int cut = kp_partition_warp<K>(v, first, last, K::key(v[first]), q);
        if (cut <= nth) first = cut; else last = cut;
    }
    if (lane == 0 && first != last) {
        for (int i = first + 1; i != last; ++i) {
            const typename K::rec val = v[i];
            if (kp_greater<K>(val, v[first])) {
                for (int k = i; k > first; --k) v[k] = v[k - 1];
                v[first] = val;
            } else {
                int k = i;
                while (kp_greater<K>(val, v[k - 1])) { v[k] = v[k - 1]; --k; }
                v[k] = val;
            }
        }
    }
    __syncwarp();
}
#endif

}  // namespace se2gpu
