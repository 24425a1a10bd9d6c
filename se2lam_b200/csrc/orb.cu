// ORB front-end on sm_90a — kernels + C ABI (include/se2gpu.h, se2gpu_orb_*).
//
// Replaces se2lam::ORBextractor::operator() (reference src/ORBextractor.cpp:727-788) and the OpenCV
// primitives underneath it, for batches of frames, bit-exactly (keypoint order included):
//   orb_pyr0 / orb_resize_w ComputePyramid :790-831 (copyMakeBorder REFLECT_101, resize INTER_LINEAR: 11-bit
//                           fixed point, each level from the previous one)
//   orb_pyr0_undistort      optional: cv::undistort of Frame.cpp:22 folded into level 0 (se2gpu_orb_set_undistort)
//   orb_fast_cells<TMA>     per-cell cv::FAST(…,fastTh)/FAST(…,7) :608-623 — one CTA per grid cell: the cell and
//                           its 3 px apron are staged in shared memory once; a branch-free necessary condition on
//                           every pixel, survivors compacted, then the threshold-free arc score
//                           M = max over the 16 nine-pixel arcs of min(+-diff) (corner at t <=> M > t, score = M-1)
//                           at full lane occupancy, cell-local 3x3 strict NMS into a bitmap, raster-ordered emission
//   orb_fast_cells_big      the same result for cells too large for the shared-memory candidate list
//   orb_harris              HARRIS_SCORE handles only: HarrisResponses(cell, kps, 7, 0.04f) :85-126, :625-629 on the un-blurred
//                           level, one 64-bit record (order key of the response, FAST record) per candidate
//   orb_select_cells<HARRIS> quota redistribution :631-679 + KeyPointsFilter::retainBest per cell :687-694, one warp per cell;
//   orb_select_levels<HARRIS> retainBest per level :706-710, one warp per level — the libstdc++ introselect permutation is
//                           reproduced exactly, warp-cooperatively (introselect.h); keyed by the FAST score, or by the Harris
//                           response on 64-bit records
//   orb_blur                GaussianBlur 7x7 sigma 2 :769 (float32 separable, fused multiply-add, RNE to u8)
//   orb_orient_describe     IC_Angle :130-157 + computeOrbDescriptor :160-200, one warp per keypoint; keypoint
//                           records are written as 28-byte cv::KeyPoint and 32-byte descriptors
// Data layout in HBM (per frame): every pyramid level is a bordered u8 plane (w+32) x (h+32) with row pitch
// rounded up to 32 B; two copies (plain, blurred); candidates are packed 32-bit records x:12|y:12|score:8.
#include <cuda.h>   // CUtensorMap + the cuTensorMapEncodeTiled prototype only: the entry point is resolved at run time (no libcuda link)

#include <algorithm>
#include <cmath>
#include <cstring>
#include <type_traits>
#include <vector>

#include "blur_px.h"
#include "common.h"
#include "fast_screen.h"
#include "introselect.h"
#include "resp_key.h"

namespace {

using se2gpu::fail;

constexpr int EDGE = 16;           // EDGE_THRESHOLD, ORBextractor.cpp:83
constexpr int HALF_PATCH = 15;     // HALF_PATCH_SIZE :82
constexpr int PATCH = 31;          // PATCH_SIZE :81
constexpr int MAX_LEVELS = 16;
constexpr int FAST_THREADS = 256;
constexpr int ORB_LANES = 4;
constexpr int BLUR_WARPS = 4;      // warps (tiles) per orb_blur CTA
constexpr int BLUR_TH = 48;        // ROI rows per orb_blur strip, before rounding to the 7-row ring (build_geometry)

__device__ const signed char d_pattern[1024] = {
#include "orb_pattern_31.inc"
};
__constant__ int c_umax[16];
__constant__ int c_vmax[16];   // c_vmax[|u|] = largest |v| of the patch disc in column u (the disc is stored row-wise as umax[|v|])
__constant__ float c_gauss[7];

struct LevelGeo {
    int w, h, pitch;
    size_t plane_off;   // byte offset of the bordered plane inside a frame's plane block
    int nDesired, cols, rows, nCells, nfeaturesCell;
    int cell_base;      // first cell of this level in the cell table
    int kp_off, kp_cap; // slot range in the per-frame level keypoint buffer
    float scale, kp_size;
    int tab_off;        // offset of this level's resize tables (xofs | yofs) in the int table
    int tile_base;      // first orb_blur tile of this level
    int blur_th, blur_strips;   // orb_blur: ROI rows per strip, strips (the last one ends at the ROI's last row)
    int fbw, fbh;       // orb_fast_cells<true>: TMA box of this level's FAST cells (bytes per row: multiple of 16; rows)
    int sel_off, sel_cap;   // slot range of the level list (the cells' survivors) in the per-frame selection buffer
};

struct CellGeo {
    int level, x0, y0, x1, y1;  // interior [x0,x1) x [y0,y1) in level ROI coordinates
    int skipped;                // the reference's `continue` cells (:579-580, :603-604)
    int cand_off, cand_cap;     // slot range in the per-frame candidate buffer
};

struct TileGeo { int level, strip, cg; };  // orb_blur warp: its first (strip, column group of 8 bytes) item; lane j takes the j-th item after it

struct CellHdr { int n_base, n_a, n_b, pad; };

struct OrbDev {  // passed by value to kernels
    int nlevels, nfeatures, fast_th, t_lo;
    int n_cells, n_tiles;
    const LevelGeo* levels;
    const CellGeo* cells;
    const TileGeo* tiles;
    const int* itab;            // xofs/yofs tables
    const short* stab;          // ialpha/ibeta tables (2 per entry)
    uint8_t* plain;             // [B][frame_plane_bytes]
    uint8_t* blurred;
    size_t frame_plane_bytes;
    uint32_t* cand;             // [B][cand_total]
    size_t cand_total;
    CellHdr* hdr;               // [B][n_cells]
    uint32_t* lkp;              // [B][lkp_total]
    int lkp_total;
    int* lcount;                // [B][nlevels]
    uint64_t* sel;              // [B][sel_total] level lists between orb_select_cells and orb_select_levels (32- or 64-bit records)
    int sel_total;
    int* err;                   // device error flag
    int frame0;                 // first frame of this launch group (pipelined host path processes the batch in chunks)
};

__device__ __forceinline__ int reflect101(int p, int len) {
    if (len == 1) return 0;
    while (p < 0 || p >= len) p = p < 0 ? -p : 2 * (len - 1) - p;
    return p;
}

// level 0: copyMakeBorder(image, temp, 16,16,16,16, BORDER_REFLECT_101). The border is 16 px wide, so when the caller's
// rows are 16 B aligned the interior is a stream of aligned 16-byte copies: blockIdx.x < gridDim.x-1 does those, one
// thread = one vector x PYR0_ROWS rows. The last blockIdx.x column fills what is left of each row (the two 16 px
// borders, a ragged interior tail, the pitch padding — everything when the input is unaligned) one word per thread.
// The level geometry comes in as a kernel parameter (constant bank), not through a dependent global load.
constexpr int PYR0_ROWS = 4;
__global__ void __launch_bounds__(256) orb_pyr0(OrbDev d, LevelGeo L, const uint8_t* __restrict__ imgs, int stride, size_t frame_stride, int nvec) {
    const int tid = threadIdx.y * 64 + threadIdx.x;
    const int f = blockIdx.z + d.frame0;
    const uint8_t* img = imgs + f * frame_stride;
    uint8_t* plane = d.plain + f * d.frame_plane_bytes + L.plane_off;
    const int rows = L.h + 2 * EDGE;
    if (blockIdx.x + 1 < gridDim.x) {
        const int vx = blockIdx.x * 64 + threadIdx.x;
        const int y0 = (blockIdx.y * 4 + threadIdx.y) * PYR0_ROWS;
        if (vx >= nvec) return;
        uint4 v[PYR0_ROWS];
#pragma unroll
        for (int k = 0; k < PYR0_ROWS; ++k)
            if (y0 + k < rows) v[k] = __ldg(reinterpret_cast<const uint4*>(img + (size_t)reflect101(y0 + k - EDGE, L.h) * stride) + vx);
#pragma unroll
        for (int k = 0; k < PYR0_ROWS; ++k)
            if (y0 + k < rows) *reinterpret_cast<uint4*>(plane + (size_t)(y0 + k) * L.pitch + EDGE + 16 * vx) = v[k];
        return;
    }
    // remainder words of the rows [16*blockIdx.y, +16): columns [0,16) and [16 + 16*nvec, pitch)
    const int tail0 = EDGE + 16 * nvec, nw = 4 + (L.pitch - tail0) / 4;
    for (int item = tid; item < 4 * PYR0_ROWS * nw; item += 256) {
        const int r = item / nw, wi = item - r * nw;
        const int y = blockIdx.y * 4 * PYR0_ROWS + r;
        if (y >= rows) break;
        const int x0 = wi < 4 ? 4 * wi : tail0 + 4 * (wi - 4);
        const uint8_t* row = img + (size_t)reflect101(y - EDGE, L.h) * stride;
        uint32_t word = 0;
#pragma unroll
        for (int q = 0; q < 4; ++q) {
            const int x = x0 + q;
            const uint32_t px = (x < L.w + 2 * EDGE) ? row[reflect101(x - EDGE, L.w)] : 0u;
            word |= px << (8 * q);
        }
        *reinterpret_cast<uint32_t*>(plane + (size_t)y * L.pitch + x0) = word;
    }
}

// level 0 with the lens undistortion of Frame::Frame folded in (reference src/Frame.cpp:22: cv::undistort(im, img, Kcam, Dcam)
// right before the extractor; SURVEY section 8(f) N3): every pixel of the bordered level-0 plane is
// remap(INTER_LINEAR, BORDER_CONSTANT 0) of the raw frame through the fixed-point map of the (reflected) pixel - integer
// source coordinates in m1, 5+5 fraction bits in m2, weights (32-a)(32-b)*32 ... (sum 2^15), (sum + 2^14) >> 15. The map
// depends on the camera only and is built once per frame size on the host with OpenCV's double arithmetic
// (build_undistort_map). One thread = 4 output pixels, one word store; the undistorted image is never materialised.
__global__ void __launch_bounds__(128) orb_pyr0_undistort(OrbDev d, LevelGeo L, const uint8_t* __restrict__ imgs, int stride, size_t frame_stride,
                                                          const short2* __restrict__ m1, const uint16_t* __restrict__ m2) {
    const int x4 = (blockIdx.x * 128 + threadIdx.x) * 4, y = blockIdx.y;
    const int f = blockIdx.z + d.frame0;
    if (x4 >= L.pitch) return;
    const uint8_t* img = imgs + f * frame_stride;
    const int dy = reflect101(y - EDGE, L.h);
    uint32_t word = 0;
#pragma unroll
    for (int q = 0; q < 4; ++q) {
        const int x = x4 + q;
        uint32_t o = 0;
        if (x < L.w + 2 * EDGE) {
            const int idx = dy * L.w + reflect101(x - EDGE, L.w);
            const short2 s = __ldg(m1 + idx);
            const int fr = __ldg(m2 + idx), a = fr & 31, b = fr >> 5;
            const int sx = s.x, sy = s.y;
            const bool x0 = (unsigned)sx < (unsigned)L.w, x1 = (unsigned)(sx + 1) < (unsigned)L.w;
            const bool y0 = (unsigned)sy < (unsigned)L.h, y1 = (unsigned)(sy + 1) < (unsigned)L.h;
            const uint8_t* p = img + (ptrdiff_t)sy * stride + sx;
            const int t00 = (x0 && y0) ? p[0] : 0, t01 = (x1 && y0) ? p[1] : 0, t10 = (x0 && y1) ? p[stride] : 0, t11 = (x1 && y1) ? p[stride + 1] : 0;
            const int val = t00 * ((32 - a) * (32 - b) * 32) + t01 * (a * (32 - b) * 32) + t10 * ((32 - a) * b * 32) + t11 * (a * b * 32);
            o = (uint32_t)min(max((val + (1 << 14)) >> 15, 0), 255);
        }
        word |= o << (8 * q);
    }
    uint8_t* plane = d.plain + f * d.frame_plane_bytes + L.plane_off;
    *reinterpret_cast<uint32_t*>(plane + (size_t)y * L.pitch + x4) = word;
}

// level l>0: resize(level l-1 -> level l, INTER_LINEAR) + copyMakeBorder(REFLECT_101) in one pass, cv::resize's
// fixed-point arithmetic (11-bit coefficients, horizontal pass kept at full precision, vertical pass >>4, >>16, +2 >>2).
// One CTA = a 128 x RESIZE_TR tile (32 or 64 rows, see below) of the bordered output plane, three stages in shared memory:
//   0  the source rows/columns the tile touches (a contiguous box, also across the reflected border) as 16 B vectors
//   1  horizontal pass h[s][x] = src[s][sx]*a0 + src[s][sx+1]*a1 for every staged source row s, ONCE per (row, column)
//      (consecutive output rows share source rows; cv::resize does the same with its row buffers)
//   2  vertical pass from two h rows per output row, 4 pixels per thread, one 32-bit store
// Column terms (xofs, ialpha) and row terms are computed once per tile (one thread per column / row) and shared through small tables.
// The kernel is bound by shared-memory wavefronts, many of them bank-conflict replays of byte gathers, so the horizontal pass reads
// a 12-byte window per row and thread (3 word loads instead of 8 byte loads; PRMT picks the byte pair, IDP.2A does
// src[sx]*a0 + src[sx+1]*a1) and keeps its results as 16-bit values (<= 32 640), which halves the wavefronts of the store and of
// the two loads per output row of the vertical pass. Values that do not fit the window form (scale factors above ~2.6, negative
// coefficients) take a byte path inside the same kernel, with the same arithmetic term by term.
// PDL: launched with programmatic stream serialisation (cudaLaunchAttributeProgrammaticStreamSerialization). Every CTA releases its
// dependents at once (griddepcontrol.launch_dependents), so the CTAs of the NEXT level's launch are scheduled into the SM slots
// the last wave of this launch frees and run their table set-up there; they read this level's plane only behind
// griddepcontrol.wait, which returns when this whole grid has completed and its writes are visible. The pyramid is a chain of seven
// dependent, short launches: this overlaps each launch's ramp-up with its predecessor's tail.
// Tile height: RESIZE_TR rows, or RESIZE_TR_TALL rows on levels whose grid of tall tiles still fills every resident CTA slot of the
// GPU at least once (run_device). A CTA's fixed costs - table loads, two dependent L2 round trips, three barriers - are then spread
// over twice the output rows, and more output rows share each staged source row; on the small levels tall tiles would leave SMs
// idle in a single partial wave. Measured on an H100 SXM (400 W), 64 frames of 640x480, 8 levels: per-level kernel times in us
// (levels 1..7, torch.profiler, tools/orb_pyramid_trace.py) and the pyramid profile group in ms:
//   32 rows everywhere       39.6 32.6 27.2 20.9 18.9 15.8 11.7   0.153
//   64 rows everywhere       32.0 29.6 25.5 20.6 19.4 15.7 21.4   0.135
//   96 rows everywhere       31.3 28.5 27.2 21.9 19.0 17.6 22.9   0.135
//  128 rows everywhere       32.5 29.3 27.6 24.3 19.0 22.4 21.6   0.136
//   64 rows on levels 1-5    32.1 29.6 25.2 21.3 19.8 16.1 11.7   0.134-0.135 (this rule; step 0.623-0.627 ms against 0.644-0.649)
constexpr int RESIZE_TR = 32, RESIZE_TR_TALL = 64;
struct ResizeRow { int s0, s1, b0, b1; };
struct ResizeCol { int sx0, sx1; short a0, a1; int valid; };   // 16 B
template <int RESIZE_TR>
__global__ void __launch_bounds__(256) orb_resize_w(OrbDev d, LevelGeo L, LevelGeo S, int max_rows, int raw_pitch) {
    static_assert(RESIZE_TR % 32 == 0 && RESIZE_TR <= 128, "row terms take one thread per row in warps 4..7");
    asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
    extern __shared__ __align__(16) uint8_t rs_smem[];
    __shared__ ResizeRow rowinfo[RESIZE_TR];
    __shared__ __align__(16) ResizeCol colinfo[128];
    __shared__ int s_lo[RESIZE_TR / 32], s_hi[RESIZE_TR / 32];   // source row range per row warp
    __shared__ int s_cmin[4], s_cmax[4]; // source column range per column warp
    uint16_t* hbuf = reinterpret_cast<uint16_t*>(rs_smem);                  // [max_rows][128], 16 bit: (255 * 2048) >> 4 = 32 640
    uint8_t* raw = rs_smem + (size_t)max_rows * 128 * sizeof(uint16_t);     // [max_rows][raw_pitch] (+16 B of slack behind the last row)
    const int tx = threadIdx.x, ty = threadIdx.y, tid = ty * 32 + tx;
    const int x4 = blockIdx.x * 128 + tx * 4, y0 = blockIdx.y * RESIZE_TR;
    const int f = blockIdx.z + d.frame0;
    const int W = L.w + 2 * EDGE, H = L.h + 2 * EDGE;
    const int* xofs = d.itab + L.tab_off;
    const int* yofs = xofs + L.w;
    const short2* ialpha = reinterpret_cast<const short2*>(d.stab + 2 * (size_t)L.tab_off);
    const short2* ibeta = ialpha + L.w;
    // column terms of the tile's 128 output columns: warps 0..3, one column per thread (the 8 thread rows share them through
    // shared memory instead of each recomputing its 4 columns); row terms: warps 4.., one row per thread
    if (tid < 128) {
        const int x = blockIdx.x * 128 + tid;
        ResizeCol c{0, 0, 0, 0, 0};
        int cmin = 0x7fffffff, cmax = -1;
        if (x < W) {
            const int dx = reflect101(x - EDGE, L.w);
            c.sx0 = __ldg(xofs + dx);
            c.sx1 = min(c.sx0 + 1, S.w - 1);
            const short2 aa = __ldg(ialpha + dx);
            c.a0 = aa.x; c.a1 = aa.y; c.valid = 1;
            cmin = c.sx0; cmax = c.sx1;
        }
        colinfo[tid] = c;
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) { cmin = min(cmin, __shfl_xor_sync(0xffffffffu, cmin, o)); cmax = max(cmax, __shfl_xor_sync(0xffffffffu, cmax, o)); }
        if (tx == 0) { s_cmin[ty] = cmin; s_cmax[ty] = cmax; }
    } else if (ty < 4 + RESIZE_TR / 32) {   // row terms of the tile's RESIZE_TR output rows and their source row range
        const int ry = tid - 128, y = y0 + ry;
        int rmin = 0x7fffffff, rmax = -1;
        if (y < H) {
            const int dy = reflect101(y - EDGE, L.h);
            const int sy = __ldg(yofs + dy);
            const short2 bb = __ldg(ibeta + dy);
            ResizeRow r{min(max(sy, 0), S.h - 1), min(max(sy + 1, 0), S.h - 1), bb.x, bb.y};
            rowinfo[ry] = r;
            rmin = r.s0; rmax = r.s1;
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) { rmin = min(rmin, __shfl_xor_sync(0xffffffffu, rmin, o)); rmax = max(rmax, __shfl_xor_sync(0xffffffffu, rmax, o)); }
        if (tx == 0) { s_lo[ty - 4] = rmin; s_hi[ty - 4] = rmax; }
    }
    __syncthreads();
    const int c_min = min(min(s_cmin[0], s_cmin[1]), min(s_cmin[2], s_cmin[3])), c_max = max(max(s_cmax[0], s_cmax[1]), max(s_cmax[2], s_cmax[3]));
    const int c_lo = c_min & ~15, nvec = c_max < 0 ? 0 : (c_max - c_lo) / 16 + 1;
    int r_lo = s_lo[0], r_hi = s_hi[0];
#pragma unroll
    for (int k = 1; k < RESIZE_TR / 32; ++k) { r_lo = min(r_lo, s_lo[k]); r_hi = max(r_hi, s_hi[k]); }
    const int nsr = r_hi - r_lo + 1;
    if (nsr > max_rows || nvec * 16 > raw_pitch) { if (tid == 0) *d.err = 3; return; }   // sized on the host from the scale factor
    const uint8_t* src = d.plain + f * d.frame_plane_bytes + S.plane_off + (size_t)EDGE * S.pitch + EDGE;
    asm volatile("griddepcontrol.wait;" ::: "memory");     // the source level is complete and visible from here on
    // stage 0: 16 vectors per source row and pass (a 128-column tile at scale <= 1.9 spans <= 16 vectors), no division
    if (nvec <= 16) {
        const int v = tid & 15;
        if (v < nvec)
            for (int r = tid >> 4; r < nsr; r += 16)
                *reinterpret_cast<uint4*>(raw + r * raw_pitch + 16 * v) = __ldg(reinterpret_cast<const uint4*>(src + (size_t)(r_lo + r) * S.pitch + c_lo) + v);
    } else {
        for (int i = tid; i < nsr * nvec; i += 256) {
            const int r = i / nvec, v = i - r * nvec;
            *reinterpret_cast<uint4*>(raw + r * raw_pitch + 16 * v) = __ldg(reinterpret_cast<const uint4*>(src + (size_t)(r_lo + r) * S.pitch + c_lo) + v);
        }
    }
    // this thread's 4 columns
    int sx0[4], sx1[4], a0[4], a1[4];
    unsigned vmask = 0;                       // byte mask of the valid columns
#pragma unroll
    for (int q = 0; q < 4; ++q) {
        const ResizeCol c = colinfo[4 * tx + q];
        sx0[q] = c.valid ? c.sx0 - c_lo : 0; sx1[q] = c.valid ? c.sx1 - c_lo : 0;
        a0[q] = c.a0; a1[q] = c.a1;
        vmask |= c.valid ? (0xFFu << (8 * q)) : 0u;
    }
    __syncthreads();
    // the 4 columns' source bytes sx0, sx0+1 lie in one 12-byte window of the staged row (3 aligned words from word w0 on) as long
    // as the scale factor is below ~2.6; byte pairs come out of the window with one PRMT (selector fixed per column), and
    // src[sx0]*a0 + src[sx0+1]*a1 is one IDP.2A. Where cv::resize clamps sx1 to sx0 (right edge) a1 is 0, so the byte behind sx0
    // may be anything. Three 32-bit loads per row instead of eight byte loads: the kernel is bound by shared-memory wavefronts.
    unsigned wq[4], selq[4];
    bool pairq[4];
    int w0 = 0;
    bool window_ok = true;
    {
        int mn = 0x7fffffff;
#pragma unroll
        for (int q = 0; q < 4; ++q) if ((vmask >> (8 * q)) & 1u) mn = min(mn, sx0[q]);
        if (mn == 0x7fffffff) mn = 0;
        w0 = mn >> 2;
#pragma unroll
        for (int q = 0; q < 4; ++q) {
            const bool valid = (vmask >> (8 * q)) & 1u;
            const int o = valid ? sx0[q] - 4 * w0 : 0;
            if (valid && (o + 1 > 11 || (sx1[q] != sx0[q] + 1 && a1[q] != 0))) window_ok = false;
            pairq[q] = o >= 7;
            const int o2 = o - (pairq[q] ? 4 : 0);
            selq[q] = (unsigned)o2 | ((unsigned)(o2 + 1) << 4);
            wq[q] = ((unsigned)a0[q] & 0xFFFFu) | ((unsigned)a1[q] << 16);
            if (a0[q] < 0 || a1[q] < 0) window_ok = false;     // cv's coefficients are in [0, 2048]; anything else takes the byte path
        }
    }
    // stage 1: horizontal pass, stored pre-shifted (the vertical pass uses S >> 4 only)
    if (x4 < W) {
        if (window_ok) {
            for (int r = ty; r < nsr; r += 8) {
                const uint32_t* rw = reinterpret_cast<const uint32_t*>(raw + r * raw_pitch) + w0;
                const uint32_t W0 = rw[0], W1 = rw[1], W2 = rw[2];
                unsigned hq[4];
#pragma unroll
                for (int q = 0; q < 4; ++q) {
                    const unsigned bytes = __byte_perm(pairq[q] ? W1 : W0, pairq[q] ? W2 : W1, selq[q]);
                    hq[q] = __dp2a_lo(wq[q], bytes, 0u) >> 4;
                }
                *reinterpret_cast<uint2*>(hbuf + r * 128 + 4 * tx) = make_uint2(hq[0] | (hq[1] << 16), hq[2] | (hq[3] << 16));
            }
        } else {
            for (int r = ty; r < nsr; r += 8) {
                const uint8_t* rp = raw + r * raw_pitch;
                const unsigned h0 = (unsigned)((rp[sx0[0]] * a0[0] + rp[sx1[0]] * a1[0]) >> 4), h1 = (unsigned)((rp[sx0[1]] * a0[1] + rp[sx1[1]] * a1[1]) >> 4);
                const unsigned h2 = (unsigned)((rp[sx0[2]] * a0[2] + rp[sx1[2]] * a1[2]) >> 4), h3 = (unsigned)((rp[sx0[3]] * a0[3] + rp[sx1[3]] * a1[3]) >> 4);
                *reinterpret_cast<uint2*>(hbuf + r * 128 + 4 * tx) = make_uint2((h0 & 0xFFFFu) | (h1 << 16), (h2 & 0xFFFFu) | (h3 << 16));
            }
        }
    }
    __syncthreads();
    // stage 2: vertical pass. With coefficients in [0, 2048] (pairs summing to 2048 +- 1) and 8-bit pixels the result is in
    // [0, 255] by construction ((2049 * (255 * 2049 >> 4) >> 16) + 2 >> 2 = 255): cv's saturate_cast never fires, no clamp here.
    if (x4 >= L.pitch) return;
    uint8_t* plane = d.plain + f * d.frame_plane_bytes + L.plane_off;
#pragma unroll
    for (int k = 0; k < RESIZE_TR / 8; ++k) {
        const int r = ty + 8 * k, y = y0 + r;
        if (y >= H) break;
        uint32_t word = 0;
        if (x4 < W) {
            const ResizeRow ri = rowinfo[r];
            const uint2 A = *reinterpret_cast<const uint2*>(hbuf + (ri.s0 - r_lo) * 128 + 4 * tx);
            const uint2 B = *reinterpret_cast<const uint2*>(hbuf + (ri.s1 - r_lo) * 128 + 4 * tx);
            const unsigned v0 = (unsigned)((((ri.b0 * (int)(A.x & 0xFFFFu)) >> 16) + ((ri.b1 * (int)(B.x & 0xFFFFu)) >> 16) + 2) >> 2);
            const unsigned v1 = (unsigned)((((ri.b0 * (int)(A.x >> 16)) >> 16) + ((ri.b1 * (int)(B.x >> 16)) >> 16) + 2) >> 2);
            const unsigned v2 = (unsigned)((((ri.b0 * (int)(A.y & 0xFFFFu)) >> 16) + ((ri.b1 * (int)(B.y & 0xFFFFu)) >> 16) + 2) >> 2);
            const unsigned v3 = (unsigned)((((ri.b0 * (int)(A.y >> 16)) >> 16) + ((ri.b1 * (int)(B.y >> 16)) >> 16) + 2) >> 2);
            word = (v0 | (v1 << 8) | (v2 << 16) | (v3 << 24)) & vmask;
        }
        *reinterpret_cast<uint32_t*>(plane + (size_t)y * L.pitch + x4) = word;
    }
}

// FAST-9-16 on packed ring differences. For centre v and ring pixel p the s16x2 word
//   q = (256 + v - p) | (256 + p - v) << 16  =  p * 0xFFFF + ((256 + v) | (256 - v) << 16)      (one IMAD; both halves in [1,511])
// carries the "darker" and the "brighter" test side by side, so the packed 3-input min/max of Hopper's DPX instructions (VIMNMX3.S16x2)
// evaluates both polarities at once. Arc score M = max over the 16 nine-pixel arcs of min(+-(v - ring)); corner at
// t <=> M > t, and cv::FAST's stored score == M-1 whatever t was.
__device__ __forceinline__ unsigned fast_cv(int v) { return (unsigned)(256 + v) | ((unsigned)(256 - v) << 16); }
__device__ __forceinline__ unsigned fast_q(unsigned p, unsigned cv) { return p * 0xFFFFu + cv; }

__device__ __forceinline__ int fast_arc_score(const uint8_t* __restrict__ p, int pw) {
    const unsigned cv = fast_cv(p[0]);
    unsigned q[16];
    q[0] = fast_q(p[3 * pw], cv);       q[1] = fast_q(p[3 * pw + 1], cv);   q[2] = fast_q(p[2 * pw + 2], cv);    q[3] = fast_q(p[pw + 3], cv);
    q[4] = fast_q(p[3], cv);            q[5] = fast_q(p[-pw + 3], cv);      q[6] = fast_q(p[-2 * pw + 2], cv);   q[7] = fast_q(p[-3 * pw + 1], cv);
    q[8] = fast_q(p[-3 * pw], cv);      q[9] = fast_q(p[-3 * pw - 1], cv);  q[10] = fast_q(p[-2 * pw - 2], cv);  q[11] = fast_q(p[-pw - 3], cv);
    q[12] = fast_q(p[-3], cv);          q[13] = fast_q(p[pw - 3], cv);      q[14] = fast_q(p[2 * pw - 2], cv);   q[15] = fast_q(p[3 * pw - 1], cv);
    unsigned m3[16];
#pragma unroll
    for (int k = 0; k < 16; ++k) m3[k] = __vimin3_s16x2(q[k], q[(k + 1) & 15], q[(k + 2) & 15]);
    unsigned best = 0;
#pragma unroll
    for (int k = 0; k < 16; k += 2) {
        const unsigned a9 = __vimin3_s16x2(m3[k], m3[(k + 3) & 15], m3[(k + 6) & 15]);
        const unsigned b9 = __vimin3_s16x2(m3[k + 1], m3[(k + 4) & 15], m3[(k + 7) & 15]);
        best = __vimax3_s16x2(best, a9, b9);
    }
    return (int)max(best & 0xFFFFu, best >> 16) - 256;
}

// ---- TMA (cp.async.bulk.tensor, SASS UTMALDG) + mbarrier helpers
struct FastMaps { CUtensorMap m[MAX_LEVELS]; };   // one 3-D map (x bytes, rows, frames) per pyramid level, box = that level's cell patch
__device__ __forceinline__ unsigned orb_smem_u32(const void* p) { return (unsigned)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void orb_mbar_init(unsigned long long* bar, unsigned count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(orb_smem_u32(bar)), "r"(count) : "memory");
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
// waits for the phase with the given parity; gives up after ~0.2 s of SM clocks (a copy that never lands - a broken tensor map -
// must end in an error code, not in a hung GPU) and returns false
__device__ __forceinline__ bool orb_mbar_wait(unsigned long long* bar, unsigned parity) {
    const long long t0 = clock64();
    for (;;) {
        unsigned done;
        asm volatile(
            "{\n"
            ".reg .pred p;\n"
            "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n"
            "selp.u32 %0, 1, 0, p;\n"
            "}\n" : "=r"(done) : "r"(orb_smem_u32(bar)), "r"(parity) : "memory");
        if (done) return true;
        if (clock64() - t0 > 400000000LL) return false;
    }
}
// one box of the 3-D tensor (x, y, z) -> shared memory; completion is signalled on `bar` with the box's byte count
__device__ __forceinline__ void orb_tma_box3(void* dst_smem, const CUtensorMap* map, int x, int y, int z, unsigned bytes, unsigned long long* bar) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(orb_smem_u32(bar)), "r"(bytes) : "memory");
    asm volatile("cp.async.bulk.tensor.3d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3, %4}], [%5];"
                 ::"r"(orb_smem_u32(dst_smem)), "l"(map), "r"(x), "r"(y), "r"(z), "r"(orb_smem_u32(bar)) : "memory");
}

// one CTA per (cell, frame): cv::FAST(cell, fastTh, NMS) and, if that yields <= 3 keypoints, cv::FAST(cell, 7, NMS)
// (ORBextractor.cpp:616-623). The cell and its 3 px apron are staged once in shared memory, by one of two means:
//   TMA    ONE cp.async.bulk.tensor.3d per CTA pulls the patch (box fbw x fbh of the level's tensor map, origin at the 16 B aligned
//          column left of the cell's first apron pixel, pitch = the level's constant fbw) while the CTA clears its score plane;
//          the threads issue no staging loads. Needs every level's patch to fit a 256 x 256 box and the driver's
//          tensor-map encoder.
//   plain  aligned 32-bit loads from the 4 B aligned column left of the first apron pixel, pitch = the cell's patch width
//          rounded up to 4 B. Takes any cell whose patch and candidate list fit shared memory with 16-bit list offsets.
// Then, at either pitch:
//   A  every pixel: necessary condition (fastpx::screen4: a 9-arc contains one pixel of each opposite pair (k, k+8), so for one
//      polarity all 4 tested pairs need a member beyond t), branch-free on two pixels per s16x2 word; one thread = the 8 pixels
//      of two neighbouring patch words, whose screens share the 16 words they read; (row, item) items walked without a division;
//      survivors are compacted into a shared list by one atomicAdd per lane, which the compiler turns into a warp scan and one
//      shared atomic per warp (280 SASS per 8-pixel item in <true> at 48 registers, 35 per pixel, FAST group 0.237-0.239 ms
//      per 64-frame batch on an H100 SXM at 700 W; the 4-pixel items with 4 ballots and a shared atomic per warp took 207 per
//      4 pixels, 52 per pixel, at 64 registers and 4 CTAs per SM, and 0.275 ms)
//   B  list entries, full warps: arc score -> score plane (same pitch as the patch, zero apron and padding, fastpx::NMS_X0)
//   C  every thread a run of consecutive bitmap words (whole words per cell row): fastpx::nms32, the strict 3x3 maximum of 32
//      pixels from the dense score plane, branch-free on two pixels per u16x2 word
//   D  CTA-wide exclusive scan of the threads' keypoint counts = raster-order output slots
//   E  every thread its own bitmap words: emit (score | y | x), (y, x) from the word's row and column
// Registers: both instantiations are bounded for at least 5 CTAs of 256 threads per SM, so they get 48 (<true>) and 47
// (<false>), without spilling. Unbounded, the 8-pixel pass A takes <true> to 74 registers (80 allocated, 3 CTAs per SM): on an
// H100 SXM (700 W, 1980 MHz) its FAST group measured 0.2507-0.2523 ms per 64-frame batch against 0.2366-0.2385 ms with the
// bound, although the bound costs pass A 280 SASS per item instead of 234 (address arithmetic recomputed per item).
template <bool TMA>
__global__ void __launch_bounds__(FAST_THREADS, 5) orb_fast_cells(OrbDev d, const __grid_constant__ FastMaps maps) {
    extern __shared__ __align__(128) uint8_t smem_raw[];
    __shared__ int s_ncand, s_wsum[FAST_THREADS / 32];
    __shared__ __align__(8) unsigned long long s_bar;
    const CellGeo c = d.cells[blockIdx.x];
    const int f = blockIdx.y + d.frame0;
    CellHdr* hdr = d.hdr + (size_t)f * d.n_cells + blockIdx.x;
    const int cw = c.x1 - c.x0, ch = c.y1 - c.y0;
    if (c.skipped || cw <= 0 || ch <= 0) {
        if (threadIdx.x == 0) { hdr->n_base = 0; hdr->n_a = 0; hdr->n_b = 0; }
        return;
    }
    const LevelGeo& L = d.levels[c.level];
    // the patch starts at the aligned bordered-plane column ax0 <= x0-3 and the kernel carries the byte shift: TMA needs the innermost
    // tile coordinate of 1-byte elements to be a multiple of 16 B, the plain loads are 32-bit (plane base and pitch are 32 B aligned)
    const int bx0 = c.x0 - 3 + EDGE, ax0 = bx0 & (TMA ? ~15 : ~3), shift = bx0 - ax0;
    const int pw = TMA ? L.fbw : (shift + cw + 6 + 3) & ~3, pww = pw >> 2;   // patch pitch
    const int ph = TMA ? L.fbh : ch + 6;                                      // patch rows
    uint8_t* smem = TMA ? smem_raw + ((128u - (orb_smem_u32(smem_raw) & 127u)) & 127u) : smem_raw;   // TMA destination: 128 B aligned
    const int g0 = fastpx::first_group(shift), G = fastpx::items_per_row(cw, shift), nitems = ch * G;   // pass A work items
    const int wpr = fastpx::nms_words_per_row(cw);                                        // bitmap words per cell row
    uint8_t* patch = smem;                                                                // [ph x pw], pixel (x,y) of the cell at (y+3)*pw + x+3+shift
    uint8_t* score = smem + ((pw * ph + 15) & ~15);                                       // [(ch+2) x pw], pixel (x,y) at (y+1)*pw + x+NMS_X0
    uint32_t* bitmap = reinterpret_cast<uint32_t*>(score + ((fastpx::nms_plane_bytes(pw, ch) + 15) & ~15));   // [ch x wpr]
    uint16_t* list = reinterpret_cast<uint16_t*>(bitmap + ch * wpr);                      // [<= cw*ch] entries y*pw + x
    if (TMA && threadIdx.x == 0) orb_mbar_init(&s_bar, 1);
    asm volatile("griddepcontrol.wait;" ::: "memory");     // programmatic dependent of the last resize: the pyramid is complete from here on
    if (TMA) {
        __syncthreads();
        if (threadIdx.x == 0) orb_tma_box3(patch, &maps.m[c.level], ax0, c.y0 - 3 + EDGE, f, (unsigned)(pw * ph), &s_bar);
    } else {
        const uint8_t* plane = d.plain + f * d.frame_plane_bytes + L.plane_off;
        const int by0 = c.y0 - 3 + EDGE;
        for (int i = threadIdx.x; i < pww * ph; i += FAST_THREADS) {
            const int py = i / pww, pxw = i - py * pww;
            reinterpret_cast<uint32_t*>(patch)[i] = *reinterpret_cast<const uint32_t*>(plane + (size_t)(by0 + py) * L.pitch + ax0 + 4 * pxw);
        }
    }
    constexpr int NW = FAST_THREADS / 32;
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    const uint8_t* p0 = patch + 3 * pw + 3 + shift;
    fastpx::ItemWalk first;      // pass A: item = y*G + g; this thread's items are threadIdx.x, +256, +512, ...
    first.init((int)threadIdx.x, FAST_THREADS, G);
    fastpx::WordRun words;       // passes C and E: this thread's run of bitmap words
    words.init((int)threadIdx.x, FAST_THREADS, ch, wpr);
    int thr = d.fast_th;
    int total = 0, pos0 = 0;     // keypoints of the cell, and the raster-order slot of this thread's first one
    for (int pass = 0; pass < 2; ++pass) {
        for (int i = threadIdx.x; i < pw * (ch + 2) / 4; i += FAST_THREADS) reinterpret_cast<uint32_t*>(score)[i] = 0u;
        if (threadIdx.x == 0) s_ncand = 0;
        if (TMA && pass == 0 && !orb_mbar_wait(&s_bar, 0)) { *d.err = 4; return; }   // the patch has landed (async-proxy writes are visible after the wait)
        __syncthreads();
        // pass A
        {
            const uint32_t* pwords = reinterpret_cast<const uint32_t*>(patch);
            const unsigned bias = fastpx::screen_bias(thr);
            fastpx::ItemWalk it = first;
            for (int it0 = wid * 32; it0 < nitems; it0 += NW * 32) {
                unsigned m = 0;
                const int col0 = fastpx::group_x0(2 * it.g, shift);   // interior x of the item's first pixel
                if (it.y < ch) {                                      // <=> it0 + lane < nitems
                    const uint32_t* c = pwords + (it.y + 3) * pww + 2 * it.g + g0;
                    const uint32_t n3a = c[-3 * pww], n3b = c[-3 * pww + 1], s3a = c[3 * pww], s3b = c[3 * pww + 1];
                    const uint32_t n2a = c[-2 * pww - 1], n2b = c[-2 * pww], n2c = c[-2 * pww + 1], n2d = c[-2 * pww + 2];
                    const uint32_t s2a = c[2 * pww - 1], s2b = c[2 * pww], s2c = c[2 * pww + 1], s2d = c[2 * pww + 2];
                    const uint32_t za = c[-1], zb = c[0], zc = c[1], zd = c[2];
                    // necessary condition on both words, then drop the item's pixels outside the cell interior
                    m = (fastpx::screen4(n3a, s3a, n2a, n2b, n2c, s2a, s2b, s2c, za, zb, zc, bias) |
                         fastpx::screen4(n3b, s3b, n2b, n2c, n2d, s2b, s2c, s2d, zb, zc, zd, bias) << 4) & fastpx::inside_mask8(col0, cw);
                }
                // list slots: the list's order does not matter (B writes each entry's own plane byte, C and E are dense), so a
                // lane's survivors take consecutive slots from its own atomicAdd
                uint16_t* dst = list + atomicAdd(&s_ncand, __popc(m));
                const int e0 = it.y * pw + col0;
#pragma unroll
                for (int j = 0; j < 8; ++j)
                    if (m & (1u << j)) *dst++ = (uint16_t)(e0 + j);
                it.next();
            }
        }
        __syncthreads();
        const int ncand = s_ncand;
        // pass B
        for (int i = threadIdx.x; i < ncand; i += FAST_THREADS) {
            const int off = list[i];
            const int m = fast_arc_score(p0 + off, pw);
            if (m > thr) score[off + pw + fastpx::NMS_X0] = (uint8_t)(m - 1);
        }
        __syncthreads();
        // pass C: whole bitmap words, dense over the score plane; D: CTA-wide exclusive scan of the threads' keypoint counts
        int nkp = 0;
        for (fastpx::WordRun r = words; r.more(); r.next()) {
            const uint32_t* u = reinterpret_cast<const uint32_t*>(score) + r.y * pww + 8 * r.k;
            const unsigned bits = fastpx::nms32(u, u + pww, u + 2 * pww) & fastpx::nms_row_mask(r.k, cw);
            bitmap[r.w] = bits;
            nkp += __popc(bits);
        }
        int inc = nkp;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) { const int u = __shfl_up_sync(0xffffffffu, inc, o); if (lane >= o) inc += u; }
        if (lane == 31) s_wsum[wid] = inc;
        __syncthreads();
        total = 0; pos0 = inc - nkp;
#pragma unroll
        for (int w = 0; w < NW; ++w) { const int v = s_wsum[w]; total += v; if (w < wid) pos0 += v; }
        if (total > 3 || thr == 7) break;
        thr = 7;                 // cellKeyPoints.size() <= 3: clear and retry with the fixed fallback threshold
    }
    // pass E: this thread's bitmap words (it wrote them in C), in raster order from its slot pos0
    uint32_t* out = d.cand + (size_t)f * d.cand_total + c.cand_off;
    int pos = pos0;
    for (fastpx::WordRun r = words; r.more(); r.next()) {
        uint32_t bits = bitmap[r.w];
        const uint8_t* srow = score + (r.y + 1) * pw + fastpx::NMS_X0 + 32 * r.k;
        const uint32_t yx = ((uint32_t)(c.y0 + r.y) << 12) | (uint32_t)(c.x0 + 32 * r.k);
        while (bits) {
            const int i = __ffs(bits) - 1;
            bits &= bits - 1;
            if (pos < c.cand_cap) out[pos] = ((uint32_t)srow[i] << 24) | (yx + i);
            else *d.err = 1;
            ++pos;
        }
    }
    if (threadIdx.x == 0) { hdr->n_base = total; hdr->n_a = total; hdr->n_b = total; }
}

// FAST-9-16 arc score M = max over the 16 nine-pixel arcs of min(+-(v - ring)); corner at t <=> M > t,
// cv::FAST's stored score == M-1 whatever t was. Returns 0 early when the pixel cannot be a corner at t:
// a 9-arc always contains one pixel of each opposite pair (k, k+8), so all 4 tested pairs must have a
// member beyond +-t of the centre.
__device__ __forceinline__ int fast_arc_score_qr(const uint8_t* __restrict__ p, int pw, int t) {
    const int v = p[0];
    const int c0 = v - p[3 * pw], c8 = v - p[-3 * pw];
    bool dk = (c0 > t) | (c8 > t), br = (c0 < -t) | (c8 < -t);
    if (!(dk | br)) return 0;
    const int c4 = v - p[3], c12 = v - p[-3];
    dk &= (c4 > t) | (c12 > t); br &= (c4 < -t) | (c12 < -t);
    if (!(dk | br)) return 0;
    const int c2 = v - p[2 * pw + 2], c10 = v - p[-2 * pw - 2];
    dk &= (c2 > t) | (c10 > t); br &= (c2 < -t) | (c10 < -t);
    if (!(dk | br)) return 0;
    const int c6 = v - p[-2 * pw + 2], c14 = v - p[2 * pw - 2];
    dk &= (c6 > t) | (c14 > t); br &= (c6 < -t) | (c14 < -t);
    if (!(dk | br)) return 0;
    // both polarities at once: each ring difference d is packed as the s16x2 pair (d, -d); an arc's score for the
    // "darker" / "brighter" test is the min over its 9 packed entries, computed with Hopper's 3-input packed min
    // (VIMNMX3.S16x2): m3_k = min(q_k,q_k+1,q_k+2), m9_k = min(m3_k, m3_k+3, m3_k+6); M = max over k and both halves.
#define SE2_PK(dv) ((static_cast<unsigned>(dv) & 0xFFFFu) | (static_cast<unsigned>(-(dv)) << 16))
    unsigned q[16];
    q[0] = SE2_PK(c0);   q[1] = SE2_PK(v - p[3 * pw + 1]);    q[2] = SE2_PK(c2);    q[3] = SE2_PK(v - p[pw + 3]);
    q[4] = SE2_PK(c4);   q[5] = SE2_PK(v - p[-pw + 3]);       q[6] = SE2_PK(c6);    q[7] = SE2_PK(v - p[-3 * pw + 1]);
    q[8] = SE2_PK(c8);   q[9] = SE2_PK(v - p[-3 * pw - 1]);   q[10] = SE2_PK(c10);  q[11] = SE2_PK(v - p[-pw - 3]);
    q[12] = SE2_PK(c12); q[13] = SE2_PK(v - p[pw - 3]);       q[14] = SE2_PK(c14);  q[15] = SE2_PK(v - p[3 * pw - 1]);
#undef SE2_PK
    unsigned m3[16];
#pragma unroll
    for (int k = 0; k < 16; ++k) m3[k] = __vimin3_s16x2(q[k], q[(k + 1) & 15], q[(k + 2) & 15]);
    unsigned best = 0x80008000u;   // (-32768, -32768)
#pragma unroll
    for (int k = 0; k < 16; k += 2) {
        const unsigned a9 = __vimin3_s16x2(m3[k], m3[(k + 3) & 15], m3[(k + 6) & 15]);
        const unsigned b9 = __vimin3_s16x2(m3[k + 1], m3[(k + 4) & 15], m3[(k + 7) & 15]);
        best = __vimax3_s16x2(best, a9, b9);
    }
    const int mdark = static_cast<short>(best & 0xFFFFu), mbright = static_cast<short>(best >> 16);
    return max(mdark, mbright);
}

// Fallback for frames whose grid cells are too large for orb_fast_cells' shared-memory candidate list (e.g. 1080p with
// 1000 features: 470 x 150 px cells): one thread per pixel, no compaction, 2.2 bytes of shared memory per pixel.
// one CTA per (cell, frame): cv::FAST(cell, fastTh, NMS) and, if that yields <= 3 keypoints, cv::FAST(cell, 7, NMS)
// (ORBextractor.cpp:616-623). The cell and its 3 px apron are staged once in shared memory with aligned 32-bit loads.
// Work unit = one 32-pixel row segment per warp iteration (no per-pixel division); segments are numbered in raster
// order, so one exclusive scan over the per-segment survivor counts gives every keypoint its raster-order slot.
__global__ void __launch_bounds__(FAST_THREADS) orb_fast_cells_big(OrbDev d) {
    extern __shared__ uint8_t smem[];
    __shared__ int s_total;
    const CellGeo c = d.cells[blockIdx.x];
    const int f = blockIdx.y + d.frame0;
    CellHdr* hdr = d.hdr + (size_t)f * d.n_cells + blockIdx.x;
    const int cw = c.x1 - c.x0, ch = c.y1 - c.y0;
    if (c.skipped || cw <= 0 || ch <= 0) {
        if (threadIdx.x == 0) { hdr->n_base = 0; hdr->n_a = 0; hdr->n_b = 0; }
        return;
    }
    const LevelGeo& L = d.levels[c.level];
    const uint8_t* plane = d.plain + f * d.frame_plane_bytes + L.plane_off;
    // patch columns start at the 4-aligned bordered-plane column ax0 <= x0-3 (plane base and pitch are 32 B aligned)
    const int bx0 = c.x0 - 3 + EDGE, by0 = c.y0 - 3 + EDGE;
    const int ax0 = bx0 & ~3, shift = bx0 - ax0;
    const int ph = ch + 6, sw = cw + 2, sh = ch + 2;
    const int pww = (shift + cw + 6 + 3) >> 2, pw = pww * 4;
    uint8_t* patch = smem;
    uint8_t* score = smem + ((pw * ph + 15) & ~15);
    const int nseg = (cw + 31) >> 5, nchunk = ch * nseg;
    int* cnt = reinterpret_cast<int*>(score + ((sw * sh + 15) & ~15));   // [nchunk] survivors per segment -> exclusive offsets
    for (int i = threadIdx.x; i < pww * ph; i += FAST_THREADS) {
        const int py = i / pww, pxw = i - py * pww;
        reinterpret_cast<uint32_t*>(patch)[i] = *reinterpret_cast<const uint32_t*>(plane + (size_t)(by0 + py) * L.pitch + ax0 + 4 * pxw);
    }
    constexpr int NW = FAST_THREADS / 32;
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    const uint8_t* p0 = patch + 3 * pw + 3 + shift;
    int thr = d.fast_th;
    unsigned long long keepmask = 0;   // bit t: this lane's pixel of the warp's t-th segment survived NMS (first 64 segments)
    for (int pass = 0; pass < 2; ++pass) {
        for (int i = threadIdx.x; i < (sw * sh + 3) / 4; i += FAST_THREADS) reinterpret_cast<uint32_t*>(score)[i] = 0u;
        __syncthreads();
        for (int cidx = wid; cidx < nchunk; cidx += NW) {
            const int y = cidx / nseg, x = (cidx - y * nseg) * 32 + lane;
            if (x < cw) {
                const int m = fast_arc_score_qr(p0 + y * pw + x, pw, thr);
                if (m > thr) score[(y + 1) * sw + (x + 1)] = (uint8_t)(m - 1);
            }
        }
        __syncthreads();
        keepmask = 0;
        int t = 0;
        for (int cidx = wid; cidx < nchunk; cidx += NW, ++t) {
            const int y = cidx / nseg, x = (cidx - y * nseg) * 32 + lane;
            bool keep = false;
            if (x < cw) {
                const uint8_t* q = score + (y + 1) * sw + (x + 1);
                const int s = q[0];
                if (s) keep = s > q[-sw - 1] && s > q[-sw] && s > q[-sw + 1] && s > q[-1] && s > q[1] && s > q[sw - 1] && s > q[sw] && s > q[sw + 1];
            }
            const unsigned bal = __ballot_sync(0xffffffffu, keep);
            if (lane == 0) cnt[cidx] = __popc(bal);
            if (keep && t < 64) keepmask |= 1ull << t;
        }
        __syncthreads();
        if (wid == 0) {   // exclusive scan of the per-segment counts, in raster order
            int run = 0;
            for (int b0 = 0; b0 < nchunk; b0 += 32) {
                const int v = (b0 + lane < nchunk) ? cnt[b0 + lane] : 0;
                int inc = v;
#pragma unroll
                for (int o = 1; o < 32; o <<= 1) { const int u = __shfl_up_sync(0xffffffffu, inc, o); if (lane >= o) inc += u; }
                if (b0 + lane < nchunk) cnt[b0 + lane] = run + inc - v;
                run += __shfl_sync(0xffffffffu, inc, 31);
            }
            if (lane == 0) s_total = run;
        }
        __syncthreads();
        if (s_total > 3 || thr == 7) break;
        thr = 7;                 // cellKeyPoints.size() <= 3: clear and retry with the fixed fallback threshold
        __syncthreads();
    }
    uint32_t* out = d.cand + (size_t)f * d.cand_total + c.cand_off;
    int t = 0;
    for (int cidx = wid; cidx < nchunk; cidx += NW, ++t) {
        const int y = cidx / nseg, x = (cidx - y * nseg) * 32 + lane;
        bool keep;
        int s = 0;
        if (t < 64) {
            keep = (keepmask >> t) & 1ull;
        } else {
            keep = false;
            if (x < cw) {
                const uint8_t* q = score + (y + 1) * sw + (x + 1);
                s = q[0];
                if (s) keep = s > q[-sw - 1] && s > q[-sw] && s > q[-sw + 1] && s > q[-1] && s > q[1] && s > q[sw - 1] && s > q[sw] && s > q[sw + 1];
            }
        }
        const unsigned bal = __ballot_sync(0xffffffffu, keep);
        if (keep) {
            s = score[(y + 1) * sw + (x + 1)];
            const int pos = cnt[cidx] + __popc(bal & ((1u << lane) - 1));
            if (pos < c.cand_cap) out[pos] = ((uint32_t)s << 24) | ((uint32_t)(c.y0 + y) << 12) | (uint32_t)(c.x0 + x);
            else *d.err = 1;
        }
    }
    if (threadIdx.x == 0) { hdr->n_base = s_total; hdr->n_a = s_total; hdr->n_b = s_total; }
}

// HARRIS_SCORE: HarrisResponses(cellImage, cellKeyPoints, 7, HARRIS_K = 0.04f) (ORBextractor.cpp:85-126, called at :625-629 after
// the FAST / FAST(7) fallback of every cell). One CTA per (cell, frame), threads striding over the cell's candidate list in the
// raster order the FAST kernel left it (any of the three FAST kernels). A candidate's 7x7 block of 3x3 Sobel-like gradients
// reads the 9x9 footprint around it on the un-blurred level (4 px beyond the keypoint: one pixel past the cell's FAST apron,
// always inside the level ROI), as three aligned 32-bit words per row funnel-shifted to the footprint's first column.
// a = sum Ix^2, b = sum Iy^2, c = sum Ix*Iy in int32 (|Ix|, |Iy| <= 1020, 49 * 1020^2 < 2^31), then the reference's float
// expression in C++ evaluation order with every operation rounded on its own (no contraction):
//   ((float)a*b - (float)c*c - k*((float)a+b)*((float)a+b)) * scale_sq_sq,   scale_sq_sq = ((s*s)*s)*s,  s = 1/(4*7*255.f).
// Output: cand64[i] = resp_key(response) << 32 | cand[i], the FAST record kept in the low word.
constexpr int HARRIS_THREADS = 128;
constexpr float HARRIS_SCALE = 1.0f / ((1 << 2) * 7 * 255.0f);   // float arithmetic, folded by the compiler
constexpr float HARRIS_SCALE_SQ_SQ = HARRIS_SCALE * HARRIS_SCALE * HARRIS_SCALE * HARRIS_SCALE;
__global__ void __launch_bounds__(HARRIS_THREADS) orb_harris(OrbDev d, uint64_t* __restrict__ cand64) {
    const CellGeo c = d.cells[blockIdx.x];
    const int f = blockIdx.y + d.frame0;
    if (c.skipped) return;
    const int n = min(d.hdr[(size_t)f * d.n_cells + blockIdx.x].n_base, c.cand_cap);
    if (n <= 0) return;
    const LevelGeo& L = d.levels[c.level];
    const uint8_t* plane = d.plain + f * d.frame_plane_bytes + L.plane_off;
    const size_t co = (size_t)f * d.cand_total + c.cand_off;
    const uint32_t* cand = d.cand + co;
    for (int i = threadIdx.x; i < n; i += HARRIS_THREADS) {
        const uint32_t rec = cand[i];
        const int x = rec & 0xFFF, y = (rec >> 12) & 0xFFF;
        const int bx = EDGE + x - 4, ax = bx & ~3;
        const unsigned sh = 8u * (unsigned)(bx - ax);
        const uint8_t* row0 = plane + (size_t)(EDGE + y - 4) * L.pitch + ax;
        int p[9][9];
#pragma unroll
        for (int r = 0; r < 9; ++r) {
            const uint32_t* w = reinterpret_cast<const uint32_t*>(row0 + (size_t)r * L.pitch);
            const uint32_t w0 = __ldg(w), w1 = __ldg(w + 1), w2 = __ldg(w + 2);
            const uint32_t lo = __funnelshift_r(w0, w1, sh), mid = __funnelshift_r(w1, w2, sh), hi = __funnelshift_r(w2, 0u, sh);
#pragma unroll
            for (int k = 0; k < 4; ++k) { p[r][k] = __byte_perm(lo, 0u, 0x4440 + k); p[r][4 + k] = __byte_perm(mid, 0u, 0x4440 + k); }
            p[r][8] = hi & 0xFF;
        }
        int a = 0, b = 0, cc = 0;
#pragma unroll
        for (int r = 1; r < 8; ++r)
#pragma unroll
            for (int k = 1; k < 8; ++k) {
                const int Ix = (p[r][k + 1] - p[r][k - 1]) * 2 + (p[r - 1][k + 1] - p[r - 1][k - 1]) + (p[r + 1][k + 1] - p[r + 1][k - 1]);
                const int Iy = (p[r + 1][k] - p[r - 1][k]) * 2 + (p[r + 1][k - 1] - p[r - 1][k - 1]) + (p[r + 1][k + 1] - p[r - 1][k + 1]);
                a += Ix * Ix; b += Iy * Iy; cc += Ix * Iy;
            }
        const float fa = __int2float_rn(a), fb = __int2float_rn(b), fc = __int2float_rn(cc);
        const float apb = __fadd_rn(fa, fb);
        const float t = __fsub_rn(__fsub_rn(__fmul_rn(fa, fb), __fmul_rn(fc, fc)), __fmul_rn(__fmul_rn(0.04f, apb), apb));
        const float resp = __fmul_rn(t, HARRIS_SCALE_SQ_SQ);
        cand64[co + i] = ((uint64_t)se2gpu::resp_key(resp) << 32) | rec;
    }
}

// Selection (:625-710) in two launches, neither of which leaves one CTA to carry a pyramid level:
//   orb_select_cells   one warp per (cell, frame): the level's quota redistribution :631-679, computed warp-cooperatively by
//                      every warp of the level (integer sums, so any summation order gives the reference's numbers), then
//                      KeyPointsFilter::retainBest of its own cell (:687-694) and the survivors copied to the cell's slot range
//                      in the level list (d.sel, cells in order); the level's cell 0 also writes the list length to d.lcount
//   orb_select_levels  one warp per (level, frame): retainBest of the level list (:706-710) into the keypoint buffer
// retainBest is std::nth_element: the warp-cooperative introselect of introselect.h reproduces libstdc++'s permutation. A cell
// list that fits the warp's SEL_STAGE_BYTES of shared memory is selected in the warp's shared memory, a longer one in place in global memory.
// Level 0, which has by far the most candidates, is then as many warps as it has cells, spread over the GPU, and its level-wide
// nth_element runs on at most about 2 * nDesired survivors.
// HARRIS: the records are orb_harris' 64-bit ones (cand64, selected by their upper word), and the level lists are written as the
// 32-bit FAST records plus the float responses in lresp.
// PDL: both launch as programmatic dependents; each releases its dependent at once, and reads what its predecessor wrote only
// behind griddepcontrol.wait.
constexpr int SEL_WARPS = 4;            // warps (cells) per orb_select_cells CTA
// shared memory per warp for its cell list. Measured on an H100 SXM (700 W), 64 frames of 640x480, ms per step: 0.5550 at
// 2 KB, 0.5545 at 4 KB, 0.5632 at 8 KB, 0.568-0.571 at 12 and 16 KB (fewer resident warps for a latency-bound kernel)
constexpr int SEL_STAGE_BYTES = 4096;
constexpr int SEL_NOMORE = 1 << 30;     // bNoMore flag next to a cell's nToRetain
struct HarrisBufs { uint64_t* cand64; float* lresp; };   // orb_select_*<true> / orb_orient_describe<true> only

__device__ __forceinline__ int warp_sum(int v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

template <bool HARRIS>
__global__ void __launch_bounds__(SEL_WARPS * 32) orb_select_cells(OrbDev d, HarrisBufs hb, int max_cells, int stage_n) {
    typedef typename std::conditional<HARRIS, se2gpu::KpKey64, se2gpu::KpScore32>::type K;
    typedef typename K::rec R;
    extern __shared__ __align__(16) uint8_t selc_smem[];   // [SEL_WARPS][stage_n] records | [SEL_WARPS][2][max_cells] ints
    __shared__ int wq[SEL_WARPS][128];
    asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    const int cell = blockIdx.y * SEL_WARPS + wid, f = blockIdx.x + d.frame0;   // frames fastest: see run_device
    if (cell >= d.n_cells) return;
    const CellGeo c = d.cells[cell];
    const int level = c.level;
    const LevelGeo& L = d.levels[level];
    const int nCells = L.nCells, cb = L.cell_base, nfc = L.nfeaturesCell, me = cell - cb;
    R* stage = reinterpret_cast<R*>(selc_smem) + wid * stage_n;
    int* nTotal = reinterpret_cast<int*>(reinterpret_cast<R*>(selc_smem) + SEL_WARPS * stage_n) + wid * 2 * max_cells;
    int* nToRetain = nTotal + max_cells;     // | SEL_NOMORE once bNoMore
    asm volatile("griddepcontrol.wait;" ::: "memory");     // the FAST (Harris) candidates are complete and visible from here on
    const CellHdr* hdr = d.hdr + (size_t)f * d.n_cells + cb;
    // :631-679; skipped cells never enter the first pass (nToRetain/nTotal stay 0, bNoMore stays false)
    int nToDistribute = 0, nNoMore = 0;
    for (int k = lane; k < nCells; k += 32) {
        const bool skipped = d.cells[cb + k].skipped;
        const int t = skipped ? 0 : hdr[k].n_base;
        int r = 0;
        if (!skipped) {
            if (t > nfc) r = nfc;
            else { r = t | SEL_NOMORE; nToDistribute += nfc - t; ++nNoMore; }
        }
        nTotal[k] = t; nToRetain[k] = r;
    }
    nToDistribute = warp_sum(nToDistribute); nNoMore = warp_sum(nNoMore);
    while (nToDistribute > 0 && nNoMore < nCells) {
        const int nNew = (int)((float)nfc + ceilf((float)nToDistribute / (float)(nCells - nNoMore)));
        int dist = 0, more = 0;
        for (int k = lane; k < nCells; k += 32) {
            if (nToRetain[k] & SEL_NOMORE) continue;
            const int t = nTotal[k];
            if (t > nNew) nToRetain[k] = nNew;
            else { nToRetain[k] = t | SEL_NOMORE; dist += nNew - t; ++more; }
        }
        nToDistribute = warp_sum(dist); nNoMore += warp_sum(more);
    }
    // the cell's slot in the level list: the survivors min(nTotal, nToRetain) of the cells before it
    int before = 0, all = 0;
    for (int k = lane; k < nCells; k += 32) {
        const int kept = min(nTotal[k], nToRetain[k] & ~SEL_NOMORE);
        all += kept;
        if (k < me) before += kept;
    }
    before = warp_sum(before); all = warp_sum(all);
    __syncwarp();
    const int cap = L.sel_cap;
    if (me == 0 && lane == 0) {
        if (all > cap) *d.err = 2;
        d.lcount[f * d.nlevels + level] = min(all, cap);
    }
    const int tot = nTotal[me], n = nToRetain[me] & ~SEL_NOMORE, kept = min(tot, n);
    if (kept <= 0 || before >= cap) return;
    R* g;
    if constexpr (HARRIS) g = hb.cand64 + (size_t)f * d.cand_total + c.cand_off;
    else g = d.cand + (size_t)f * d.cand_total + c.cand_off;
    R* v = g;
    if (tot > n) {   // KeyPointsFilter::retainBest + resize (:692-694)
        if (tot <= stage_n) {
            v = stage;
            for (int i = lane; i < tot; i += 32) v[i] = g[i];
            __syncwarp();
        }
        se2gpu::kp_nth_element_warp<K>(v, tot, n - 1, wq[wid]);
    }
    R* out = reinterpret_cast<R*>(d.sel) + (size_t)f * d.sel_total + L.sel_off + before;
    for (int i = lane; i < kept && before + i < cap; i += 32) out[i] = v[i];
}

template <bool HARRIS>
__global__ void __launch_bounds__(32) orb_select_levels(OrbDev d, HarrisBufs hb) {
    typedef typename std::conditional<HARRIS, se2gpu::KpKey64, se2gpu::KpScore32>::type K;
    typedef typename K::rec R;
    extern __shared__ __align__(16) uint8_t sell_smem[];   // [sel_cap] records of the level list
    __shared__ int wq[128];
    asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
    const int lane = threadIdx.x, level = blockIdx.x, f = blockIdx.y + d.frame0;
    const LevelGeo& L = d.levels[level];
    R* v = reinterpret_cast<R*>(sell_smem);
    const R* g = reinterpret_cast<const R*>(d.sel) + (size_t)f * d.sel_total + L.sel_off;
    int* lc = d.lcount + f * d.nlevels + level;
    asm volatile("griddepcontrol.wait;" ::: "memory");     // the level list is complete and visible from here on
    int total = *lc;
    for (int i = lane; i < total; i += 32) v[i] = g[i];
    __syncwarp();
    if (total > L.nDesired) {  // :706-710
        se2gpu::kp_nth_element_warp<K>(v, total, L.nDesired - 1, wq);
        total = L.nDesired;
    }
    uint32_t* out = d.lkp + (size_t)f * d.lkp_total + L.kp_off;
    if constexpr (HARRIS) {
        float* resp = hb.lresp + (size_t)f * d.lkp_total + L.kp_off;
        for (int i = lane; i < total; i += 32) { const R r = v[i]; out[i] = (uint32_t)r; resp[i] = se2gpu::resp_from_key((uint32_t)(r >> 32)); }
    } else {
        for (int i = lane; i < total; i += 32) out[i] = v[i];
    }
    __syncwarp();
    if (lane == 0) *lc = total;
}

// test hook: one warp per list, lists in global memory
__global__ void __launch_bounds__(128) orb_debug_nth(uint32_t* v, const int* __restrict__ offs, const int* __restrict__ nth, int count) {
    __shared__ int wq[4][128];
    const int k = blockIdx.x * 4 + (threadIdx.x >> 5);
    if (k >= count) return;
    se2gpu::kp_nth_element_warp(v + offs[k], offs[k + 1] - offs[k], nth[k], wq[threadIdx.x >> 5]);
}

// test hook: the same on 64-bit records keyed by their upper word (the Harris-score selection)
__global__ void __launch_bounds__(128) orb_debug_nth64(uint64_t* v, const int* __restrict__ offs, const int* __restrict__ nth, int count) {
    __shared__ int wq[4][128];
    const int k = blockIdx.x * 4 + (threadIdx.x >> 5);
    if (k >= count) return;
    se2gpu::kp_nth_element_warp<se2gpu::KpKey64>(v + offs[k], offs[k + 1] - offs[k], nth[k], wq[threadIdx.x >> 5]);
}

// GaussianBlur 7x7 sigma 2 on the level ROI; the 16 px ring keeps its un-blurred reflect-101 copies.
// cv::GaussianBlur's float arithmetic: row pass = sequential fmaf over the 7 taps, column pass = centre tap then the
// three symmetric pairs, round-to-nearest-even, saturate. No shared memory, so the CTAs co-reside with the resize and FAST CTAs.
// A thread owns 8 adjacent columns (one column group) of one strip of ROI rows and walks down it with the last 7 row-pass results
// in a register ring: per source row one 8-byte load of its columns and two 4-byte loads of the neighbouring bytes (L1 hits), per
// output row one 8-byte store. A level's strips have one height (the last one is moved up to end at the ROI's last row, so a few
// rows are blurred twice, with the same result); a warp takes 32 consecutive (strip, column group) items of one level, so lanes
// idle only in a level's last warp. Only ROI rows are blurred: their 7-row windows and the neighbour words stay inside the
// bordered plane (beyond a row's ends the neighbour word is the adjacent row's, which only feeds ring columns), so no row index is
// clamped and no load is tested; the lanes of the first and the last strip copy the 16 ring rows above and below.
// The kernel is issue bound: bytes become floats and rounded sums become bytes through the float bit patterns (blur_px.h), which
// keeps it off the conversion pipe; 8 columns per thread share the 6 neighbour conversions of a row.
__global__ void __launch_bounds__(BLUR_WARPS * 32, 4) orb_blur(OrbDev d, int tile0, int tile_end) {
    const int tile = tile0 + blockIdx.x * BLUR_WARPS + (threadIdx.x >> 5);
    if (tile >= tile_end) return;
    const TileGeo t = d.tiles[tile];
    const LevelGeo& L = d.levels[t.level];
    const int pitch = L.pitch, Lw = L.w, Lh = L.h, th = L.blur_th, strips = L.blur_strips, ncg = pitch / 8;
    int s = t.strip, cg = t.cg + (threadIdx.x & 31);   // lane j: item j after the tile's first one, strip by strip
    while (cg >= ncg) { cg -= ncg; ++s; }
    if (s >= strips) return;
    const int x8 = 8 * cg;
    const size_t off = (size_t)(blockIdx.y + d.frame0) * d.frame_plane_bytes + L.plane_off + x8;
    const uint8_t* __restrict__ src = d.plain + off;
    uint8_t* __restrict__ dst = d.blurred + off;
    if (s == 0)
        for (int y = 0; y < EDGE; ++y) *reinterpret_cast<uint2*>(dst + (size_t)y * pitch) = __ldg(reinterpret_cast<const uint2*>(src + (size_t)y * pitch));
    if (s == strips - 1)
        for (int y = EDGE + Lh; y < Lh + 2 * EDGE; ++y) *reinterpret_cast<uint2*>(dst + (size_t)y * pitch) = __ldg(reinterpret_cast<const uint2*>(src + (size_t)y * pitch));
    uint32_t m0 = 0, m1 = 0;       // 0xFF in the byte lanes of ROI columns
#pragma unroll
    for (int q = 0; q < 4; ++q) {
        m0 |= (x8 + q >= EDGE && x8 + q < EDGE + Lw) ? (0xFFu << (8 * q)) : 0u;
        m1 |= (x8 + 4 + q >= EDGE && x8 + 4 + q < EDGE + Lw) ? (0xFFu << (8 * q)) : 0u;
    }
    const int y0 = EDGE + min(s * th, Lh - th);   // first output row of the strip
    const uint8_t* rp = src + (size_t)(y0 - 3) * pitch;
    uint8_t* wp = dst + (size_t)y0 * pitch;
    float hr[7][8];      // row-pass results of the last 7 source rows
    uint2 cw[7];         // their own 8 bytes (ring columns are copied through)
    uint2 nc = __ldg(reinterpret_cast<const uint2*>(rp));     // the next source row (software prefetch, one row ahead)
    uint32_t nl = __ldg(reinterpret_cast<const uint32_t*>(rp - 4)), nr = __ldg(reinterpret_cast<const uint32_t*>(rp + 8));
    auto row = [&](const int k) {      // row pass of the next source row into ring slot k
        const uint2 c = nc;
        const uint32_t l = nl, r = nr;
        rp += pitch;
        nc = __ldg(reinterpret_cast<const uint2*>(rp));
        nl = __ldg(reinterpret_cast<const uint32_t*>(rp - 4));
        nr = __ldg(reinterpret_cast<const uint32_t*>(rp + 8));
        float b[14];                    // bytes x8-3 .. x8+10
#pragma unroll
        for (int j = 0; j < 3; ++j) b[j] = blurpx::byte_to_float(l, j + 1);
#pragma unroll
        for (int j = 0; j < 4; ++j) { b[3 + j] = blurpx::byte_to_float(c.x, j); b[7 + j] = blurpx::byte_to_float(c.y, j); }
#pragma unroll
        for (int j = 0; j < 3; ++j) b[11 + j] = blurpx::byte_to_float(r, j);
#pragma unroll
        for (int q = 0; q < 8; ++q) {
            float a = __fmul_rn(c_gauss[0], b[q]);
            a = __fmaf_rn(c_gauss[1], b[q + 1], a); a = __fmaf_rn(c_gauss[2], b[q + 2], a); a = __fmaf_rn(c_gauss[3], b[q + 3], a);
            a = __fmaf_rn(c_gauss[4], b[q + 4], a); a = __fmaf_rn(c_gauss[5], b[q + 5], a); a = __fmaf_rn(c_gauss[6], b[q + 6], a);
            hr[k][q] = a;
        }
        cw[k] = c;
    };
    auto out = [&](const int k) {      // column pass of the output row whose 7-row window ends in slot k; centre row in slot (k + 4) % 7
        unsigned o[8];
#pragma unroll
        for (int q = 0; q < 8; ++q) {
            float a = __fmul_rn(c_gauss[3], hr[(k + 4) % 7][q]);
            a = __fmaf_rn(c_gauss[4], __fadd_rn(hr[(k + 5) % 7][q], hr[(k + 3) % 7][q]), a);
            a = __fmaf_rn(c_gauss[5], __fadd_rn(hr[(k + 6) % 7][q], hr[(k + 2) % 7][q]), a);
            a = __fmaf_rn(c_gauss[6], __fadd_rn(hr[k][q], hr[(k + 1) % 7][q]), a);
            o[q] = blurpx::round_sat_bits(a);
        }
        const uint2 ctr = cw[(k + 4) % 7];
        const uint32_t v0 = blurpx::pack_low_bytes(o[0], o[1], o[2], o[3]), v1 = blurpx::pack_low_bytes(o[4], o[5], o[6], o[7]);
        *reinterpret_cast<uint2*>(wp) = make_uint2((v0 & m0) | (ctr.x & ~m0), (v1 & m1) | (ctr.y & ~m1));
        wp += pitch;
    };
#pragma unroll
    for (int k = 0; k < 7; ++k) row(k);   // source rows y0-3 .. y0+3
    out(6);                                // output row y0
    for (int i = 1; i < th; i += 7) {      // th - 1 is a multiple of 7 (build_geometry)
#pragma unroll
        for (int k = 0; k < 7; ++k) { row(k); out(k); }
    }
}

// cv::fastAtan2 (degrees), scalar float path without contraction
__device__ __forceinline__ float fast_atan2_deg(float y, float x) {
    const float p1 = 0.9997878412794807f * (float)(180 / M_PI);
    const float p3 = -0.3258083974640975f * (float)(180 / M_PI);
    const float p5 = 0.1555786518463281f * (float)(180 / M_PI);
    const float p7 = -0.04432655554792128f * (float)(180 / M_PI);
    const float ax = fabsf(x), ay = fabsf(y);
    float a, c, c2;
    if (ax >= ay) {
        c = __fdiv_rn(ay, __fadd_rn(ax, (float)2.2204460492503131e-16));
        c2 = __fmul_rn(c, c);
        a = __fmul_rn(__fadd_rn(__fmul_rn(__fadd_rn(__fmul_rn(__fadd_rn(__fmul_rn(p7, c2), p5), c2), p3), c2), p1), c);
    } else {
        c = __fdiv_rn(ax, __fadd_rn(ay, (float)2.2204460492503131e-16));
        c2 = __fmul_rn(c, c);
        a = __fsub_rn(90.f, __fmul_rn(__fadd_rn(__fmul_rn(__fadd_rn(__fmul_rn(__fadd_rn(__fmul_rn(p7, c2), p5), c2), p3), c2), p1), c));
    }
    if (x < 0) a = __fsub_rn(180.f, a);
    if (y < 0) a = __fsub_rn(360.f, a);
    return a;
}

// one warp per output keypoint slot: orientation on the plain level, descriptor on the blurred level.
// The disc column of a lane is read in three batches of 5 row pairs with all 10 loads of a batch issued before their sums
// (predicated off beyond the column's half-height) instead of one dependent +-v pair per loop trip, and the 16 descriptor taps of
// a lane are loaded back to back: the kernel is bound by the latency of first-touch sectors (every plane byte comes from DRAM
// once), so the loads in flight per warp set its speed. Integer moments: any summation order gives the reference's m10, m01.
// HARRIS: the keypoint's response is the Harris response orb_select_levels<true> left in lresp, else the FAST score of the record.
template <bool HARRIS>
__global__ void __launch_bounds__(256) orb_orient_describe(OrbDev d, se2gpu_keypoint* __restrict__ kps, uint8_t* __restrict__ desc,
                                                           int* __restrict__ counts, const float* __restrict__ lresp) {
    __shared__ float4 patf[256];     // the 256 point pairs of the rBRIEF pattern as floats (x0, y0, x1, y1); test 8*lane+k at [k][lane]
    for (int i = threadIdx.x; i < 256; i += blockDim.x) patf[(i & 7) * 32 + (i >> 3)] = make_float4((float)d_pattern[4 * i], (float)d_pattern[4 * i + 1], (float)d_pattern[4 * i + 2], (float)d_pattern[4 * i + 3]);
    __syncthreads();
    asm volatile("griddepcontrol.wait;" ::: "memory");     // programmatic dependent of the selection: the level lists are complete from here on
    const int f = blockIdx.y + d.frame0;
    const int slot = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    const int* lc = d.lcount + f * d.nlevels;
    int level = -1, off = 0, total = 0;
    for (int l = 0; l < d.nlevels; ++l) {
        const int c = lc[l];
        if (level < 0 && slot < total + c) { level = l; off = total; }
        total += c;
    }
    if (slot == 0 && lane == 0) counts[f] = total;
    if (level < 0) return;
    const LevelGeo& L = d.levels[level];
    const size_t kslot = (size_t)f * d.lkp_total + L.kp_off + (slot - off);
    const uint32_t rec = d.lkp[kslot];
    const int x = rec & 0xFFF, y = (rec >> 12) & 0xFFF, score = rec >> 24;
    const size_t base = f * d.frame_plane_bytes + L.plane_off + (size_t)(EDGE + y) * L.pitch + (EDGE + x);
    const uint8_t* center = d.plain + base;
    // IC_Angle: lane = column u = lane-15 of the 31x31 patch disc; it sums its rows in +-v pairs up to the column's half-height
    int m10 = 0, m01 = 0;
    if (lane < 31) {
        const int u = lane - HALF_PATCH, vm = c_vmax[abs(u)];
        const uint8_t* col = center + u;
        const int pitch = L.pitch;
        int colsum = col[0];
#pragma unroll
        for (int v0 = 1; v0 <= HALF_PATCH; v0 += 5) {
            int p[5], m[5];
#pragma unroll
            for (int k = 0; k < 5; ++k) {       // rows beyond the half-height re-read row vm (a cache hit) and are dropped below
                const int off = min(v0 + k, vm) * pitch;
                p[k] = col[off]; m[k] = col[-off];
            }
#pragma unroll
            for (int k = 0; k < 5; ++k)
                if (v0 + k <= vm) { colsum += p[k] + m[k]; m01 += (v0 + k) * (p[k] - m[k]); }
        }
        m10 = u * colsum;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) { m10 += __shfl_xor_sync(0xffffffffu, m10, o); m01 += __shfl_xor_sync(0xffffffffu, m01, o); }
    const float angle = fast_atan2_deg((float)m01, (float)m10);
    // steered BRIEF: a = (float)cos((double)angle_rad), b = (float)sin(...)
    const float factorPI = (float)(M_PI / 180.f);
    const float ang = __fmul_rn(angle, factorPI);
    double sd, cd;
    sincos((double)ang, &sd, &cd);
    const float a = (float)cd, b = (float)sd;
    const uint8_t* bc = d.blurred + base;
    unsigned val = 0;
    // all 16 tap offsets first, then the 16 loads back to back, then the comparisons
    int o0[8], o1[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) {
        const float4 pt = patf[k * 32 + lane];
        const float x0 = pt.x, y0 = pt.y, x1 = pt.z, y1 = pt.w;
        const int r0 = __float2int_rn(__fadd_rn(__fmul_rn(x0, b), __fmul_rn(y0, a)));
        const int c0 = __float2int_rn(__fsub_rn(__fmul_rn(x0, a), __fmul_rn(y0, b)));
        const int r1 = __float2int_rn(__fadd_rn(__fmul_rn(x1, b), __fmul_rn(y1, a)));
        const int c1 = __float2int_rn(__fsub_rn(__fmul_rn(x1, a), __fmul_rn(y1, b)));
        o0[k] = r0 * L.pitch + c0; o1[k] = r1 * L.pitch + c1;
    }
    int t0[8], t1[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) { t0[k] = bc[o0[k]]; t1[k] = bc[o1[k]]; }
#pragma unroll
    for (int k = 0; k < 8; ++k) val |= (unsigned)(t0[k] < t1[k]) << k;
    // pack 4 bytes per lane group: lane 4q gets bytes 4q..4q+3
    unsigned w = val;
    w |= __shfl_down_sync(0xffffffffu, val, 1) << 8;
    w |= __shfl_down_sync(0xffffffffu, val, 2) << 16;
    w |= __shfl_down_sync(0xffffffffu, val, 3) << 24;
    const size_t oslot = (size_t)f * d.nfeatures + slot;
    if ((lane & 3) == 0) reinterpret_cast<unsigned*>(desc + oslot * 32)[lane >> 2] = w;
    if (lane == 0) {
        se2gpu_keypoint kp;
        kp.x = level ? __fmul_rn((float)x, L.scale) : (float)x;
        kp.y = level ? __fmul_rn((float)y, L.scale) : (float)y;
        kp.size = L.kp_size; kp.angle = angle; kp.response = HARRIS ? lresp[kslot] : (float)score; kp.octave = level; kp.class_id = -1;
        kps[oslot] = kp;
    }
}

inline int cv_round_f(float v) { return (int)lrintf(v); }

}  // namespace

// =================================================================================================
struct se2gpu_orb {
    int device = 0, nfeatures = 0, nlevels = 0, fast_th = 20, max_w = 0, max_h = 0, max_batch = 0;
    bool harris = false;         // scoreType == HARRIS_SCORE: orb_harris + the 64-bit selection
    double scaleFactor = 1.2;
    std::vector<float> mvScaleFactor, mvInvScaleFactor;
    std::vector<int> mnFeaturesPerLevel;
    // geometry of the current frame size
    int cur_w = -1, cur_h = -1;
    std::vector<LevelGeo> levels;
    std::vector<CellGeo> cells;
    std::vector<TileGeo> tiles;
    size_t fast_smem = 0, select_smem = 0, select_levels_smem = 0, resize_w_smem = 0;
    int sel_max_cells = 0;       // most cells of a level: orb_select_cells' per-warp quota arrays
    int sel_stage_n = 0;         // records of a cell list orb_select_cells stages per warp
    int resize_rows = 0, resize_raw_pitch = 0;   // shared-memory box of orb_resize_w, sized from the scale factor
    int resize_tall_rows = 0; size_t resize_tall_smem = 0;   // the same for RESIZE_TR_TALL-row tiles
    int resize_tall_ctas = 0;    // resident CTAs of orb_resize_w<RESIZE_TR_TALL> on the whole GPU; 0: tall tiles are not used
    bool fast_big = false;       // cells too large for the compacting FAST kernel: use orb_fast_cells_big
    bool fast_tma = false;       // cells staged by the TMA unit: orb_fast_cells<true>, else orb_fast_cells<false>
    size_t fast_tma_smem = 0;
    FastMaps fast_maps{};        // kernel parameter (__grid_constant__): one tensor map per level over d.plain
    // optional lens undistortion folded into level 0 (se2gpu_orb_set_undistort)
    bool und_on = false;
    float und_K[9] = {}, und_D[14] = {};
    int und_nd = 0, und_w = 0, und_h = 0;
    short2* d_und_m1 = nullptr; uint16_t* d_und_m2 = nullptr; size_t und_cap = 0;
    // capacities (computed for max_w x max_h)
    size_t cap_plane = 0, cap_cand = 0, cap_cells = 0, cap_tiles = 0, cap_tab = 0, cap_lkp = 0, cap_sel = 0;
    OrbDev d{};
    LevelGeo* d_levels = nullptr; CellGeo* d_cells = nullptr; TileGeo* d_tiles = nullptr; int* d_itab = nullptr; short* d_stab = nullptr;

    uint8_t* d_in = nullptr; se2gpu_keypoint* d_kps = nullptr; uint8_t* d_desc = nullptr; int* d_counts = nullptr;
    HarrisBufs hb{};             // HARRIS_SCORE handles only: [B][cand_total] 64-bit records, [B][lkp_total] level-list responses
    se2gpu::DeviceBuffers bufs;
    int last_n = 0;
    se2gpu::Profiler prof;
    cudaStream_t side = nullptr;          // blur runs here, concurrently with FAST + selection
    cudaEvent_t ev_pyr = nullptr, ev_blur = nullptr;
    // host-buffer path: two pipeline lanes (stream + side stream + events) so that the H2D of chunk c+1 and the D2H of
    // chunk c-1 overlap the kernels of chunk c
    cudaStream_t pipe[ORB_LANES] = {};   // host-path pipeline lanes (chunk k runs on lane k % lanes)
    // pinned staging for results when the caller's buffers are pageable (a D2H copy into pageable memory blocks the
    // host and would serialise the pipeline)
    int* pin_counts = nullptr; se2gpu_keypoint* pin_kps = nullptr; uint8_t* pin_desc = nullptr;
    // a host-buffer job that has been enqueued but not yet finished (se2gpu_orb_submit / _wait; se2gpu_orb_extract = both)
    struct Pending { bool on = false; int n = 0, lanes = 0; bool pipelined = false; se2gpu_keypoint* kps = nullptr; uint8_t* desc = nullptr; int* counts = nullptr;
                     se2gpu_keypoint* out_kps = nullptr; uint8_t* out_desc = nullptr; int* out_counts = nullptr; } pend;
    // asynchronous two-deep submission: a second, identical context so that two batches can be in flight (the copy engines move
    // batch k+1 in and batch k-1 out while the SMs work on batch k)
    se2gpu_orb* twin = nullptr;
    int submit_next = 0, wait_next = 0, in_flight = 0;
    int create_args[9] = {};
};

namespace {

// level geometry exactly as ORBextractor::ComputePyramid / ComputeKeyPoints derive it (float32 arithmetic)
int build_geometry(se2gpu_orb* h, int w, int hgt, bool dry, size_t* plane_bytes, size_t* cand_total, size_t* n_cells,
                   size_t* n_tiles, size_t* tab_total, size_t* max_fast_smem,
                   std::vector<LevelGeo>* Lv, std::vector<CellGeo>* Cv, std::vector<TileGeo>* Tv, bool* fast_big_out = nullptr,
                   size_t* fast_tma_smem_out = nullptr) {
    (void)dry;
    const int nl = h->nlevels;
    std::vector<LevelGeo> L(nl);
    std::vector<CellGeo> C;
    std::vector<TileGeo> T;
    size_t poff = 0, coff = 0, toff = 0, fsm = 0, fsm_big = 0, fsm_tma = 0;
    bool fast_big = false;   // some cell is too large for orb_fast_cells' shared-memory candidate list -> orb_fast_cells_big
    bool tma_ok = true;      // every level's cell patch fits a TMA box (<= 256 x 256) and 16-bit list offsets
    int kp_off = 0, sel_off = 0;
    const float imageRatio = (float)w / (float)hgt;   // mvImagePyramid[0].cols/rows (:538)
    for (int l = 0; l < nl; ++l) {
        LevelGeo& g = L[l];
        const float scale = h->mvInvScaleFactor[l];
        g.w = cv_round_f((float)w * scale); g.h = cv_round_f((float)hgt * scale);   // :794-795
        if (g.w < 2 * EDGE + 7 || g.h < 2 * EDGE + 7) return fail(SE2GPU_ERR_INVALID, "level %d of a %dx%d frame is %dx%d: too small for the 16 px border", l, w, hgt, g.w, g.h);
        if (g.w + 2 * EDGE > 4095 || g.h + 2 * EDGE > 4095) return fail(SE2GPU_ERR_CAPACITY, "frames wider/taller than 4063 px are not supported");
        g.pitch = (g.w + 2 * EDGE + 31) & ~31;
        g.plane_off = poff;
        poff += (size_t)g.pitch * (g.h + 2 * EDGE);
        poff = (poff + 255) & ~(size_t)255;
        g.nDesired = h->mnFeaturesPerLevel[l];
        g.cols = (int)sqrtf((float)g.nDesired / (5 * imageRatio));   // :542
        g.rows = (int)(imageRatio * g.cols);                          // :543
        if (g.cols < 1 || g.rows < 1) return fail(SE2GPU_ERR_INVALID, "level %d has a %dx%d cell grid (nfeatures too small): undefined in the reference", l, g.cols, g.rows);
        const int minB = EDGE, maxBX = g.w - EDGE, maxBY = g.h - EDGE;
        const int W = maxBX - minB, H = maxBY - minB;
        const int cellW = (int)ceilf((float)W / g.cols), cellH = (int)ceilf((float)H / g.rows);
        g.nCells = g.rows * g.cols;
        g.nfeaturesCell = (int)ceilf((float)g.nDesired / g.nCells);
        g.cell_base = (int)C.size();
        g.kp_off = kp_off; g.kp_cap = g.nDesired; kp_off += g.nDesired;
        g.scale = h->mvScaleFactor[l];
        g.kp_size = (float)(int)(PATCH * h->mvScaleFactor[l]);
        g.tab_off = (int)toff; toff += (size_t)g.w + g.h;
        std::vector<int> iniXCol(g.cols, 0);
        const size_t first_cell = C.size();
        int max_cw = 0, max_ch = 0;
        float hY = cellH + 6;
        for (int i = 0; i < g.rows; ++i) {
            const float iniY = minB + i * cellH - 3;
            bool rowSkipped = false;
            if (i == g.rows - 1) { hY = maxBY + 3 - iniY; if (hY <= 0) rowSkipped = true; }
            float hX = cellW + 6;
            for (int j = 0; j < g.cols; ++j) {
                CellGeo c{};
                c.level = l;
                if (rowSkipped) { c.skipped = 1; C.push_back(c); continue; }
                float iniX;
                if (i == 0) { iniX = minB + j * cellW - 3; iniXCol[j] = (int)iniX; } else iniX = iniXCol[j];
                if (j == g.cols - 1) { hX = maxBX + 3 - iniX; if (hX <= 0) { c.skipped = 1; C.push_back(c); continue; } }
                const int r0 = (int)iniY, r1 = (int)(iniY + hY), c0 = (int)iniX, c1 = (int)(iniX + hX);
                if (r1 > g.h || c1 > g.w || r0 < 0 || c0 < 0) return fail(SE2GPU_ERR_INVALID, "cell grid of level %d leaves the image (the reference asserts here)", l);
                c.x0 = c0 + 3; c.x1 = c1 - 3; c.y0 = r0 + 3; c.y1 = r1 - 3;
                const int cw = std::max(c.x1 - c.x0, 0), chh = std::max(c.y1 - c.y0, 0);
                c.cand_off = (int)coff;
                c.cand_cap = ((cw + 1) / 2) * ((chh + 1) / 2) + 8;   // strict 3x3 maxima: at most one per 2x2 block
                coff += c.cand_cap;
                if (cw > 0 && chh > 0) {
                    max_cw = std::max(max_cw, ((c.x0 - 3 + EDGE) & 15) + cw); max_ch = std::max(max_ch, chh);   // incl. the TMA alignment shift
                    const size_t pwb = (size_t)((cw + 6 + 3 + 3) / 4 + 1) * 4;   // worst-case alignment shift
                    const size_t bitmap = (size_t)chh * fastpx::nms_words_per_row(cw) * 4;
                    if (pwb * (chh + 6) > 65535) fast_big = true;    // 16-bit patch offsets in the candidate list
                    fsm = std::max(fsm, ((pwb * (chh + 6) + 15) & ~(size_t)15) + (((size_t)fastpx::nms_plane_bytes((int)pwb, chh) + 15) & ~(size_t)15) + bitmap + (size_t)cw * chh * 2 + 64);
                    const size_t nchunk = (size_t)chh * ((cw + 31) / 32);
                    fsm_big = std::max(fsm_big, ((pwb * (chh + 6) + 15) & ~(size_t)15) + (((size_t)(cw + 2) * (chh + 2) + 15) & ~(size_t)15) + nchunk * 4 + 64);
                }
                C.push_back(c);
            }
        }
        // orb_fast_cells<true>: one TMA box per level = its widest x tallest cell patch (3 px apron), rows a multiple of 16 bytes
        g.fbw = (max_cw + 6 + 15) & ~15; g.fbh = max_ch + 6;
        if (max_cw > 0) {
            if (g.fbw > 256 || g.fbh > 256 || (size_t)g.fbw * g.fbh > 65535) tma_ok = false;
            for (size_t ci = first_cell; ci < C.size(); ++ci) {
                const int cw = C[ci].x1 - C[ci].x0, chh = C[ci].y1 - C[ci].y0;
                if (C[ci].skipped || cw <= 0 || chh <= 0) continue;
                const size_t pw = (size_t)g.fbw, bitmap = (size_t)chh * fastpx::nms_words_per_row(cw) * 4;
                // 128 B of alignment slack, patch, score plane, bitmap, candidate list (one 16-bit entry per interior pixel)
                fsm_tma = std::max(fsm_tma, (size_t)128 + ((pw * g.fbh + 15) & ~(size_t)15) + (((size_t)fastpx::nms_plane_bytes(g.fbw, chh) + 15) & ~(size_t)15) + bitmap + (size_t)cw * chh * 2 + 64);
            }
        }
        // level list: every cell's survivors, at most nToRetain each (the reference's cap on the concatenation)
        g.sel_cap = 2 * g.nDesired + 4 * g.nCells + 64;
        g.sel_off = sel_off; sel_off += g.sel_cap;
        // orb_blur: at least 2 strips of at most about BLUR_TH rows, of one height: with its 6 warm-up rows a strip is a whole number
        // of turns of the kernel's 7-row ring, and at most the ROI's height (h >= 39). A tile = 32 consecutive (strip, column group)
        // items. The tile count grows with w and h, so the table sized at create time holds every smaller frame's.
        // Strip height measured on an H100 SXM (400 W), 64 frames of 640x480, kernel alone: 0.093 ms per batch at BLUR_TH = 48 (and
        // at 32), 0.096 at 64, 0.103 at 96, 0.114 at 128. Shorter strips make more, shorter warps and a shorter tail, although more
        // lane-steps go to warm-up rows: at 48, 79 % of the lane-steps produce new pixels, 10 % are warm-up rows, 6 % rows blurred
        // twice and 4 % idle lanes.
        g.tile_base = (int)T.size();
        g.blur_strips = std::max(2, (g.h + BLUR_TH - 1) / BLUR_TH);
        g.blur_th = ((g.h + g.blur_strips - 1) / g.blur_strips + 12) / 7 * 7 - 6;
        for (int it = 0; it < g.blur_strips * (g.pitch / 8); it += 32) T.push_back(TileGeo{l, it / (g.pitch / 8), it % (g.pitch / 8)});
    }
    *plane_bytes = poff; *cand_total = coff; *n_cells = C.size(); *n_tiles = T.size(); *tab_total = toff;
    if (fsm > 227 * 1024) fast_big = true;
    *max_fast_smem = fast_big ? fsm_big : fsm;
    if (fast_big_out) *fast_big_out = fast_big;
    if (fast_tma_smem_out) *fast_tma_smem_out = (tma_ok && !fast_big && fsm_tma <= 227 * 1024) ? fsm_tma : 0;
    if (Lv) *Lv = L;
    if (Cv) *Cv = C;
    if (Tv) *Tv = T;
    return SE2GPU_OK;
}

// cuTensorMapEncodeTiled through the runtime's driver entry point table (the library does not link libcuda, so that it also
// loads on a box without a driver, e.g. for the symbol check of the CPU test suite)
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                                  const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
EncodeTiledFn tensor_map_encoder() {
    static EncodeTiledFn fn = [] {
        void* p = nullptr;
        cudaDriverEntryPointQueryResult q = cudaDriverEntryPointSymbolNotFound;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) != cudaSuccess || q != cudaDriverEntryPointSuccess) { cudaGetLastError(); p = nullptr; }
        return (EncodeTiledFn)p;
    }();
    return fn;
}

// The kernel choices below were measured on an H100 SXM (80 GB HBM3, 400 W power limit), 64 frames of 640x480 per step, every
// alternative bit-identical: programmatic dependent launch along the resize chain takes the pyramid from 0.169 to 0.151 ms;
// orb_fast_cells<true> (TMA box, 4-pixel items) takes 0.314 ms against 0.329 ms for the plain-load instantiation and 0.346 ms for
// a TMA kernel with 8-pixel items and per-warp candidate lists (whole step 0.72 ms against 0.74 / 0.76 ms); batched loads in
// orb_orient_describe take it from 0.1045 to 0.097 ms against one dependent load pair per loop trip. The plain-load
// instantiation stays for geometries whose cell patch exceeds a 256 x 256 TMA box and for drivers without the tensor-map encoder.
// Blur schedule (run_device): one event behind the last resize forks the blur onto the side stream as two back-to-back launches,
// group A = levels [0, BLUR_SPLIT), then the rest; the main stream joins before the descriptors. Measured on an H100 SXM
// (700 W), 64 frames of 640x480, ms per step with the two-launch selection (A fork / B fork; P = right behind level
// BLUR_SPLIT-1, L = behind the last resize, F = behind the FAST launch):
//   split 1: P/L 0.5633, P/F 0.5607-0.5646, L/F 0.5546-0.5583, L/L 0.5544-0.5584      split 2: P/L 0.5650, L/F 0.5545, L/L 0.5545
//   split 3: P/L 0.5663                             one launch of every level behind the last resize: 0.5672
// Blurring level 0 next to the resize chain lengthens the pyramid (0.132 -> 0.158 ms span) by more than it hides, and a
// fork behind FAST leaves the blur later than the selection, now that the selection is short. The event between the last
// resize and FAST does not keep FAST from starting before the resize ends (tools/orb_pyramid_trace.py: -3.7 us).
constexpr int BLUR_SPLIT = 1;
// host-buffer pipeline shape (orb_enqueue): se2gpu_orb_extract splits a batch into PIPE_CHUNKS chunks round-robin over all
// pipeline lanes, the first PIPE_FIRST_PCT percent of an even share so that less of the initial H2D copy is exposed;
// se2gpu_orb_submit already overlaps a batch with its twin's, so chunking a submitted batch would only add launches
constexpr int PIPE_CHUNKS = 4, PIPE_FIRST_PCT = 50, SUBMIT_CHUNKS = 1;

// one 3-D u8 tensor per level over the batch of bordered planes: x = byte in the row (pitch), y = row, z = frame
bool encode_fast_maps(se2gpu_orb* h, size_t frame_plane_bytes) {
    EncodeTiledFn enc = tensor_map_encoder();
    if (!enc || (frame_plane_bytes & 15)) return false;
    for (int l = 0; l < h->nlevels; ++l) {
        const LevelGeo& g = h->levels[l];
        if (g.fbw <= 6) { memset(&h->fast_maps.m[l], 0, sizeof(CUtensorMap)); continue; }   // no cell on this level ever launches a copy
        const cuuint64_t gdim[3] = {(cuuint64_t)g.pitch, (cuuint64_t)(g.h + 2 * EDGE), (cuuint64_t)h->max_batch};
        const cuuint64_t gstr[2] = {(cuuint64_t)g.pitch, (cuuint64_t)frame_plane_bytes};      // bytes, multiples of 16
        const cuuint32_t box[3] = {(cuuint32_t)g.fbw, (cuuint32_t)g.fbh, 1u};
        const cuuint32_t estr[3] = {1u, 1u, 1u};
        void* base = h->d.plain + g.plane_off;
        if (((uintptr_t)base & 15) || (g.pitch & 15)) return false;
        if (enc(&h->fast_maps.m[l], CU_TENSOR_MAP_DATA_TYPE_UINT8, 3, base, gdim, gstr, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) != CUDA_SUCCESS) return false;
    }
    return true;
}

int set_geometry(se2gpu_orb* h, int w, int hgt, cudaStream_t s) {
    if (w == h->cur_w && hgt == h->cur_h) return SE2GPU_OK;
    size_t pb, ct, nc, nt, tt, fsm, fsm_tma = 0;
    bool big = false;
    int rc = build_geometry(h, w, hgt, false, &pb, &ct, &nc, &nt, &tt, &fsm, &h->levels, &h->cells, &h->tiles, &big, &fsm_tma);
    if (rc != SE2GPU_OK) return rc;
    if (pb > h->cap_plane || ct > h->cap_cand || nc > h->cap_cells || nt > h->cap_tiles || tt > h->cap_tab)
        return fail(SE2GPU_ERR_CAPACITY, "frame %dx%d exceeds the capacity this extractor was created with (%dx%d)", w, hgt, h->max_w, h->max_h);
    if (fsm > 227 * 1024) return fail(SE2GPU_ERR_CAPACITY, "a FAST cell of a %dx%d frame needs %zu B of shared memory", w, hgt, fsm);
    // resize tables [upstream OpenCV resize.cpp: fixed-point bilinear coefficient tables]
    std::vector<int> itab(tt, 0);
    std::vector<short> stab(2 * tt, 0);
    for (int l = 1; l < h->nlevels; ++l) {
        const LevelGeo& g = h->levels[l];
        const LevelGeo& sg = h->levels[l - 1];
        const double scale_x = 1. / ((double)g.w / sg.w), scale_y = 1. / ((double)g.h / sg.h);
        int* xofs = itab.data() + g.tab_off; int* yofs = xofs + g.w;
        short* ialpha = stab.data() + 2 * (size_t)g.tab_off; short* ibeta = ialpha + 2 * g.w;
        for (int dx = 0; dx < g.w; ++dx) {
            float fx = (float)((dx + 0.5) * scale_x - 0.5);
            int sx = (int)floorf(fx);
            fx -= sx;
            if (sx < 0) { fx = 0; sx = 0; }
            if (sx >= sg.w - 1) { fx = 0; sx = sg.w - 1; }
            xofs[dx] = sx;
            ialpha[2 * dx] = (short)std::min(std::max(cv_round_f((1.f - fx) * 2048.f), -32768), 32767);
            ialpha[2 * dx + 1] = (short)std::min(std::max(cv_round_f(fx * 2048.f), -32768), 32767);
        }
        for (int dy = 0; dy < g.h; ++dy) {
            float fy = (float)((dy + 0.5) * scale_y - 0.5);
            int sy = (int)floorf(fy);
            fy -= sy;
            yofs[dy] = sy;
            ibeta[2 * dy] = (short)cv_round_f((1.f - fy) * 2048.f);
            ibeta[2 * dy + 1] = (short)cv_round_f(fy * 2048.f);
        }
    }
    SE2_CUDA(cudaMemcpyAsync(h->d_levels, h->levels.data(), sizeof(LevelGeo) * h->levels.size(), cudaMemcpyHostToDevice, s));
    SE2_CUDA(cudaMemcpyAsync(h->d_cells, h->cells.data(), sizeof(CellGeo) * h->cells.size(), cudaMemcpyHostToDevice, s));
    SE2_CUDA(cudaMemcpyAsync(h->d_tiles, h->tiles.data(), sizeof(TileGeo) * h->tiles.size(), cudaMemcpyHostToDevice, s));
    SE2_CUDA(cudaMemcpyAsync(h->d_itab, itab.data(), sizeof(int) * itab.size(), cudaMemcpyHostToDevice, s));
    SE2_CUDA(cudaMemcpyAsync(h->d_stab, stab.data(), sizeof(short) * stab.size(), cudaMemcpyHostToDevice, s));
    SE2_CUDA(cudaStreamSynchronize(s));
    h->fast_smem = fsm; h->fast_big = big;
    {   // consecutive pyramid levels differ by mvScaleFactor[1] up to rounding of the level sizes
        double ratio = 1.0;
        for (size_t l = 1; l < h->levels.size(); ++l)
            ratio = std::max(ratio, std::max((double)h->levels[l - 1].w / h->levels[l].w, (double)h->levels[l - 1].h / h->levels[l].h));
        h->resize_rows = (int)ceil(RESIZE_TR * ratio) + 4;
        h->resize_raw_pitch = (((int)ceil(128 * ratio) + 4 + 15 + 15) / 16) * 16;
        h->resize_w_smem = (size_t)h->resize_rows * (128 * sizeof(uint16_t) + h->resize_raw_pitch) + 16;   // 16-bit row-pass results, 16 B of slack behind the last staged row
        if (h->resize_w_smem > 200 * 1024) return fail(SE2GPU_ERR_CAPACITY, "scale factor %.3f needs %zu B of shared memory in orb_resize_w", ratio, h->resize_w_smem);
        SE2_CUDA(cudaFuncSetAttribute(orb_resize_w<RESIZE_TR>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)h->resize_w_smem));
        h->resize_tall_rows = (int)ceil(RESIZE_TR_TALL * ratio) + 4;
        h->resize_tall_smem = (size_t)h->resize_tall_rows * (128 * sizeof(uint16_t) + h->resize_raw_pitch) + 16;
        h->resize_tall_ctas = 0;
        if (h->resize_tall_smem <= 200 * 1024) {     // else every level keeps RESIZE_TR-row tiles
            SE2_CUDA(cudaFuncSetAttribute(orb_resize_w<RESIZE_TR_TALL>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)h->resize_tall_smem));
            int per_sm = 0, sms = 0;
            SE2_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, orb_resize_w<RESIZE_TR_TALL>, 256, h->resize_tall_smem));
            SE2_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, h->device));
            h->resize_tall_ctas = per_sm * sms;
        }
    }
    SE2_CUDA(cudaFuncSetAttribute(orb_fast_cells_big, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)std::max<size_t>(fsm, 1024)));
    SE2_CUDA(cudaFuncSetAttribute(orb_fast_cells<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)std::max<size_t>(fsm, 1024)));
    // TMA-staged cells when every level's patch fits a box and the driver hands out the tensor-map encoder
    h->fast_tma = fsm_tma > 0 && encode_fast_maps(h, pb);
    h->fast_tma_smem = fsm_tma;
    if (h->fast_tma) SE2_CUDA(cudaFuncSetAttribute(orb_fast_cells<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)std::max<size_t>(fsm_tma, 1024)));
    int max_cells = 0, sel_total = 0, max_sel_cap = 0, max_cand = 0;
    for (const LevelGeo& g : h->levels) { max_cells = std::max(max_cells, g.nCells); max_sel_cap = std::max(max_sel_cap, g.sel_cap); sel_total += g.sel_cap; }
    for (const CellGeo& c : h->cells) max_cand = std::max(max_cand, c.skipped ? 0 : c.cand_cap);
    const int rec = h->harris ? 8 : 4;
    const int stage_n = std::min((max_cand + 31) & ~31, SEL_STAGE_BYTES / rec);
    const size_t ssm = (size_t)SEL_WARPS * ((size_t)stage_n * rec + 2 * 4 * (size_t)max_cells);
    if ((size_t)sel_total > h->cap_sel) return fail(SE2GPU_ERR_CAPACITY, "frame %dx%d exceeds the selection capacity this extractor was created with", w, hgt);
    const size_t lsm = (size_t)max_sel_cap * (h->harris ? 8 : 4);
    if (ssm > 227 * 1024 || lsm > 227 * 1024) return fail(SE2GPU_ERR_CAPACITY, "the selection of a %dx%d frame needs %zu / %zu B of shared memory", w, hgt, ssm, lsm);
    if (h->harris) {
        SE2_CUDA(cudaFuncSetAttribute(orb_select_cells<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)ssm));
        SE2_CUDA(cudaFuncSetAttribute(orb_select_levels<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)lsm));
    } else {
        SE2_CUDA(cudaFuncSetAttribute(orb_select_cells<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)ssm));
        SE2_CUDA(cudaFuncSetAttribute(orb_select_levels<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)lsm));
    }
    h->select_smem = ssm; h->select_levels_smem = lsm; h->sel_max_cells = max_cells; h->sel_stage_n = stage_n;
    OrbDev& d = h->d;
    d.sel_total = sel_total;
    d.n_cells = (int)h->cells.size(); d.n_tiles = (int)h->tiles.size();
    d.frame_plane_bytes = pb; d.cand_total = ct;
    int lk = 0; for (auto& g : h->levels) lk += g.kp_cap;
    d.lkp_total = lk;
    h->cur_w = w; h->cur_h = hgt;
    return SE2GPU_OK;
}

// cv::undistort's map for a w x h frame [upstream OpenCV imgproc/undistort]: stripes of max(1, 4096/w) rows, for the stripe at
// row y0 the new camera matrix is A with cy - y0; ir = its LU inverse; rays accumulated column by column in double;
// radial/tangential/thin-prism model; CV_16SC2 + CV_16UC1 fixed point with 5 fraction bits (cvRound(u*32)).
int build_undistort_map(const float* K, const float* dist, int nd, int w, int hgt, std::vector<short2>& m1, std::vector<uint16_t>& m2) {
    double A[9], D[14] = {0};
    for (int i = 0; i < 9; ++i) A[i] = K[i];
    for (int i = 0; i < nd; ++i) D[i] = dist[i];
    m1.resize((size_t)w * hgt); m2.resize((size_t)w * hgt);
    const int stripe = std::min(std::max(1, 4096 / std::max(w, 1)), hgt);
    for (int y0 = 0; y0 < hgt; y0 += stripe) {
        double M[9], inv[9] = {1, 0, 0, 0, 1, 0, 0, 0, 1};
        for (int i = 0; i < 9; ++i) M[i] = A[i];
        M[5] = A[5] - y0;
        for (int c = 0; c < 3; ++c) {                 // LU with partial pivoting, identity carried as right-hand side
            int piv = c;
            for (int r = c + 1; r < 3; ++r) if (std::fabs(M[r * 3 + c]) > std::fabs(M[piv * 3 + c])) piv = r;
            if (std::fabs(M[piv * 3 + c]) < 2.220446049250313e-14) return fail(SE2GPU_ERR_INVALID, "singular camera matrix");
            if (piv != c) for (int q = 0; q < 3; ++q) { std::swap(M[c * 3 + q], M[piv * 3 + q]); std::swap(inv[c * 3 + q], inv[piv * 3 + q]); }
            const double dneg = -1 / M[c * 3 + c];
            for (int r = c + 1; r < 3; ++r) {
                const double al = M[r * 3 + c] * dneg;
                for (int q = c + 1; q < 3; ++q) M[r * 3 + q] += al * M[c * 3 + q];
                for (int q = 0; q < 3; ++q) inv[r * 3 + q] += al * inv[c * 3 + q];
            }
        }
        for (int r = 2; r >= 0; --r)
            for (int q = 0; q < 3; ++q) {
                double acc = inv[r * 3 + q];
                for (int t = r + 1; t < 3; ++t) acc -= M[r * 3 + t] * inv[t * 3 + q];
                inv[r * 3 + q] = acc / M[r * 3 + r];
            }
        const int rows = std::min(stripe, hgt - y0);
        for (int i = 0; i < rows; ++i) {
            double X = i * inv[1] + inv[2], Y = i * inv[4] + inv[5], Wc = i * inv[7] + inv[8];
            short2* o1 = m1.data() + (size_t)(y0 + i) * w;
            uint16_t* o2 = m2.data() + (size_t)(y0 + i) * w;
            for (int jx = 0; jx < w; ++jx, X += inv[0], Y += inv[3], Wc += inv[6]) {
                const double iw = 1. / Wc, x = X * iw, y = Y * iw;
                const double x2 = x * x, y2 = y * y, r2 = x2 + y2, xy2 = 2 * x * y;
                const double kr = (1 + ((D[4] * r2 + D[1]) * r2 + D[0]) * r2) / (1 + ((D[7] * r2 + D[6]) * r2 + D[5]) * r2);
                const double xd = (x * kr + D[2] * xy2 + D[3] * (r2 + 2 * x2) + D[8] * r2 + D[9] * r2 * r2);
                const double yd = (y * kr + D[2] * (r2 + 2 * y2) + D[3] * xy2 + D[10] * r2 + D[11] * r2 * r2);
                const double su = (A[0] * xd + A[2]) * 32, sv = (A[4] * yd + A[5]) * 32;
                const int iu = su >= 2147483647.0 ? 2147483647 : su <= -2147483648.0 ? (int)-2147483648LL : (int)lrint(su);
                const int iv = sv >= 2147483647.0 ? 2147483647 : sv <= -2147483648.0 ? (int)-2147483648LL : (int)lrint(sv);
                o1[jx] = make_short2((short)(iu >> 5), (short)(iv >> 5));
                o2[jx] = (uint16_t)((iv & 31) * 32 + (iu & 31));
            }
        }
    }
    return SE2GPU_OK;
}

int ensure_undistort_map(se2gpu_orb* h, int w, int hgt, cudaStream_t s) {
    if (h->und_w == w && h->und_h == hgt) return SE2GPU_OK;
    std::vector<short2> m1; std::vector<uint16_t> m2;
    int rc = build_undistort_map(h->und_K, h->und_D, h->und_nd, w, hgt, m1, m2);
    if (rc != SE2GPU_OK) return rc;
    const size_t px = (size_t)w * hgt;
    if (px > h->und_cap) {
        if (h->d_und_m1) cudaFree(h->d_und_m1);
        if (h->d_und_m2) cudaFree(h->d_und_m2);
        h->d_und_m1 = nullptr; h->d_und_m2 = nullptr; h->und_cap = 0;
        SE2_CUDA(cudaMalloc((void**)&h->d_und_m1, px * sizeof(short2)));
        SE2_CUDA(cudaMalloc((void**)&h->d_und_m2, px * sizeof(uint16_t)));
        h->und_cap = px;
    }
    SE2_CUDA(cudaMemcpyAsync(h->d_und_m1, m1.data(), px * sizeof(short2), cudaMemcpyHostToDevice, s));
    SE2_CUDA(cudaMemcpyAsync(h->d_und_m2, m2.data(), px * sizeof(uint16_t), cudaMemcpyHostToDevice, s));
    SE2_CUDA(cudaStreamSynchronize(s));      // the host vectors go out of scope
    h->und_w = w; h->und_h = hgt;
    return SE2GPU_OK;
}

// a launch that may begin while its predecessor in the stream drains (programmatic dependent launch): the kernel reads what
// its predecessor wrote only behind griddepcontrol.wait, which returns once that grid has completed and its writes are visible
template <typename... KArgs, typename... Args>
cudaError_t launch_pdl(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t s, Args... args) {
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = grid; cfg.blockDim = block; cfg.dynamicSmemBytes = smem; cfg.stream = s;
    cudaLaunchAttribute at[1];
    at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    at[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = at; cfg.numAttrs = 1;
    ::se2gpu::g_launches.fetch_add(1, std::memory_order_relaxed);
    return cudaLaunchKernelEx(&cfg, kernel, args...);
}

int run_device(se2gpu_orb* h, const uint8_t* d_imgs, int n, int w, int hgt, int stride, size_t frame_stride,
               se2gpu_keypoint* d_kps, uint8_t* d_desc, int* d_counts, cudaStream_t s, int frame0 = 0, int lane = -1) {
    int rc = set_geometry(h, w, hgt, s);
    if (rc != SE2GPU_OK) return rc;
    if (h->und_on && (rc = ensure_undistort_map(h, w, hgt, s)) != SE2GPU_OK) return rc;
    OrbDev d = h->d;             // by-value copy carrying this launch group's frame offset
    d.frame0 = frame0;
    // pipeline lanes get their concurrency from each other, not from a blur side stream
    cudaStream_t side = lane < 0 ? h->side : nullptr;
    cudaEvent_t ev_pyr = h->ev_pyr, ev_blur = h->ev_blur;
    se2gpu::Profiler& pr = h->prof;
    SE2_NVTX("se2gpu.orb.run_device");
    nvtxRangePushA("se2gpu.orb.pyramid");
    pr.begin(0, s);
    {
        const LevelGeo& g = h->levels[0];
        if (h->und_on) {
            dim3 grid((g.pitch / 4 + 127) / 128, g.h + 2 * EDGE, n);
            SE2_LAUNCH(orb_pyr0_undistort, grid, 128, 0, s, d, g, d_imgs, stride, frame_stride, h->d_und_m1, h->d_und_m2);
        } else {
            const int aligned = (((uintptr_t)d_imgs | (uintptr_t)stride | (uintptr_t)frame_stride) & 15) == 0;
            const int nvec = aligned ? g.w / 16 : 0;      // aligned 16-byte interior vectors per row
            dim3 grid((nvec + 63) / 64 + 1, (g.h + 2 * EDGE + 4 * PYR0_ROWS - 1) / (4 * PYR0_ROWS), n);
            SE2_LAUNCH(orb_pyr0, grid, dim3(64, 4), 0, s, d, g, d_imgs, stride, frame_stride, nvec);
        }
    }
    const bool overlap = !pr.on && side != nullptr;
    for (int l = 1; l < h->nlevels; ++l) {
        const LevelGeo& g = h->levels[l];
        cudaLaunchConfig_t cfg = {};
        // tall tiles where their grid fills every resident CTA slot at least once (see RESIZE_TR_TALL)
        const int ncx = (g.pitch + 127) / 128, H = g.h + 2 * EDGE;
        const int tall_grid = ncx * ((H + RESIZE_TR_TALL - 1) / RESIZE_TR_TALL) * n;
        const bool tall = h->resize_tall_ctas > 0 && tall_grid >= h->resize_tall_ctas;
        const int tr = tall ? RESIZE_TR_TALL : RESIZE_TR;
        cfg.gridDim = dim3(ncx, (H + tr - 1) / tr, n);
        cfg.blockDim = dim3(32, 8); cfg.dynamicSmemBytes = tall ? h->resize_tall_smem : h->resize_w_smem; cfg.stream = s;
        cudaLaunchAttribute at[1];   // programmatic dependent launch along the resize chain (see orb_resize_w)
        at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
        at[0].val.programmaticStreamSerializationAllowed = 1;
        cfg.attrs = at; cfg.numAttrs = 1;
        if (tall) SE2_CUDA(cudaLaunchKernelEx(&cfg, orb_resize_w<RESIZE_TR_TALL>, d, g, h->levels[l - 1], h->resize_tall_rows, h->resize_raw_pitch));
        else SE2_CUDA(cudaLaunchKernelEx(&cfg, orb_resize_w<RESIZE_TR>, d, g, h->levels[l - 1], h->resize_rows, h->resize_raw_pitch));
        ::se2gpu::g_launches.fetch_add(1, std::memory_order_relaxed);
    }
    // the blur is forked here, behind the whole pyramid (see BLUR_SPLIT); with the profiler on everything stays on one stream
    // so that the per-kernel event times are not polluted by the overlap
    if (overlap) SE2_CUDA(cudaEventRecord(ev_pyr, s));
    pr.end(s);
    nvtxRangePop();
    auto launch_blur = [&](cudaStream_t st, int t0, int t1) {
        if (t1 > t0) SE2_LAUNCH(orb_blur, dim3((t1 - t0 + BLUR_WARPS - 1) / BLUR_WARPS, n), BLUR_WARPS * 32, 0, st, d, t0, t1);
    };
    const int split = std::min(BLUR_SPLIT, h->nlevels);
    const int tilesA = split < h->nlevels ? h->levels[split].tile_base : d.n_tiles;
    if (overlap) {
        SE2_CUDA(cudaStreamWaitEvent(side, ev_pyr, 0));
        launch_blur(side, 0, tilesA);
        launch_blur(side, tilesA, d.n_tiles);
        SE2_CUDA(cudaEventRecord(ev_blur, side));
    }
    SE2_NVTX("se2gpu.orb.fast_select_blur_describe");
    pr.begin(1, s);
    // FAST is a programmatic dependent of the last resize; orb_fast_cells_big, for cells too large for it, keeps a plain launch
    if (h->fast_big) SE2_LAUNCH(orb_fast_cells_big, dim3(d.n_cells, n), FAST_THREADS, h->fast_smem, s, d);
    else if (h->fast_tma) SE2_CUDA(launch_pdl(orb_fast_cells<true>, dim3(d.n_cells, n), FAST_THREADS, h->fast_tma_smem, s, d, h->fast_maps));
    else SE2_CUDA(launch_pdl(orb_fast_cells<false>, dim3(d.n_cells, n), FAST_THREADS, h->fast_smem, s, d, h->fast_maps));
    if (h->harris) SE2_LAUNCH(orb_harris, dim3(d.n_cells, n), HARRIS_THREADS, 0, s, d, h->hb.cand64);   // timed with FAST (group 1)
    pr.end(s);
    pr.begin(2, s);
    // frames vary fastest in the CTA order: the CTAs of every frame's first cells (level 0) are dispatched together, first
    const dim3 sel_grid(n, (d.n_cells + SEL_WARPS - 1) / SEL_WARPS);
    if (h->harris) {
        SE2_CUDA(launch_pdl(orb_select_cells<true>, sel_grid, SEL_WARPS * 32, h->select_smem, s, d, h->hb, h->sel_max_cells, h->sel_stage_n));
        SE2_CUDA(launch_pdl(orb_select_levels<true>, dim3(h->nlevels, n), 32, h->select_levels_smem, s, d, h->hb));
    } else {
        SE2_CUDA(launch_pdl(orb_select_cells<false>, sel_grid, SEL_WARPS * 32, h->select_smem, s, d, h->hb, h->sel_max_cells, h->sel_stage_n));
        SE2_CUDA(launch_pdl(orb_select_levels<false>, dim3(h->nlevels, n), 32, h->select_levels_smem, s, d, h->hb));
    }
    pr.end(s);
    if (overlap) {
        SE2_CUDA(cudaStreamWaitEvent(s, ev_blur, 0));
    } else {
        pr.begin(3, s);
        launch_blur(s, 0, d.n_tiles);
        pr.end(s);
    }
    const int warps = 8;
    const dim3 desc_grid((h->nfeatures + warps - 1) / warps, n);
    pr.begin(4, s);
    if (h->harris) SE2_CUDA(launch_pdl(orb_orient_describe<true>, desc_grid, warps * 32, 0, s, d, d_kps, d_desc, d_counts, (const float*)h->hb.lresp));
    else SE2_CUDA(launch_pdl(orb_orient_describe<false>, desc_grid, warps * 32, 0, s, d, d_kps, d_desc, d_counts, (const float*)h->hb.lresp));
    pr.end(s);
    h->last_n = std::max(h->last_n * (frame0 > 0), frame0 + n);
    return SE2GPU_OK;
}

}  // namespace

int se2gpu::orb_prepare_shape(se2gpu_orb* h, int w, int hgt, cudaStream_t s) {
    SE2_CUDA(cudaSetDevice(h->device));
    int rc = set_geometry(h, w, hgt, s);
    if (rc == SE2GPU_OK && h->und_on) rc = ensure_undistort_map(h, w, hgt, s);
    return rc;
}

extern "C" {

se2gpu_orb* se2gpu_orb_create_scored(int nfeatures, float scale_factor, int nlevels, int score_type, int fast_th, int max_w, int max_h,
                                     int max_batch, int device) {
    if (score_type != SE2GPU_ORB_HARRIS_SCORE && score_type != SE2GPU_ORB_FAST_SCORE) {
        fail(SE2GPU_ERR_INVALID, "unknown ORB score type %d (HARRIS_SCORE = 0, FAST_SCORE = 1)", score_type); return nullptr;
    }
    if (nfeatures <= 0 || nlevels <= 0 || nlevels > MAX_LEVELS || !(scale_factor > 1.0f) || fast_th < 1 || fast_th > 254 ||
        max_w <= 0 || max_h <= 0 || max_batch <= 0) { fail(SE2GPU_ERR_INVALID, "bad ORB parameters"); return nullptr; }
    if (se2gpu::select_device(device) != SE2GPU_OK) return nullptr;
    se2gpu_orb* h = new se2gpu_orb;
    h->device = device; h->nfeatures = nfeatures; h->nlevels = nlevels; h->fast_th = fast_th;
    h->harris = score_type == SE2GPU_ORB_HARRIS_SCORE;
    h->max_w = max_w; h->max_h = max_h; h->max_batch = max_batch;
    { int* a = h->create_args; a[0] = nfeatures; memcpy(&a[1], &scale_factor, sizeof(float)); a[2] = nlevels; a[3] = fast_th; a[4] = max_w; a[5] = max_h; a[6] = max_batch; a[7] = device; a[8] = score_type; }
    h->scaleFactor = scale_factor;   // the reference keeps it in a double member (ORBextractor.h:67)
    // ORBextractor::ORBextractor, ORBextractor.cpp:463-520
    h->mvScaleFactor.resize(nlevels); h->mvInvScaleFactor.resize(nlevels); h->mnFeaturesPerLevel.resize(nlevels);
    h->mvScaleFactor[0] = 1;
    for (int i = 1; i < nlevels; i++) h->mvScaleFactor[i] = (float)(h->mvScaleFactor[i - 1] * h->scaleFactor);
    const float invScaleFactor = (float)(1.0f / h->scaleFactor);
    h->mvInvScaleFactor[0] = 1;
    for (int i = 1; i < nlevels; i++) h->mvInvScaleFactor[i] = h->mvInvScaleFactor[i - 1] * invScaleFactor;
    const float factor = (float)(1.0 / h->scaleFactor);
    float nDesired = nfeatures * (1 - factor) / (1 - (float)pow((double)factor, (double)nlevels));
    int sum = 0;
    for (int l = 0; l < nlevels - 1; l++) { h->mnFeaturesPerLevel[l] = cv_round_f(nDesired); sum += h->mnFeaturesPerLevel[l]; nDesired *= factor; }
    h->mnFeaturesPerLevel[nlevels - 1] = std::max(nfeatures - sum, 0);
    if (sum > nfeatures) { fail(SE2GPU_ERR_INVALID, "per-level quotas sum to %d > nfeatures %d for these parameters", sum, nfeatures); delete h; return nullptr; }
    int umax[16];
    {
        int v, v0, vmax = (int)floorf(HALF_PATCH * sqrtf(2.f) / 2 + 1), vmin = (int)ceilf(HALF_PATCH * sqrtf(2.f) / 2);
        const double hp2 = HALF_PATCH * HALF_PATCH;
        for (v = 0; v <= vmax; ++v) umax[v] = (int)lrint(sqrt(hp2 - v * v));
        for (v = HALF_PATCH, v0 = 0; v >= vmin; --v) { while (umax[v0] == umax[v0 + 1]) ++v0; umax[v] = v0; ++v0; }
    }
    float gk[7];
    { double g[7], s = 0; for (int i = 0; i < 7; ++i) { double x = i - 3; g[i] = std::exp(-0.5 * x * x / 4.0); s += g[i]; } for (int i = 0; i < 7; ++i) gk[i] = (float)(g[i] * (1. / s)); }
    size_t pb, ct, nc, nt, tt, fsm;
    int rc = build_geometry(h, max_w, max_h, true, &pb, &ct, &nc, &nt, &tt, &fsm, nullptr, nullptr, nullptr);
    if (rc != SE2GPU_OK) { delete h; return nullptr; }
    // head-room so that smaller frames (different cell rounding) always fit
    h->cap_plane = pb + 4096; h->cap_cand = ct + ct / 8 + 4096; h->cap_cells = nc + 64; h->cap_tiles = nt + 64; h->cap_tab = tt + 64;
    h->cap_lkp = nfeatures + 64;
    h->cap_sel = 2 * (size_t)nfeatures + 4 * h->cap_cells + 64 * (size_t)nlevels;   // the level lists' sel_cap summed over levels
    const size_t B = max_batch;
    bool ok = true;
    auto A = [&](auto** p, size_t c) { ok = ok && h->bufs.alloc(p, c) == cudaSuccess; };
    OrbDev& d = h->d;
    A(&h->d_levels, (size_t)nlevels); A(&h->d_cells, h->cap_cells); A(&h->d_tiles, h->cap_tiles); A(&h->d_itab, h->cap_tab); A(&h->d_stab, 2 * h->cap_tab);
    A(&d.plain, B * h->cap_plane); A(&d.blurred, B * h->cap_plane);
    A(&d.cand, B * h->cap_cand); A(&d.hdr, B * h->cap_cells); A(&d.lkp, B * h->cap_lkp); A(&d.lcount, B * nlevels); A(&d.sel, B * h->cap_sel); A(&d.err, 1);
    A(&h->d_in, B * (size_t)max_w * max_h); A(&h->d_kps, B * nfeatures); A(&h->d_desc, B * nfeatures * 32); A(&h->d_counts, B);
    if (h->harris) { A(&h->hb.cand64, B * h->cap_cand); A(&h->hb.lresp, B * h->cap_lkp); }
    if (!ok) { fail(SE2GPU_ERR_CUDA, "device allocation failed (%s)", cudaGetErrorString(cudaGetLastError())); se2gpu_orb_destroy(h); return nullptr; }
    cudaMemset(d.err, 0, sizeof(int));
    if (cudaStreamCreateWithFlags(&h->side, cudaStreamNonBlocking) != cudaSuccess || cudaEventCreateWithFlags(&h->ev_pyr, cudaEventDisableTiming) != cudaSuccess ||
        cudaEventCreateWithFlags(&h->ev_blur, cudaEventDisableTiming) != cudaSuccess) { h->side = nullptr; cudaGetLastError(); }
    for (int l = 0; l < ORB_LANES && h->side; ++l)
        if (cudaStreamCreateWithFlags(&h->pipe[l], cudaStreamNonBlocking) != cudaSuccess) { h->pipe[l] = nullptr; cudaGetLastError(); break; }
    cudaMemcpyToSymbol(c_umax, umax, sizeof umax);
    {
        int vmax[16];
        for (int u = 0; u <= HALF_PATCH; ++u) { vmax[u] = 0; for (int v = 0; v <= HALF_PATCH; ++v) if (umax[v] >= u) vmax[u] = v; }
        cudaMemcpyToSymbol(c_vmax, vmax, sizeof vmax);
    }
    cudaMemcpyToSymbol(c_gauss, gk, sizeof gk);
    d.nlevels = nlevels; d.nfeatures = nfeatures; d.fast_th = fast_th; d.t_lo = std::min(fast_th, 7);
    d.levels = h->d_levels; d.cells = h->d_cells; d.tiles = h->d_tiles; d.itab = h->d_itab; d.stab = h->d_stab;
    if (cudaDeviceSynchronize() != cudaSuccess) { fail(SE2GPU_ERR_CUDA, "init failed"); se2gpu_orb_destroy(h); return nullptr; }
    return h;
}

se2gpu_orb* se2gpu_orb_create(int nfeatures, float scale_factor, int nlevels, int fast_th, int max_w, int max_h,
                              int max_batch, int device) {
    return se2gpu_orb_create_scored(nfeatures, scale_factor, nlevels, SE2GPU_ORB_FAST_SCORE, fast_th, max_w, max_h, max_batch, device);
}

void se2gpu_orb_destroy(se2gpu_orb* h) {
    if (!h) return;
    if (h->twin) { se2gpu_orb_destroy(h->twin); h->twin = nullptr; }
    cudaSetDevice(h->device);
    if (h->side) cudaStreamDestroy(h->side);
    if (h->ev_pyr) cudaEventDestroy(h->ev_pyr);
    if (h->d_und_m1) cudaFree(h->d_und_m1);
    if (h->d_und_m2) cudaFree(h->d_und_m2);
    if (h->ev_blur) cudaEventDestroy(h->ev_blur);
    if (h->pin_counts) cudaFreeHost(h->pin_counts);
    if (h->pin_kps) cudaFreeHost(h->pin_kps);
    if (h->pin_desc) cudaFreeHost(h->pin_desc);
    for (int l = 0; l < ORB_LANES; ++l)
        if (h->pipe[l]) cudaStreamDestroy(h->pipe[l]);
    delete h;
}

int se2gpu_orb_extract_device(se2gpu_orb* h, const uint8_t* d_imgs, int n, int w, int hgt, int stride, size_t frame_stride,
                              se2gpu_keypoint* d_kps, uint8_t* d_desc, int* d_counts, void* stream) {
    if (!h) return fail(SE2GPU_ERR_INVALID, "null handle");
    if (n < 0 || n > h->max_batch) return fail(SE2GPU_ERR_CAPACITY, "batch %d exceeds max_batch %d", n, h->max_batch);
    SE2_CUDA(cudaSetDevice(h->device));
    cudaStream_t s = (cudaStream_t)stream;
    if (n == 0) return SE2GPU_OK;
    if (!d_imgs || w <= 0 || hgt <= 0) { SE2_CUDA(cudaMemsetAsync(d_counts, 0, sizeof(int) * n, s)); return SE2GPU_OK; }
    if (stride < w) return fail(SE2GPU_ERR_INVALID, "stride < width");
    return run_device(h, d_imgs, n, w, hgt, stride, frame_stride, d_kps, d_desc, d_counts, s);
}

// enqueue one host-buffer batch on this context (copies in, kernels, copies out); nothing is waited for
static int orb_enqueue(se2gpu_orb* h, const uint8_t* imgs, int n, int w, int hgt, int stride, size_t frame_stride,
                       se2gpu_keypoint* kps, uint8_t* desc, int* counts, bool submit_mode = false) {
    SE2_NVTX("se2gpu.orb.enqueue");
    if (!h) return fail(SE2GPU_ERR_INVALID, "null handle");
    if (h->pend.on) return fail(SE2GPU_ERR_INVALID, "a submitted batch is still pending on this context: call se2gpu_orb_wait first");
    if (n < 0 || n > h->max_batch) return fail(SE2GPU_ERR_CAPACITY, "batch %d exceeds max_batch %d", n, h->max_batch);
    if (n == 0) return SE2GPU_OK;
    if (!imgs || w <= 0 || hgt <= 0) { for (int i = 0; i < n; ++i) counts[i] = 0; return SE2GPU_OK; }   // :730-731
    if (stride < w) return fail(SE2GPU_ERR_INVALID, "stride < width");
    if (w > h->max_w || hgt > h->max_h) return fail(SE2GPU_ERR_CAPACITY, "frame %dx%d exceeds %dx%d", w, hgt, h->max_w, h->max_h);
    SE2_CUDA(cudaSetDevice(h->device));
    int rc = set_geometry(h, w, hgt, nullptr);
    if (rc != SE2GPU_OK) return rc;
    // pipeline shape (PIPE_CHUNKS): chunks round-robin over all lanes (H2D copy, kernels and D2H copies of a chunk are
    // stream-ordered; different lanes overlap); 1 chunk = one synchronous pass
    int lanes = 0;
    while (lanes < ORB_LANES && h->pipe[lanes]) ++lanes;
    const int nchunks = submit_mode ? SUBMIT_CHUNKS : PIPE_CHUNKS;
    const bool pipelined = lanes >= 2 && !h->prof.on && n > 1 && (nchunks > 1 || submit_mode);
    const int chunk = pipelined ? std::max(1, (n + nchunks - 1) / nchunks) : n;
    const int first = (pipelined && nchunks > 1) ? std::max(1, std::min(n, chunk * PIPE_FIRST_PCT / 100)) : n;
    auto is_pinned = [](const void* p) {
        cudaPointerAttributes at;
        if (cudaPointerGetAttributes(&at, p) != cudaSuccess) { cudaGetLastError(); return false; }
        return at.type == cudaMemoryTypeHost;
    };
    se2gpu_keypoint* out_kps = kps; uint8_t* out_desc = desc; int* out_counts = counts;
    if (pipelined) {
        if (!h->pin_counts && cudaMallocHost((void**)&h->pin_counts, sizeof(int) * h->max_batch) != cudaSuccess) return fail(SE2GPU_ERR_CUDA, "cudaMallocHost failed");
        out_counts = h->pin_counts;
        if (!is_pinned(kps) || !is_pinned(desc)) {
            if (!h->pin_kps && (cudaMallocHost((void**)&h->pin_kps, sizeof(se2gpu_keypoint) * (size_t)h->max_batch * h->nfeatures) != cudaSuccess ||
                                cudaMallocHost((void**)&h->pin_desc, (size_t)32 * h->max_batch * h->nfeatures) != cudaSuccess))
                return fail(SE2GPU_ERR_CUDA, "cudaMallocHost failed");
            out_kps = h->pin_kps; out_desc = h->pin_desc;
        }
    }
    int lane = 0;
    for (int f0 = 0, m = 0; f0 < n; f0 += m, lane = (lane + 1) % std::max(lanes, 1)) {
        m = std::min(f0 == 0 ? first : std::max(chunk, (n - first + nchunks - 2) / std::max(1, nchunks - 1)), n - f0);
        cudaStream_t s = pipelined ? h->pipe[lane] : nullptr;
        // pack rows tightly on the device (pitch = w); frames of different chunks use disjoint device buffers
        if (stride == w && frame_stride == (size_t)w * hgt)
            SE2_CUDA(cudaMemcpyAsync(h->d_in + (size_t)f0 * w * hgt, imgs + (size_t)f0 * frame_stride, (size_t)m * w * hgt, cudaMemcpyHostToDevice, s));
        else
            for (int i = f0; i < f0 + m; ++i)
                SE2_CUDA(cudaMemcpy2DAsync(h->d_in + (size_t)i * w * hgt, w, imgs + i * frame_stride, stride, w, hgt, cudaMemcpyHostToDevice, s));
        // a single chunk keeps the blur on the context's side stream (like the device-resident entry); several chunks overlap each other
        rc = run_device(h, h->d_in, m, w, hgt, w, (size_t)w * hgt, h->d_kps, h->d_desc, h->d_counts, s, f0, (pipelined && nchunks > 1) ? lane : -1);
        if (rc != SE2GPU_OK) return rc;
        SE2_CUDA(cudaMemcpyAsync(out_counts + f0, h->d_counts + f0, sizeof(int) * m, cudaMemcpyDeviceToHost, s));
        SE2_CUDA(cudaMemcpyAsync(out_kps + (size_t)f0 * h->nfeatures, h->d_kps + (size_t)f0 * h->nfeatures, sizeof(se2gpu_keypoint) * (size_t)m * h->nfeatures, cudaMemcpyDeviceToHost, s));
        SE2_CUDA(cudaMemcpyAsync(out_desc + (size_t)32 * f0 * h->nfeatures, h->d_desc + (size_t)32 * f0 * h->nfeatures, (size_t)32 * m * h->nfeatures, cudaMemcpyDeviceToHost, s));
    }
    h->pend.on = true; h->pend.n = n; h->pend.lanes = lanes; h->pend.pipelined = pipelined;
    h->pend.kps = kps; h->pend.desc = desc; h->pend.counts = counts; h->pend.out_kps = out_kps; h->pend.out_desc = out_desc; h->pend.out_counts = out_counts;
    return SE2GPU_OK;
}

// wait for the batch enqueued by orb_enqueue and hand the results to the caller's buffers
static int orb_finish(se2gpu_orb* h) {
    SE2_NVTX("se2gpu.orb.finish");
    if (!h->pend.on) return SE2GPU_OK;
    SE2_CUDA(cudaSetDevice(h->device));
    const se2gpu_orb::Pending p = h->pend;
    h->pend.on = false;
    if (p.pipelined) {
        for (int l = 0; l < p.lanes; ++l) SE2_CUDA(cudaStreamSynchronize(h->pipe[l]));
        memcpy(p.counts, p.out_counts, sizeof(int) * p.n);
        if (p.out_kps != p.kps) { memcpy(p.kps, p.out_kps, sizeof(se2gpu_keypoint) * (size_t)p.n * h->nfeatures); memcpy(p.desc, p.out_desc, (size_t)32 * p.n * h->nfeatures); }
    }
    int err = 0;
    SE2_CUDA(cudaMemcpyAsync(&err, h->d.err, sizeof(int), cudaMemcpyDeviceToHost, nullptr));
    SE2_CUDA(cudaStreamSynchronize(nullptr));
    h->last_n = p.n;
    if (err) {
        cudaMemset(h->d.err, 0, sizeof(int));
        if (err == 4) return fail(SE2GPU_ERR_CUDA, "the TMA copy of a FAST cell did not complete (tensor map / driver problem)");
        return fail(SE2GPU_ERR_CAPACITY, "internal candidate buffer overflow (code %d)", err);
    }
    return SE2GPU_OK;
}

int se2gpu_orb_extract(se2gpu_orb* h, const uint8_t* imgs, int n, int w, int hgt, int stride, size_t frame_stride,
                       se2gpu_keypoint* kps, uint8_t* desc, int* counts) {
    if (!h) return fail(SE2GPU_ERR_INVALID, "null handle");
    if (h->in_flight) return fail(SE2GPU_ERR_INVALID, "se2gpu_orb_extract while submitted batches are in flight: drain them with se2gpu_orb_wait");
    int rc = orb_enqueue(h, imgs, n, w, hgt, stride, frame_stride, kps, desc, counts);
    if (rc != SE2GPU_OK) return rc;
    return orb_finish(h);
}

int se2gpu_orb_submit(se2gpu_orb* h, const uint8_t* imgs, int n, int w, int hgt, int stride, size_t frame_stride,
                      se2gpu_keypoint* kps, uint8_t* desc, int* counts) {
    if (!h) return fail(SE2GPU_ERR_INVALID, "null handle");
    if (h->in_flight >= 2) return fail(SE2GPU_ERR_INVALID, "two batches are already in flight: call se2gpu_orb_wait first");
    if (!h->twin) {
        const int* a = h->create_args;
        float sf; memcpy(&sf, &a[1], sizeof sf);
        h->twin = se2gpu_orb_create_scored(a[0], sf, a[2], a[8], a[3], a[4], a[5], a[6], a[7]);
        if (!h->twin) return SE2GPU_ERR_CUDA;
        if (h->und_on && se2gpu_orb_set_undistort(h->twin, h->und_K, h->und_nd ? h->und_D : nullptr, h->und_nd) != SE2GPU_OK) return SE2GPU_ERR_CUDA;
    }
    se2gpu_orb* ctx = (h->submit_next & 1) ? h->twin : h;
    int rc = orb_enqueue(ctx, imgs, n, w, hgt, stride, frame_stride, kps, desc, counts, true);
    if (rc != SE2GPU_OK) return rc;
    if (!ctx->pend.on) {          // empty image / n == 0: finished synchronously (outputs as se2gpu_orb_extract leaves them)
        return SE2GPU_OK;
    }
    h->submit_next ^= 1; h->in_flight++;
    return SE2GPU_OK;
}

int se2gpu_orb_wait(se2gpu_orb* h) {
    if (!h) return fail(SE2GPU_ERR_INVALID, "null handle");
    if (!h->in_flight) return SE2GPU_OK;
    se2gpu_orb* ctx = (h->wait_next & 1) ? h->twin : h;
    h->wait_next ^= 1; h->in_flight--;
    return orb_finish(ctx);
}



int se2gpu_orb_debug_nth_element(uint32_t* values, const int* offsets, const int* nth, int count, int device) {
    if (count <= 0) return SE2GPU_OK;
    if (!values || !offsets || !nth) return fail(SE2GPU_ERR_INVALID, "null argument");
    se2gpu::HostStage st(device);
    if (const int rc = st.status()) return rc;
    uint32_t* dv = st.inout(values, (size_t)offsets[count]);
    const int* dofs = st.upload(offsets, (size_t)count + 1);
    const int* dn = st.upload(nth, count);
    if (const int rc = st.status()) return rc;
    SE2_LAUNCH(orb_debug_nth, (count + 3) / 4, 128, 0, nullptr, dv, dofs, dn, count);
    st.check(cudaGetLastError(), "kernel launch");
    return st.finish();
}

int se2gpu_orb_debug_nth_element_f32(const float* values, const int* offsets, const int* nth, int count, int* perm, int device) {
    if (count <= 0) return SE2GPU_OK;
    if (!values || !offsets || !nth || !perm) return fail(SE2GPU_ERR_INVALID, "null argument");
    se2gpu::HostStage st(device);
    if (const int rc = st.status()) return rc;
    const size_t total = (size_t)offsets[count];
    std::vector<uint64_t> rec(total);
    for (int k = 0; k < count; ++k)
        for (int i = offsets[k]; i < offsets[k + 1]; ++i) rec[i] = ((uint64_t)se2gpu::resp_key(values[i]) << 32) | (uint32_t)(i - offsets[k]);
    uint64_t* dv = st.inout(rec.data(), total);
    const int* dofs = st.upload(offsets, (size_t)count + 1);
    const int* dn = st.upload(nth, count);
    if (const int rc = st.status()) return rc;
    SE2_LAUNCH(orb_debug_nth64, (count + 3) / 4, 128, 0, nullptr, dv, dofs, dn, count);
    st.check(cudaGetLastError(), "kernel launch");
    if (const int rc = st.finish()) return rc;
    for (size_t i = 0; i < total; ++i) perm[i] = (int)(uint32_t)rec[i];
    return SE2GPU_OK;
}

int se2gpu_orb_set_undistort(se2gpu_orb* h, const float* K, const float* dist, int ndist) {
    if (!h) return fail(SE2GPU_ERR_INVALID, "null handle");
    if (!K) { h->und_on = false; return SE2GPU_OK; }
    if (ndist != 0 && ndist != 4 && ndist != 5 && ndist != 8 && ndist != 12 && ndist != 14) return fail(SE2GPU_ERR_INVALID, "distortion vector must have 0, 4, 5, 8, 12 or 14 coefficients");
    if (ndist > 0 && !dist) return fail(SE2GPU_ERR_INVALID, "null distortion vector");
    if (ndist == 14 && (dist[12] != 0.f || dist[13] != 0.f)) return fail(SE2GPU_ERR_INVALID, "tilted-sensor coefficients (tauX, tauY) are not supported");
    memcpy(h->und_K, K, sizeof h->und_K);
    memset(h->und_D, 0, sizeof h->und_D);
    if (ndist > 0) memcpy(h->und_D, dist, sizeof(float) * ndist);
    h->und_nd = ndist; h->und_w = h->und_h = 0; h->und_on = true;
    return SE2GPU_OK;
}

int se2gpu_orb_debug_undistort_map(const float* K, const float* dist, int ndist, int w, int hgt, int16_t* m1, uint16_t* m2) {
    if (!K || !m1 || !m2 || w <= 0 || hgt <= 0 || ndist < 0 || ndist > 14 || (ndist > 0 && !dist)) return fail(SE2GPU_ERR_INVALID, "bad argument");
    std::vector<short2> a; std::vector<uint16_t> b;
    int rc = build_undistort_map(K, dist, ndist, w, hgt, a, b);
    if (rc != SE2GPU_OK) return rc;
    memcpy(m1, a.data(), a.size() * sizeof(short2));
    memcpy(m2, b.data(), b.size() * sizeof(uint16_t));
    return SE2GPU_OK;
}

int se2gpu_orb_profile(se2gpu_orb* h, int enable) {
    if (!h) return fail(SE2GPU_ERR_INVALID, "null handle");
    SE2_CUDA(cudaSetDevice(h->device));
    h->prof.enable(enable != 0);
    return SE2GPU_OK;
}

int se2gpu_orb_profile_read(se2gpu_orb* h, double* ms, int* launches) {
    if (!h) return fail(SE2GPU_ERR_INVALID, "null handle");
    SE2_CUDA(cudaSetDevice(h->device));
    h->prof.flush();
    for (int g = 0; g < SE2GPU_ORB_PROFILE_GROUPS; ++g) { if (ms) ms[g] = h->prof.ms[g]; if (launches) launches[g] = h->prof.launches[g]; }
    return SE2GPU_OK;
}

int se2gpu_orb_level_dims(se2gpu_orb* h, int level, int* w, int* hgt, int* pitch) {
    if (!h || level < 0 || level >= h->nlevels || h->cur_w < 0) return fail(SE2GPU_ERR_INVALID, "no geometry");
    *w = h->levels[level].w; *hgt = h->levels[level].h; *pitch = h->levels[level].pitch;
    return SE2GPU_OK;
}

int se2gpu_orb_get_level(se2gpu_orb* h, int frame, int level, int blurred, uint8_t* out) {
    if (!h || level < 0 || level >= h->nlevels || h->cur_w < 0 || frame < 0 || frame >= h->last_n) return fail(SE2GPU_ERR_INVALID, "bad frame/level");
    SE2_CUDA(cudaSetDevice(h->device));
    const LevelGeo& g = h->levels[level];
    const uint8_t* src = (blurred ? h->d.blurred : h->d.plain) + (size_t)frame * h->d.frame_plane_bytes + g.plane_off;
    SE2_CUDA(cudaMemcpy(out, src, (size_t)g.pitch * (g.h + 2 * EDGE), cudaMemcpyDeviceToHost));
    return SE2GPU_OK;
}

}  // extern "C"
