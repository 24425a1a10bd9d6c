// Local BA: what the kernels (ba.cu) and the loader (ba_loader.cu) share - the constants both sides size things by, the
// kernel parameter structs, and the context behind the opaque se2gpu_ba handle. Internal to libse2gpu.
#pragma once
#include <algorithm>
#include <vector>

#include "common.h"
#include "ba_band.h"

namespace se2ba {

constexpr int EB = 12;             // doubles per edge record (9 used + padding to 96 B = 3 L2 sectors)
constexpr int LM_THREADS = 128;   // threads per block in per-landmark kernels
constexpr int SMEM_CHOL_MAX_N = 156;  // ldlt_smem_bytes(n) <= 227 KB, n a multiple of 3
constexpr int TW_MAX_W = 16;       // separator blocks of the two-sided reduced solve
constexpr int PK_THREADS = 512;    // threads per CTA of the persistent kernel
constexpr int PK_MAXOWN = 16;      // blocks of S a worker CTA of the persistent kernel caches in shared memory
constexpr int PK_RED_SCRATCH_BYTES = (PK_THREADS / 32) * 21 * 33 * 8;   // per-warp reduction scratch at the top of a worker's arena

struct Cam {
    double fx, cx, cy, Rcb[9], tcb[3], delta;
};

struct LMState {  // device-resident scalars of the LM loop (host mirrors it once per trial)
    double lambda, ni, chi_cur, chi_before, chi_trial, scale, rho, max_diag;
    int cur, solve_ok, accepted, trials, terminate, retry, iter, stop_all;   // stop_all: abort flag, OR-ed over the ranks of a sharded run
    long long epoch;   // sharded persistent kernel: last exchange epoch used (continues across optimize() calls)
    int error, pad;    // 1: a peer did not show up within the exchange timeout
};

struct Dev {  // all device pointers of one context (passed by value to kernels)
    int P, L, E, O, nf, n, nblk;
    int rank, world;
    int sbw;   // 0: S dense [n*n]; > 0: S in band storage, row r holds columns r-sbw..r (large windows, ba_band.cu)
    // two-sided ("twisted") reduced solve of the persistent kernel: pose blocks [0, tw_m0) are eliminated top-down by CTA 0,
    // blocks [tw_m0 + tw_w, nf) bottom-up by CTA 1, the tw_w separator blocks in between last (tw_m0 == 0: off)
    int tw_m0, tw_w;
    const int* tw_cmax1;   // [3 (nf - tw_m0)] envelope of the mirrored bottom part
    double* tw_buf;        // CTA 1 -> CTA 0: separator Schur complement | rhs | ok; CTA 0 -> CTA 1 at TW_XM: separator solution, mirrored
    unsigned* tw_flag;     // [0] bottom part ready (sequence number), [1] published separator entries (count), [2] (sequence << 1) | ok
    // state
    double* xp[2];
    double* xl[2];
    LMState* st;
    // edges, landmark-sorted
    const int *e_pose, *e_hidx, *lm_ptr;
    const double *e_u, *e_v, *e_w00, *e_w01, *e_w11;
    const int* hidx;
    // odometry edges
    const int *o_i, *o_j;
    const double *o_m, *o_w;  // [3][O], [6][O]
    // per-edge / per-landmark outputs (SoA, component-major)
    // per-edge records, array-of-structures with a 96 B stride so that one record is exactly 3 L2 sectors:
    //   Hpl[e] = 3x3 pose-landmark block; PH[e] = pose-side Hessian (6 unique) + gradient (3); Y[e] = Hpl Hll^-1 (9) + g (3)
    double *Hpl, *PH, *Y;
    double *Hll, *bl, *HllInv;            // [6][L] [3][L] [6][L]
    double *oAii, *oAij, *oAjj, *obi, *obj;  // [6][O] [9][O] [6][O] [3][O] [3][O]
    // pose-side gathers
    const int *pose_ptr, *pose_edges, *pose_odo_ptr, *pose_odo;
    double *Hpp, *bp;                     // [6][nf], [n]
    // reduced system
    const int *blk_a, *blk_b, *blk_pair_ptr, *pair_e1, *pair_e2, *blk_odo_ptr, *blk_odo;
    const int* colmax;                    // [n] envelope of the reduced system (last structurally non-zero row per column)
    const int* blk_order;                 // [nord] serving order of the persistent kernel: position p belongs to worker p % W; -1 = hole
    int nord;
    double *S, *bs, *scal, *dxp, *dxl;    // S [n*n] | bs [n] | scal [8] contiguous (all-reduce buffer)
    double *part_chi, *part_scale;
    int nb_lm, nb_odo;
};

// bytes of dynamic shared memory the shared-memory block LDL^T needs for n unknowns
__host__ __device__ inline size_t ldlt_smem_bytes(int n) { return ((size_t)n * n + n + 3 * (size_t)n + 2) * 8 + (size_t)n * 4 + 16 + 128; }
// dynamic shared memory of the persistent launch: CTA 0's reduced solve, and on worker CTAs pair lists + reduction scratch
inline size_t pk_dyn_smem_bytes(int n) { return std::max(ldlt_smem_bytes(n), (size_t)160 * 1024); }

// Run-time switches, read from the environment when a context is created (INTEGRATION.md section 5)
struct Switches {
    int pk_grid_limit = 0;          // SE2GPU_BA_PK_GRID: cap on the cooperative grid (several contexts on one GPU); 0 = none
    double peer_timeout_s = 10.0;   // SE2GPU_BA_PEER_TIMEOUT_S
    bool debug = false;             // SE2GPU_BA_DEBUG: set_problem timings and per-CTA phase cycles to stderr
    bool no_band = false;           // SE2GPU_BA_NO_BAND: large windows take the global-memory envelope solver
    bool no_twist = false;          // SE2GPU_BA_NO_TWIST: the persistent kernel's reduced solve stays on one CTA
    int batch_cluster = 0;          // SE2GPU_BA_BATCH_CLUSTER: cluster size (2, 4, 8) of the window in se2gpu_ba_optimize_batch
                                    // instead of 8; for measuring the sizes against each other (tools/ba_batch_bench.py)
};

// What se2gpu_ba_set_problem_device keeps between calls (ba_loader.cu): the loaded topology as device copies, the
// landmark sort as a device array, and the scratch of the structure build. Every buffer is allocated on first use and grown
// on demand; the topology copies are valid only after a device load (a host load clears `valid`).
struct DevLoad {
    bool valid = false;
    uint8_t* fixed = nullptr;                                          // [maxP]
    int *edge_pose = nullptr, *edge_point = nullptr, *odo_i = nullptr, *odo_j = nullptr;   // [maxE], [maxE], [maxO], [maxO]
    int* perm = nullptr;                                               // [maxE] sorted edge position -> original edge
    int* sc = nullptr;                                                 // [16] device scalars of the build (DL_* in ba_loader.cu)
    int* sc_host = nullptr;                                            // [16] page-locked mirror
    int *k0 = nullptr, *v0 = nullptr, *k1 = nullptr, *v1 = nullptr;   // radix sort ping-pong keys / values
    int *g1 = nullptr, *g2 = nullptr;                                  // pair (k1, k2) in generation order
    int *hist = nullptr, *aux = nullptr;                               // radix digit counts, scan block totals
    int *lo = nullptr, *hi = nullptr;                                  // [L] per-landmark first / last free pose
    int *pair_off = nullptr;                                           // [El + 1] first pair of each sorted edge
    unsigned* bits = nullptr; int* wprefix = nullptr;                  // nf x nf block bitmap, popcount prefix per word
    int* planin = nullptr; std::vector<int> planin_host;               // bmax [nf] | pairs per block | pose edges per diagonal block
    size_t cap_sort = 0, cap_pairs = 0, cap_hist = 0, cap_aux = 0, cap_lm = 0, cap_off = 0, cap_bits = 0, cap_wprefix = 0, cap_plan = 0;
};

}  // namespace se2ba

struct se2gpu_ba {
    se2gpu::PinnedArena arena;    // page-locked staging of set_problem's uploads
    se2gpu::PinnedArena arena2;   // page-locked arrays that set_problem builds in place (per-edge and per-pair lists)
    int device = 0;
    int maxP = 0, maxL = 0, maxE = 0, maxO = 0, maxN = 0;
    size_t cap_pairs = 0, cap_blk = 0;
    cudaStream_t stream = nullptr;
    int rank = 0, world = 1;
    se2gpu_allreduce_fn allreduce = nullptr;
    se2ba::Switches sw;
    // sharded persistent kernel: exchange through peer memory (se2gpu_ba_peer_export / _import / _peer_attach_local)
    double* xch = nullptr;                      // this rank's exchange block: flags + 2 scalar slots
    int xslot = 0;                              // doubles per scalar slot
    double* ssum = nullptr;                     // rank-summed [S | bs]
    long long* go = nullptr;                    // [2] local hand-off words of pk_wait_peers
    int* env_idx = nullptr; int nenv = 0; size_t env_cap = 0;   // envelope entries of [S | bs] (what the exchange sums)
    void* peer_opened[16] = {};                 // mappings opened with cudaIpcOpenMemHandle (closed on destroy)
    const double* peer_red[8] = {};
    const double* peer_xch[8] = {};
    bool peer_on = false;
    long long peer_epoch = 0;
    void* ar_user = nullptr;
    se2ba::Dev d{};               // the device pointers, and the sizes of the loaded window
    se2ba::Cam cam{};
    se2gpu::DeviceBuffers bufs;   // owns every device buffer of the context except xch, ssum and go (se2gpu_ba_destroy)
    double* red = nullptr;     // all-reduce buffer [maxN*maxN + maxN + 8]
    double* ywork = nullptr;
    se2gpu_ba_iter_stats* stats_dev = nullptr;
    int max_stats = 64;
    se2ba::LMState* st_host = nullptr;  // pinned
    std::vector<int> perm;       // sorted edge position -> original edge index
    int P = 0, L = 0, E = 0, O = 0;
    int nb_scale = 0;
    bool loaded = false;
    double *xp0 = nullptr, *xl0 = nullptr;   // estimates as loaded (se2gpu_ba_reset)
    float* wb32 = nullptr;                   // [3 maxP + 8 + 3 maxL] se2gpu_ba_get_f32's narrowed estimates
    se2gpu::Profiler prof;
    // persistent cooperative path
    int mode = 0;              // 0 auto, 1 multi-launch, 2 persistent
    int pk_grid = 0;           // co-resident CTAs (0 = unavailable)
    double *pk_part_chi = nullptr, *pk_part_scale = nullptr, *pk_part_max = nullptr;
    int* abort_host = nullptr; int* abort_host_dev = nullptr; int* abort_dev = nullptr;
    double *trace_p = nullptr, *trace_l = nullptr; size_t trace_cap_p = 0, trace_cap_l = 0;
    long long* phase_cycles = nullptr;   // device [8]
    long long* cta_work = nullptr;       // device [1024][8]
    int pk_launches = 0, clock_khz = 0;
    // topology of the loaded window (host copies): a set_problem with the same graph structure only refreshes the values
    std::vector<int> t_edge_pose, t_edge_point, t_odo_i, t_odo_j; std::vector<uint8_t> t_fixed; int t_rank = -1, t_world = -1;
    se2band::Plan band;        // partitioned band solver for reduced systems beyond one CTA's shared memory
    int smem_optin = 0;
    int plan[SE2GPU_BA_PLAN_FIELDS] = {};   // host-side decisions of the last full set_problem (se2gpu_ba_debug_plan)
    se2ba::DevLoad dl;                      // se2gpu_ba_set_problem_device
    // decide()'s inputs for the loaded window - bmax [nf] | pairs per block [nblk] | pose edges per diagonal block [nblk] - and
    // the grid the uploaded plan (tw_*, blk_order) was made for: a batched optimize runs a window on a cluster of another size
    std::vector<int> plan_in;
    int plan_grid = 0;
    unsigned long long* bdesc = nullptr; size_t bdesc_cap = 0;   // se2gpu_ba_optimize_batch: window descriptors, in 8-byte words
    long long struct_len[SE2GPU_BA_STRUCT_COUNT] = {};   // element count of each se2gpu_ba_debug_structure array
};

namespace se2ba {

// Makes the uploaded plan the one decide() makes for `grid` CTAs (ba_loader.cu); enqueued on the context's stream
int plan_for_grid(se2gpu_ba* h, int grid);

// LM scalars of a freshly loaded (or reset) window, enqueued on the context's stream
inline int reset_lm_state(se2gpu_ba* h) {
    LMState st0{};
    st0.ni = 2;
    *h->st_host = st0;
    SE2_CUDA(cudaMemcpyAsync(h->d.st, h->st_host, sizeof(LMState), cudaMemcpyHostToDevice, h->stream));
    return SE2GPU_OK;
}

}  // namespace se2ba
