// Loader-side kernels of the local BA (SURVEY.md section 8f N1): what Map::loadLocalGraph computes per EdgeSE2XYZ right
// before handing the graph to the optimiser (reference src/Map.cpp:1024-1049) - the 2x2 information matrix
//   Omega = (sigma_rot * J_rotxy J_rotxy^T + sigma_z * J_z J_z^T + sigma_l^2 I)^-1
// evaluated ONCE at load time from the keyframe's float Tcw / Twb, the float camera-frame measurement mViewMPs[ftrIdx],
// the float landmark position and mvLevelSigma2[octave]; all arithmetic in double on the widened floats, like the
// reference's toVector3d / toMatrix3d conversions. One thread per edge, coalesced SoA reads, three doubles out.
#include "common.h"

namespace {

using se2gpu::fail;

struct InfoArgs {
    int E;
    const float* lc;          // [E*3] pKF->mViewMPs[ftrIdx]
    const int* edge_pose;     // [E] keyframe slot
    const int* edge_point;    // [E] landmark slot
    const int* octave;        // [E]
    const float* Rcw;         // [P*9] rows of pKF->Tcw(0:3,0:3)
    const float* twb;         // [P*2] pKF->Twb.x, .y
    const float* lw;          // [L*3] pMP->getPos()
    const float* level_sigma2;  // [nlevels] mvLevelSigma2
    int nlevels;
    float fx, sigma_rotxy, sigma_z;
    double* info;             // [E*3] xx, xy, yy
};

__global__ void __launch_bounds__(256) k_edge_information(InfoArgs a) {
    const int e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= a.E) return;
    const int p = a.edge_pose[e], j = a.edge_point[e];
    int oc = a.octave[e];
    oc = oc < 0 ? 0 : (oc >= a.nlevels ? a.nlevels - 1 : oc);
    const double sigma2 = (double)a.level_sigma2[oc];
    const double lc0 = a.lc[3 * e], lc1 = a.lc[3 * e + 1], lc2 = a.lc[3 * e + 2];
    const double zc_inv = 1. / lc2, zc_inv2 = zc_inv * zc_inv;
    const double fx = (double)a.fx;
    const double Jpi[6] = {fx * zc_inv, 0, -fx * lc0 * zc_inv2, 0, fx * zc_inv, -fx * lc1 * zc_inv2};
    double R[9];
#pragma unroll
    for (int k = 0; k < 9; ++k) R[k] = (double)a.Rcw[9 * (size_t)p + k];
    double M[6];    // J_pi * Rcw (2x3)
#pragma unroll
    for (int r = 0; r < 2; ++r)
#pragma unroll
        for (int c = 0; c < 3; ++c) M[r * 3 + c] = Jpi[r * 3] * R[c] + Jpi[r * 3 + 1] * R[3 + c] + Jpi[r * 3 + 2] * R[6 + c];
    const double d0 = (double)a.lw[3 * (size_t)j] - (double)a.twb[2 * (size_t)p], d1 = (double)a.lw[3 * (size_t)j + 1] - (double)a.twb[2 * (size_t)p + 1];
    const double d2 = (double)a.lw[3 * (size_t)j + 2];
    // (M * skew(d))[:, 0:2] with skew(d) = [[0,-d2,d1],[d2,0,-d0],[-d1,d0,0]];  J_z = -M[:, 2]
    double Jr[4], Jz[2];
#pragma unroll
    for (int r = 0; r < 2; ++r) {
        Jr[r * 2 + 0] = M[r * 3 + 1] * d2 - M[r * 3 + 2] * d1;
        Jr[r * 2 + 1] = -M[r * 3 + 0] * d2 + M[r * 3 + 2] * d0;
        Jz[r] = -M[r * 3 + 2];
    }
    const double sr = (double)a.sigma_rotxy, sz = (double)a.sigma_z;
    // Sigma_all = sr * Jr Jr^T + sz * Jz Jz^T + sigma2 I   (Eigen evaluates (sr*Jr)*Jr^T; the difference is below 1 ulp of the sum)
    const double s00 = (sr * Jr[0]) * Jr[0] + (sr * Jr[1]) * Jr[1] + (sz * Jz[0]) * Jz[0] + sigma2;
    const double s01 = (sr * Jr[0]) * Jr[2] + (sr * Jr[1]) * Jr[3] + (sz * Jz[0]) * Jz[1];
    const double s10 = (sr * Jr[2]) * Jr[0] + (sr * Jr[3]) * Jr[1] + (sz * Jz[1]) * Jz[0];
    const double s11 = (sr * Jr[2]) * Jr[2] + (sr * Jr[3]) * Jr[3] + (sz * Jz[1]) * Jz[1] + sigma2;
    // Matrix2d::inverse(): adjugate / determinant
    const double invdet = 1. / (s00 * s11 - s10 * s01);
    const double i00 = s11 * invdet, i01 = -s01 * invdet, i10 = -s10 * invdet, i11 = s00 * invdet;
    a.info[3 * (size_t)e] = i00;
    a.info[3 * (size_t)e + 1] = 0.5 * (i01 + i10);     // se2gpu_ba_set_problem stores the symmetric part (xx, xy, yy)
    a.info[3 * (size_t)e + 2] = i11;
}

}  // namespace

extern "C" {

int se2gpu_ba_build_information(int P, int L, int E, const float* view_mp, const int* edge_pose, const int* edge_point,
                                const int* octave, const float* kf_Rcw, const float* kf_twb_xy, const float* mp_pos,
                                const float* level_sigma2, int nlevels, float fx, float xrot_info, float z_info, double* info,
                                int device) {
    if (P <= 0 || L < 0 || E < 0 || nlevels <= 0) return fail(SE2GPU_ERR_INVALID, "bad sizes");
    if (E == 0) return SE2GPU_OK;
    if (!view_mp || !edge_pose || !edge_point || !octave || !kf_Rcw || !kf_twb_xy || !mp_pos || !level_sigma2 || !info)
        return fail(SE2GPU_ERR_INVALID, "null argument");
    for (int e = 0; e < E; ++e)
        if (edge_pose[e] < 0 || edge_pose[e] >= P || edge_point[e] < 0 || edge_point[e] >= L) return fail(SE2GPU_ERR_INVALID, "edge %d references a missing vertex", e);
    se2gpu::HostStage st(device);
    if (const int rc = st.status()) return rc;
    InfoArgs a{};
    a.E = E; a.nlevels = nlevels; a.fx = fx;
    a.sigma_rotxy = 1.f / xrot_info;       // float Sigma_rotxy = 1./Config::PLANEMOTION_XROT_INFO   (Map.cpp:1043)
    a.sigma_z = 1.f / z_info;              // float Sigma_z = 1./Config::PLANEMOTION_Z_INFO          (Map.cpp:1044)
    a.info = st.output(info, 3 * (size_t)E);
    a.lc = st.upload(view_mp, 3 * (size_t)E); a.edge_pose = st.upload(edge_pose, E); a.edge_point = st.upload(edge_point, E);
    a.octave = st.upload(octave, E); a.Rcw = st.upload(kf_Rcw, 9 * (size_t)P); a.twb = st.upload(kf_twb_xy, 2 * (size_t)P);
    a.lw = st.upload(mp_pos, 3 * (size_t)L); a.level_sigma2 = st.upload(level_sigma2, nlevels);
    if (const int rc = st.status()) return rc;
    SE2_LAUNCH(k_edge_information, (E + 255) / 256, 256, 0, 0, a);
    st.check(cudaGetLastError(), "kernel launch");
    return st.finish();
}

}  // extern "C"
