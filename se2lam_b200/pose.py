"""Pose-only SE(3) bundle adjustment (Localizer::DoLocalBA, reference src/Localizer.cpp:233-302) over the C ABI.

`poseOnlyBA` takes batched host arrays and returns new ones; `localizerBA` runs the Localizer-shaped device entry on
device buffers (torch CUDA tensors or raw device pointers), e.g. the outputs of the extractor and
MatchByProjectionDevice, so the ORB -> BoW -> MatchByProjection -> pose BA chain never leaves the GPU.
"""
from __future__ import annotations

import ctypes as C

import numpy as np

from ._capi import BA_STATS_DTYPE, PoseBAParams, check, lib, ptr

OK, NO_EDGES, NOT_PD, GATED = 0, 1, 2, 3


def params(fx, cx, cy, Tbc, huber_delta, xrot_info=1e6, yrot_info=1e6, z_info=1.0, iterations=30) -> PoseBAParams:
    """fx, cx, cy = Config::Kcam's focal length and principal point; Tbc = Config::bTc [4,4]; huber_delta = Config::TH_HUBER;
    the plane-motion information values default to the reference's Config (1e6, 1e6, 1); DoLocalBA runs 30 iterations."""
    p = PoseBAParams()
    p.fx, p.cx, p.cy = float(fx), float(cx), float(cy)
    p.Tbc[:] = [float(v) for v in np.asarray(Tbc, np.float32).reshape(16)]
    p.huber_delta = float(huber_delta)
    p.xrot_info, p.yrot_info, p.z_info = float(xrot_info), float(yrot_info), float(z_info)
    p.iterations = int(iterations)
    return p


def poseOnlyBA(Tcw, edge_ptr, xyz, uv, info, prm: PoseBAParams, device=0, trace=False):
    """B problems in CSR form: Tcw [B,4,4] start poses, edge_ptr [B+1], xyz [E,3], uv [E,2], info [E] (information scale).
    Returns dict(Tcw [B,4,4] float32, pose [B,7] (qx,qy,qz,qw,tx,ty,tz), iterations [B], status [B],
    stats [B, iterations] BA_STATS_DTYPE) and with trace=True also trace [B, iterations, 7], the pose after every iteration.
    The inputs are not modified."""
    T = np.ascontiguousarray(Tcw, np.float32).reshape(-1, 16).copy()
    B = len(T)
    ep = np.ascontiguousarray(edge_ptr, np.int32)
    if len(ep) != B + 1:
        raise ValueError("edge_ptr must have B + 1 entries")
    E = int(ep[-1]) if B else 0
    x = np.ascontiguousarray(xyz, np.float32).reshape(-1, 3)
    u = np.ascontiguousarray(uv, np.float32).reshape(-1, 2)
    w = np.ascontiguousarray(info, np.float32).reshape(-1)
    if len(x) < E or len(u) < E or len(w) < E:
        raise ValueError("edge arrays shorter than edge_ptr[-1]")
    its = max(prm.iterations, 1)
    st = np.zeros((B, its), BA_STATS_DTYPE)
    n = np.zeros(B, np.int32); status = np.zeros(B, np.int32); pose = np.zeros((B, 7))
    if trace:
        tr = np.zeros((B, its, 7))
        check(lib().se2gpu_pose_ba_debug_trace(B, ptr(T), ptr(ep), ptr(x), ptr(u), ptr(w), C.byref(prm), ptr(st), ptr(n), ptr(status),
                                               ptr(pose), ptr(tr), device), "se2gpu_pose_ba_debug_trace")
    else:
        check(lib().se2gpu_pose_ba(B, ptr(T), ptr(ep), ptr(x), ptr(u), ptr(w), C.byref(prm), ptr(st), ptr(n), ptr(status), ptr(pose),
                                   device), "se2gpu_pose_ba")
    out = dict(Tcw=T.reshape(B, 4, 4), pose=pose, iterations=n, status=status, stats=st[:, :prm.iterations])
    if trace:
        out["trace"] = tr[:, :prm.iterations]
    return out


def poseOnlyBADevice(B, d_Tcw, d_edge_ptr, d_xyz, d_uv, d_info, prm: PoseBAParams, d_stats=None, d_iterations=None, d_status=None,
                     d_pose=None, stream=0):
    """se2gpu_pose_ba_device on device buffers (laid out as poseOnlyBA's arrays), asynchronous on `stream`."""
    check(lib().se2gpu_pose_ba_device(int(B), ptr(d_Tcw), ptr(d_edge_ptr), ptr(d_xyz), ptr(d_uv), ptr(d_info), C.byref(prm),
                                      ptr(d_stats), ptr(d_iterations), ptr(d_status), ptr(d_pose), C.c_void_p(int(stream) if stream else 0)),
          "se2gpu_pose_ba_device")


class Localizer:
    """Device workspace of se2gpu_localizer_ba_device for up to max_map_points local map points."""

    def __init__(self, max_map_points, device=0):
        self.h = lib().se2gpu_localizer_create(int(max_map_points), int(device))
        if not self.h:
            check(-1, "se2gpu_localizer_create")

    def __del__(self):
        if getattr(self, "h", None):
            lib().se2gpu_localizer_destroy(self.h)
            self.h = None

    def localizerBA(self, d_kf_kp, n_kf, d_matches_idx_mp, n_mp, d_mp_xyz, d_mp_use, d_inv_sigma2, nlevels, d_Tcw, prm: PoseBAParams,
                    min_edges=30, d_n_kf=None, d_n_edges=None, d_stats=None, d_iterations=None, d_status=None, d_pose=None, stream=0):
        """MatchLocalMap's observations + DoLocalBA on device buffers; d_Tcw [16] float32 is updated in place."""
        check(lib().se2gpu_localizer_ba_device(self.h, ptr(d_kf_kp), int(n_kf), ptr(d_n_kf), ptr(d_matches_idx_mp), int(n_mp), ptr(d_mp_xyz),
                                               ptr(d_mp_use), ptr(d_inv_sigma2), int(nlevels), ptr(d_Tcw), C.byref(prm), int(min_edges),
                                               ptr(d_n_edges), ptr(d_stats), ptr(d_iterations), ptr(d_status), ptr(d_pose),
                                               C.c_void_p(int(stream) if stream else 0)), "se2gpu_localizer_ba_device")


def localizerBA(kf_kp, matches_idx_mp, mp_xyz, mp_use, inv_sigma2, Tcw, prm: PoseBAParams, min_edges=30, device=0):
    """Host-array convenience over se2gpu_localizer_ba_device: uploads, runs, and returns
    dict(Tcw [4,4] float32, n_edges, iterations, status, pose [7], stats)."""
    import torch
    dev = torch.device("cuda", device)

    def up(a, dt):
        a = np.ascontiguousarray(a, dt)
        return torch.from_numpy(a.view(np.uint8) if a.dtype.fields else a).to(dev)
    kp = np.ascontiguousarray(kf_kp)
    n_kf, n_mp = len(kp), len(np.asarray(mp_use))
    d_kp = up(kp, kp.dtype) if n_kf else torch.zeros(28, dtype=torch.uint8, device=dev)
    d_m = up(matches_idx_mp, np.int32)
    d_x = up(np.asarray(mp_xyz, np.float32).reshape(-1, 3), np.float32)
    d_use = up(mp_use, np.uint8)
    d_s = up(inv_sigma2, np.float32)
    d_T = up(np.asarray(Tcw, np.float32).reshape(16), np.float32)
    its = max(prm.iterations, 1)
    d_ne = torch.zeros(1, dtype=torch.int32, device=dev); d_it = torch.zeros(1, dtype=torch.int32, device=dev)
    d_st = torch.zeros(1, dtype=torch.int32, device=dev); d_pose = torch.zeros(7, dtype=torch.float64, device=dev)
    d_stats = torch.zeros(its * BA_STATS_DTYPE.itemsize, dtype=torch.uint8, device=dev)
    loc = Localizer(max(n_mp, 1), device)
    with torch.cuda.device(dev):
        stream = torch.cuda.current_stream().cuda_stream
        loc.localizerBA(d_kp, n_kf, d_m, n_mp, d_x, d_use, d_s, len(np.asarray(inv_sigma2)), d_T, prm, min_edges, None, d_ne, d_stats, d_it,
                        d_st, d_pose, stream)
        torch.cuda.synchronize()
    n = int(d_it.item())
    return dict(Tcw=d_T.cpu().numpy().reshape(4, 4), n_edges=int(d_ne.item()), iterations=n, status=int(d_st.item()),
                pose=d_pose.cpu().numpy(), stats=d_stats.cpu().numpy().view(BA_STATS_DTYPE)[:n].copy())


def localizer_edges(kf_kp, matches_idx_mp, mp_xyz, mp_use, inv_sigma2):
    """The host flattening se2gpu_localizer_ba_device performs on the device (for callers that hold host arrays):
    (xyz [E,3], uv [E,2], info [E]) in ascending map-point index."""
    m = np.asarray(matches_idx_mp, np.int64)
    n_mp = len(np.asarray(mp_use))
    best = np.full(n_mp, -1, np.int64)
    for i, j in enumerate(m):
        if 0 <= j < n_mp:
            best[j] = i                 # ascending i: the last (highest) keypoint index wins
    js = np.flatnonzero((best >= 0) & (np.asarray(mp_use) != 0))
    kp = np.asarray(kf_kp)
    w0 = np.float32(inv_sigma2[kp["octave"][0]]) if len(kp) else np.float32(0)
    xyz = np.asarray(mp_xyz, np.float32).reshape(-1, 3)[js]
    uv = np.stack([kp["x"][best[js]], kp["y"][best[js]]], axis=1).astype(np.float32) if len(js) else np.zeros((0, 2), np.float32)
    return xyz, uv, np.full(len(js), w0, np.float32)
