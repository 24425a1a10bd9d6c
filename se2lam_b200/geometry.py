"""Two-view geometry over matches (reference src/cvutil.cpp, src/Track.cpp, src/LocalMapper.cpp) over the C ABI.

`triangulate`, `doTriangulate`, `calcSE3toXYZInfo` and `findCorrespdProjection` take host arrays and return new ones; the
raw `_device` entry points (include/se2gpu.h) take device pointers, e.g. torch tensors' data_ptr(), and run on a stream.
"""
from __future__ import annotations

import numpy as np

from ._capi import KP_DTYPE, check, lib, ptr


def _c(a, dt):
    return np.ascontiguousarray(a, dt)


def _kp(a):
    a = np.ascontiguousarray(a)
    if a.dtype != KP_DTYPE:
        raise TypeError("keypoints must be a KP_DTYPE array")
    return a


def triangulate(pt1, pt2, P, idx1=None, idx2=None, device=0):
    """cvu::triangulate for n pairs. pt1/pt2 [n,2]; P [n_proj,3,4] (or one [3,4] pair P1/P2 with idx None: P = (P1, P2)).
    Returns xyz [n,3] float32."""
    pt1 = _c(pt1, np.float32).reshape(-1, 2); pt2 = _c(pt2, np.float32).reshape(-1, 2)
    n = len(pt1)
    if idx1 is None and idx2 is None:
        P = _c(np.stack([np.asarray(P[0]), np.asarray(P[1])]), np.float32)
        idx1 = np.zeros(n, np.int32); idx2 = np.ones(n, np.int32)
    P = _c(P, np.float32).reshape(-1, 12)
    idx1 = _c(idx1, np.int32); idx2 = _c(idx2, np.int32)
    xyz = np.zeros((n, 3), np.float32)
    check(lib().se2gpu_triangulate(n, ptr(pt1), ptr(pt2), ptr(P), len(P), ptr(idx1), ptr(idx2), ptr(xyz), device), "se2gpu_triangulate")
    return xyz


def doTriangulate(kp_kf, kp_frame, matches12, kf_observed, kf_view_mp, Tcr, K, lower_depth, upper_depth, local_mps,
                  min_parallax_deg=2, device=0):
    """Track::doTriangulate (Track.cpp:389-416) past its nMinFrames check. Returns
    (nTrackedOld, matches12, local_mps, good_prl, nGoodPrl); the inputs are not modified."""
    kp_kf = _kp(kp_kf); kp_frame = _kp(kp_frame)
    n = len(kp_kf)
    m = _c(matches12, np.int32).copy(); obs = _c(kf_observed, np.uint8); vm = _c(kf_view_mp, np.float32)
    lm = _c(local_mps, np.float32).copy(); Tcr = _c(Tcr, np.float32); K = _c(K, np.float32)
    good = np.zeros(n, np.uint8); counts = np.zeros(2, np.int32)
    check(lib().se2gpu_track_triangulate(ptr(kp_kf), n, ptr(kp_frame), len(kp_frame), ptr(m), ptr(obs), ptr(vm), ptr(Tcr), ptr(K),
                                         float(lower_depth), float(upper_depth), int(min_parallax_deg), ptr(lm), ptr(good),
                                         ptr(counts), device), "se2gpu_track_triangulate")
    return int(counts[0]), m, lm, good.astype(bool), int(counts[1])


def removeOutliers(kp1, kp2, matches12, device=0, return_details=False):
    """Track::removeOutliers (Track.cpp:308-344): cv::findFundamentalMat's RANSAC / LMedS mask applied to matches12, then
    every match dropped below 10 inliers. kp1 / kp2 are KP_DTYPE arrays, or lists of them for a batch of frame pairs (one
    call). Returns (nInlier, matches12) - lists for a batch - and with return_details also F [3,3] (zeros when
    cv::findFundamentalMat returns none) and the number of hypotheses run. The inputs are not modified."""
    batch = isinstance(kp1, (list, tuple))
    K1 = [_kp(k) for k in (kp1 if batch else [kp1])]
    K2 = [_kp(k) for k in (kp2 if batch else [kp2])]
    M = [_c(m, np.int32) for m in (matches12 if batch else [matches12])]
    B = len(K1)
    if len(K2) != B or len(M) != B or any(len(m) != len(k) for m, k in zip(M, K1)):
        raise ValueError("kp1, kp2 and matches12 must describe the same frame pairs")
    cap1 = max([len(k) for k in K1] + [0]); cap2 = max([len(k) for k in K2] + [0])
    k1 = np.zeros((B, cap1), KP_DTYPE); k2 = np.zeros((B, cap2), KP_DTYPE); m = np.full((B, cap1), -1, np.int32)
    for b in range(B):
        k1[b, :len(K1[b])] = K1[b]; k2[b, :len(K2[b])] = K2[b]; m[b, :len(M[b])] = M[b]
    n1 = np.array([len(k) for k in K1], np.int32); n2 = np.array([len(k) for k in K2], np.int32)
    nin = np.zeros(B, np.int32); F = np.zeros((B, 3, 3)); it = np.zeros(B, np.int32)
    check(lib().se2gpu_remove_outliers(B, ptr(k1), ptr(n1), cap1, ptr(k2), ptr(n2), cap2, ptr(m), ptr(nin), ptr(F), ptr(it),
                                       device), "se2gpu_remove_outliers")
    out = [(int(nin[b]), m[b, :n1[b]].copy(), F[b], int(it[b])) for b in range(B)]
    out = [o if return_details else o[:2] for o in out]
    return out if batch else out[0]


def calcSE3toXYZInfo(xyz1, pose1, pose2, Tcw, fxCam, device=0):
    """Track::calcSE3toXYZInfo for n points: xyz1 [n,3], Tcw [n_pose,4,4], pose1/pose2 [n] indices into Tcw.
    Returns (info1, info2), each [n,3,3] float64."""
    xyz1 = _c(xyz1, np.float32).reshape(-1, 3); Tcw = _c(Tcw, np.float32).reshape(-1, 16)
    pose1 = _c(pose1, np.int32); pose2 = _c(pose2, np.int32)
    n = len(xyz1)
    i1 = np.zeros((n, 3, 3)); i2 = np.zeros((n, 3, 3))
    check(lib().se2gpu_xyz_info(n, ptr(xyz1), ptr(pose1), ptr(pose2), ptr(Tcw), len(Tcw), float(fxCam), ptr(i1), ptr(i2), device),
          "se2gpu_xyz_info")
    return i1, i2


def findCorrespdProjection(kf_kp, matches_idx_mp, Tcw_new, mp, Tcw_table, K, lower_depth, upper_depth, fxCam, device=0):
    """The MatchByProjection branch of LocalMapper::findCorrespd (LocalMapper.cpp:119-141) without the object-graph updates.
    mp = dict(main_measure [M,2], main_pose [M], main_octave [M], normal [M,3], min_dist [M], max_dist [M]).
    Returns (accept [n] bool, posNewKF [n,3] float32, infoNew [n,3,3] float64); rows not accepted are zero."""
    kf_kp = _kp(kf_kp); n = len(kf_kp)
    a = [_c(mp["main_measure"], np.float32), _c(mp["main_pose"], np.int32), _c(mp["main_octave"], np.int32),
         _c(mp["normal"], np.float32), _c(mp["min_dist"], np.float32), _c(mp["max_dist"], np.float32)]
    mi = _c(matches_idx_mp, np.int32); Tn = _c(Tcw_new, np.float32); tab = _c(Tcw_table, np.float32).reshape(-1, 16)
    K = _c(K, np.float32)
    acc = np.zeros(n, np.uint8); pos = np.zeros((n, 3), np.float32); info = np.zeros((n, 3, 3))
    check(lib().se2gpu_projection_observations(ptr(kf_kp), n, ptr(mi), ptr(Tn), *[ptr(x) for x in a], len(a[1]), ptr(tab), len(tab),
                                               ptr(K), float(lower_depth), float(upper_depth), float(fxCam), ptr(acc), ptr(pos),
                                               ptr(info), device), "se2gpu_projection_observations")
    return acc.astype(bool), pos, info


def debug_svd4(A, device=0):
    """The device 4x4 Jacobi SVD (cv::SVD::compute) on [n,4,4] float32: returns (w [n,4], vt [n,4,4])."""
    A = _c(A, np.float32).reshape(-1, 16); n = len(A)
    w = np.zeros((n, 4), np.float32); vt = np.zeros((n, 4, 4), np.float32)
    check(lib().se2gpu_debug_svd4(n, ptr(A), ptr(w), ptr(vt), device), "se2gpu_debug_svd4")
    return w, vt
