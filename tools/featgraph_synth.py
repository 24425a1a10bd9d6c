"""Seeded planar scenes for the feature-graph constraint (GlobalMapper::CreateFeatEdge): two SE(2) keyframes lifted through
Tbc, points in both frusta, per-keyframe measurements z with noise drawn from Omega^-1, Omega from the formula of
Track::calcSE3toXYZInfo (the one se2gpu_xyz_info implements), and a stated share of gross outliers for the matched mode.
"""
from __future__ import annotations

import numpy as np

FX = 500.0
# camera (z forward, x right, y down) in the robot frame (x forward, y left, z up), 10 cm ahead and 30 cm up
TBC = np.array([[0, 0, 1, 0.1], [-1, 0, 0, 0.0], [0, -1, 0, 0.3], [0, 0, 0, 1]], np.float64)


def se2_to_Twb(x, y, th):
    c, s = np.cos(th), np.sin(th)
    return np.array([[c, -s, 0, x], [s, c, 0, y], [0, 0, 1, 0], [0, 0, 0, 1]], np.float64)


def rodrigues(k):
    th = np.linalg.norm(k)
    if th < 1e-12:
        return np.eye(3)
    a = k / th
    K = np.array([[0, -a[2], a[1]], [a[2], 0, -a[0]], [-a[1], a[0], 0]])
    return np.eye(3) + np.sin(th) * K + (1 - np.cos(th)) * K @ K


def xyz_info(xyz1, Tcw1, Tcw2, fx=FX):
    """Track::calcSE3toXYZInfo for one point given in camera 1: (info1, info2), 3 x 3 each."""
    Twc1, Twc2 = np.linalg.inv(Tcw1), np.linalg.inv(Tcw2)
    O1, O2 = Twc1[:3, 3], Twc2[:3, 3]
    xyz = Twc1[:3, :3] @ xyz1 + Twc1[:3, 3]
    v1, v2 = xyz - O1, xyz - O2
    sin_par = np.linalg.norm(np.cross(v1, v2)) / (np.linalg.norm(v1) * np.linalg.norm(v2))
    sin_par = max(sin_par, 1e-4)
    xyz2 = Tcw2[:3, :3] @ xyz + Tcw2[:3, 3]
    l1, l2 = np.linalg.norm(xyz1), np.linalg.norm(xyz2)
    dxy1, dxy2 = 2 * l1 / fx, 2 * l2 / fx
    dz1, dz2 = dxy2 / sin_par, dxy1 / sin_par
    out = []
    for p, l, dxy, dz in ((xyz1, l1, dxy1, dz1), (xyz2, l2, dxy2, dz2)):
        k = np.cross(p, [0, 0, l])
        nk = np.linalg.norm(k)
        R = rodrigues(k * (np.arcsin(min(nk / (l * l), 1.0)) / nk)) if nk > 1e-12 else np.eye(3)
        out.append(R.T @ np.diag([1 / dxy ** 2, 1 / dxy ** 2, 1 / dz ** 2]) @ R)
    return out[0], out[1]


def scene(seed, n_points, motion=(0.4, 0.05, 0.1), start=(1.0, -2.0, 0.3), noise=1.0, init_noise=0.02, pose_noise=(0.03, 0.01),
          outlier_share=0.0, outlier_size=(0.6, 1.2), info_scale=1.0):
    """One keyframe pair. motion = (dx, dy, dtheta) of the robot in its own frame; start = the first robot pose (x, y, theta).
    noise scales the measurement noise drawn from Omega^-1; init_noise [m] perturbs the points' start estimates;
    pose_noise = (metres, radians) perturbs the second keyframe's start estimate in the plane. outlier_share of the points
    get a gross lateral offset of outlier_size metres in keyframe 1's measurement. info_scale multiplies every Omega (a
    coarser sensor: the constraint's information then stays below InfoSE3's 1e4 clamp).
    Returns dict(Tcw0, Tcw1 [4,4] f32, xyz [P,3] f32, z0, z1 [P,3] f32, info0, info1 [P,9] f64, Tbc [4,4] f32,
    Tc0c1_true [4,4] f64, planted [P] bool, Tcw_true [2,4,4])."""
    rng = np.random.default_rng(seed)
    Twb0 = se2_to_Twb(*start)
    Twb1 = Twb0 @ se2_to_Twb(*motion)
    Tcw_true = [np.linalg.inv(Twb0 @ TBC), np.linalg.inv(Twb1 @ TBC)]
    pts_c0 = []
    while len(pts_c0) < n_points:
        d = rng.uniform(2.0, 8.0)
        p = np.array([rng.uniform(-0.4, 0.4) * d, rng.uniform(-0.3, 0.3) * d, d])
        pw = np.linalg.inv(Tcw_true[0]) @ np.append(p, 1)
        if (Tcw_true[1] @ pw)[2] > 0.5:
            pts_c0.append(p)
    pts_c0 = np.array(pts_c0).reshape(-1, 3)
    Twc0 = np.linalg.inv(Tcw_true[0])
    pw = pts_c0 @ Twc0[:3, :3].T + Twc0[:3, 3]
    z = [pw @ T[:3, :3].T + T[:3, 3] for T in Tcw_true]
    info = [np.zeros((n_points, 9)), np.zeros((n_points, 9))]
    planted = np.zeros(n_points, bool)
    n_out = int(round(outlier_share * n_points))
    if n_out:
        planted[rng.choice(n_points, n_out, replace=False)] = True
    for j in range(n_points):
        i0, i1 = xyz_info(z[0][j], Tcw_true[0], Tcw_true[1])
        for k, Ik in enumerate((info_scale * i0, info_scale * i1)):
            info[k][j] = Ik.ravel()
            if noise > 0:
                z[k][j] += noise * np.linalg.cholesky(np.linalg.inv(Ik)) @ rng.standard_normal(3)
        if planted[j]:
            a = rng.uniform(0, 2 * np.pi)
            z[1][j] += rng.uniform(*outlier_size) * np.array([np.cos(a), np.sin(a), 0.0])
    xyz = pw + init_noise * rng.standard_normal(pw.shape)
    dp = pose_noise[0] * rng.standard_normal(2)
    Twb1_start = Twb1 @ se2_to_Twb(dp[0], dp[1], pose_noise[1] * rng.standard_normal())
    f32 = lambda a: np.ascontiguousarray(a, np.float32)
    return dict(Tcw0=f32(Tcw_true[0]), Tcw1=f32(np.linalg.inv(Twb1_start @ TBC)), xyz=f32(xyz), z0=f32(z[0]), z1=f32(z[1]),
                info0=info[0], info1=info[1], Tbc=f32(TBC), Tc0c1_true=Tcw_true[0] @ np.linalg.inv(Tcw_true[1]), planted=planted,
                Tcw_true=np.array(Tcw_true))
