"""Seeded two-view scenes for the geometry entry points (tests/test_geom_*.py, tools/geom_bench.py).

Poses follow Track::updateFramePose: an SE(2) odometry pose of the base mapped into the camera through cTb / bTc
(camera z along the base's x axis, mounted 0.1 m ahead and 0.3 m above the base origin). Everything handed to the
entry points is float32, as in the reference.
"""
from __future__ import annotations

import numpy as np

KP_DTYPE = np.dtype([("x", "f4"), ("y", "f4"), ("size", "f4"), ("angle", "f4"), ("response", "f4"),
                     ("octave", "i4"), ("class_id", "i4")])
W, H = 640, 480
K = np.array([[231.976, 0, 326.923], [0, 232.443, 227.637], [0, 0, 1]], np.float32)
FX = np.float32(K[0, 0])
LOWER_DEPTH, UPPER_DEPTH = 0.1, 10.0

# cTb: base (x forward, y left, z up) -> camera (x right, y down, z forward)
_R_CB = np.array([[0, -1, 0], [0, 0, -1], [1, 0, 0]], np.float64)
CTB = np.eye(4); CTB[:3, :3] = _R_CB; CTB[:3, 3] = -_R_CB @ np.array([0.1, 0.0, 0.3])
BTC = np.linalg.inv(CTB)


def se2(x, y, th):
    c, s = np.cos(th), np.sin(th)
    T = np.eye(4); T[:2, :2] = [[c, -s], [s, c]]; T[0, 3] = x; T[1, 3] = y
    return T


def tcw_of_odom(x, y, th):
    """Tcw = cTb * Tbw (Twb from the SE(2) odometry)."""
    return (CTB @ np.linalg.inv(se2(x, y, th))).astype(np.float32)


def project(P, X):
    h = P.astype(np.float64) @ np.append(X, 1.0)
    return h[:2] / h[2]


def _keypoints(xy, octave):
    kp = np.zeros(len(xy), KP_DTYPE)
    kp["x"] = xy[:, 0]; kp["y"] = xy[:, 1]; kp["size"] = 31; kp["octave"] = octave; kp["class_id"] = -1
    return kp


def track_scene(n, seed=0, noise=0.5, frac_matched=0.8, frac_observed=0.25, degenerate=True, translation=0.3):
    """One reference keyframe and a frame: the inputs of se2gpu_track_triangulate. Returns a dict; truth [n,3] are the
    reference-camera points the keypoints were projected from."""
    rng = np.random.default_rng(seed)
    Tref = tcw_of_odom(1.0, 0.5, 0.2)
    Tcur = tcw_of_odom(1.0 + translation * np.cos(0.2), 0.5 + translation * np.sin(0.2), 0.2 + rng.uniform(-0.05, 0.05))
    Tcr = (Tcur.astype(np.float64) @ np.linalg.inv(Tref.astype(np.float64))).astype(np.float32)
    Tcr[3] = [0, 0, 0, 1]
    z = rng.uniform(0.5, 9.0, n)
    u = rng.uniform(0, W, n); v = rng.uniform(0, H, n)
    truth = np.stack([(u - K[0, 2]) / K[0, 0] * z, (v - K[1, 2]) / K[1, 1] * z, z], 1).astype(np.float32)
    P0 = K.astype(np.float64) @ np.eye(3, 4)
    P1 = K.astype(np.float64) @ Tcr[:3].astype(np.float64)
    pk = np.array([project(P0, X) for X in truth.astype(np.float64)])
    pf = np.array([project(P1, X) for X in truth.astype(np.float64)])
    pk += rng.normal(0, noise, pk.shape) if noise else 0
    pf += rng.normal(0, noise, pf.shape) if noise else 0
    if degenerate and n >= 8:
        pf[0] = pk[0]                                # identical points
        pf[1] = pk[1] + [0.0, 0.0]
        truth[2] *= -1                               # behind the camera
        pk[2] = project(P0, truth[2].astype(np.float64)); pf[2] = project(P1, truth[2].astype(np.float64))
        pk[3] = pf[3] = [K[0, 2], K[1, 2]]           # on the optical axis in both views
        pk[4] = [0, 0]; pf[4] = [W - 1, H - 1]       # far apart: depth out of range
    octave = rng.integers(0, 8, n)
    kp_kf = _keypoints(pk.astype(np.float32), octave)
    perm = rng.permutation(n)
    kp_fr = np.zeros(n, KP_DTYPE)
    kp_fr[perm] = _keypoints(pf.astype(np.float32), octave)
    matches = np.where(rng.random(n) < frac_matched, perm, -1).astype(np.int32)
    observed = (rng.random(n) < frac_observed).astype(np.uint8)
    view_mp = rng.normal(0, 3, (n, 3)).astype(np.float32)
    local_mps = rng.normal(0, 3, (n, 3)).astype(np.float32)
    return dict(kp_kf=kp_kf, kp_frame=kp_fr, matches12=matches, kf_observed=observed, kf_view_mp=view_mp, Tcr=Tcr, K=K,
                lower=LOWER_DEPTH, upper=UPPER_DEPTH, local_mps=local_mps, truth=truth, perm=perm)


def pose_table(n_pose, seed=0):
    rng = np.random.default_rng(seed)
    x = np.cumsum(rng.uniform(0.1, 0.4, n_pose)); y = rng.uniform(-0.3, 0.3, n_pose); th = rng.uniform(-0.5, 0.5, n_pose)
    return np.stack([tcw_of_odom(x[i], y[i], th[i]) for i in range(n_pose)])


def projection_scene(n_kf, n_mp=None, n_pose=8, seed=0, noise=0.5):
    """Inputs of se2gpu_projection_observations: a new keyframe (pose n_pose - 1 of the table), map points with main
    keyframes among the others, and a MatchByProjection result."""
    rng = np.random.default_rng(seed)
    n_mp = n_mp or max(n_kf, 1)
    tab = pose_table(n_pose, seed)
    Tnew = tab[-1]
    main = rng.integers(0, max(n_pose - 1, 1), n_mp).astype(np.int32)
    # world points in front of the new keyframe
    Twc_new = np.linalg.inv(Tnew.astype(np.float64))
    zc = rng.uniform(0.5, 9.0, n_mp)
    uc = rng.uniform(0, W, n_mp); vc = rng.uniform(0, H, n_mp)
    Xc = np.stack([(uc - K[0, 2]) / K[0, 0] * zc, (vc - K[1, 2]) / K[1, 1] * zc, zc, np.ones(n_mp)], 1)
    Xw = (Twc_new @ Xc.T).T[:, :3]
    meas = np.zeros((n_mp, 2)); normal = np.zeros((n_mp, 3)); dist = np.zeros(n_mp)
    for m in range(n_mp):
        Tm = tab[main[m]].astype(np.float64)
        meas[m] = project(K.astype(np.float64) @ Tm[:3], Xw[m])
        # MapPoint::acceptNewObserve dots posKF (new-keyframe coordinates) with mNormalVector: a direction near the
        # point's new-keyframe bearing passes its 30 degree test, a few are turned away from it
        d = Xc[m, :3] / np.linalg.norm(Xc[m, :3]) + rng.normal(0, 0.25 if m % 5 else 0.8, 3)
        normal[m] = d / np.linalg.norm(d)
        dist[m] = np.linalg.norm(Xc[m, :3])
    meas += rng.normal(0, noise, meas.shape) if noise else 0
    scale = rng.choice([0.5, 0.9, 1.0, 1.0, 1.0, 1.5], n_mp)
    min_dist = (dist * 0.6 * scale).astype(np.float32); max_dist = (dist * 1.6 * scale).astype(np.float32)
    main_oct = rng.integers(0, 8, n_mp).astype(np.int32)
    mp_idx = rng.integers(0, n_mp, n_kf)
    uv = np.array([project(K.astype(np.float64) @ Tnew[:3].astype(np.float64), Xw[m]) for m in mp_idx]).reshape(-1, 2)
    uv += rng.normal(0, noise, uv.shape) if noise else 0
    kp = _keypoints(uv.astype(np.float32), np.clip(main_oct[mp_idx] + rng.integers(-3, 4, n_kf), 0, 7))
    matches = np.where(rng.random(n_kf) < 0.8, mp_idx, -1).astype(np.int32)
    mp = dict(main_measure=meas.astype(np.float32), main_pose=main, main_octave=main_oct, normal=normal.astype(np.float32),
              min_dist=min_dist, max_dist=max_dist)
    return dict(kf_kp=kp, matches_idx_mp=matches, Tcw_new=Tnew, mp=mp, Tcw_table=tab, K=K, lower=LOWER_DEPTH,
                upper=UPPER_DEPTH, fx=FX)


def xyz_info_scene(n, n_pose=8, seed=0):
    rng = np.random.default_rng(seed)
    tab = pose_table(n_pose, seed)
    xyz = np.stack([rng.uniform(-3, 3, n), rng.uniform(-2, 2, n), rng.uniform(0.3, 9, n)], 1).astype(np.float32)
    if n >= 4:
        xyz[0] = [0, 0, 2]            # on the optical axis: k = 0, asin(0)/0
        xyz[1] = [0, 0, 0]
    p1 = rng.integers(0, n_pose, n).astype(np.int32)
    p2 = rng.integers(0, n_pose, n).astype(np.int32)
    if n >= 4:
        p2[2] = p1[2]                 # same pose twice: zero parallax
    return dict(xyz1=xyz, pose1=p1, pose2=p2, Tcw=tab, fx=FX)


def triangulate_scene(n, n_proj=8, seed=0, noise=0.5):
    rng = np.random.default_rng(seed)
    tab = pose_table(n_proj, seed)
    P = np.stack([(K.astype(np.float64) @ T[:3].astype(np.float64)).astype(np.float32) for T in tab])
    i1 = rng.integers(0, n_proj, n).astype(np.int32); i2 = rng.integers(0, n_proj, n).astype(np.int32)
    Xw = np.stack([rng.uniform(-2, 6, n), rng.uniform(-4, 4, n), rng.uniform(-1, 2, n)], 1)
    pt1 = np.array([project(P[a].astype(np.float64), X) for a, X in zip(i1, Xw)]).reshape(-1, 2)
    pt2 = np.array([project(P[b].astype(np.float64), X) for b, X in zip(i2, Xw)]).reshape(-1, 2)
    pt1 += rng.normal(0, noise, pt1.shape) if noise else 0
    pt2 += rng.normal(0, noise, pt2.shape) if noise else 0
    return dict(pt1=pt1.astype(np.float32), pt2=pt2.astype(np.float32), P=P, idx1=i1, idx2=i2, Xw=Xw)
