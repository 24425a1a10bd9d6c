"""Seeded SE(3)-XYZ windows lifted from the SE(2)-XYZ synthetic windows (tools/synth.py), so that the SE(3) BA
(se2gpu_se3_ba) and the SE(2) BA (se2gpu_ba) see the same keyframes, points and observations: a VertexSE2 pose
(x, y, theta) of Twb becomes Tcw = Tcb * Twb^-1, an EdgeSE2XYZ becomes an EdgeProjectXYZ2UV with information xx * I, and
an odometry link i -> j gets the measurement Tcw_j Tcw_i^-1 of the ground truth and a [trans rot] information."""
from __future__ import annotations

import math

import numpy as np

from se2lam_b200.se3ba import Window, params
from tools import synth

ODO_INFO = np.diag([1e2, 1e2, 1e2, 1e3, 1e3, 1e3]).astype(np.float32)


def tbc_matrix():
    Rbc, tbc = synth.default_Tbc()
    T = np.eye(4); T[:3, :3] = Rbc; T[:3, 3] = tbc
    return T


def tcw_of(pose):
    """Tcw = Tcb * Tbw of a VertexSE2 (x, y, theta) of Twb."""
    x, y, th = pose
    c, s = math.cos(th), math.sin(th)
    Twb = np.array([[c, -s, 0, x], [s, c, 0, y], [0, 0, 1, 0], [0, 0, 0, 1.0]])
    return np.linalg.inv(tbc_matrix()) @ np.linalg.inv(Twb)


def lift(prob, with_prior=True, odometry=True, n_ref=0):
    """The Window of a BAProblem. with_prior / odometry = False give loadLocalGraphOnlyBa's graph; the first n_ref
    keyframes are made reference keyframes (fixed, no prior)."""
    N = prob.P
    Tcw = np.stack([tcw_of(p) for p in prob.poses]).astype(np.float32)
    fixed = prob.fixed.astype(np.uint8).copy()
    prior = np.full(N, 1 if with_prior else 0, np.uint8)
    fixed[:n_ref] = 1; prior[:n_ref] = 0
    of, ot, om, oi = [], [], [], []
    if odometry:
        for i, j in zip(prob.odo_i, prob.odo_j):
            if i == j or prior[i] == 0 and i < n_ref or prior[j] == 0 and j < n_ref:
                continue
            Ti, Tj = tcw_of(prob.gt_poses[i]) if prob.gt_poses is not None else tcw_of(prob.poses[i]), \
                tcw_of(prob.gt_poses[j]) if prob.gt_poses is not None else tcw_of(prob.poses[j])
            of.append(int(i)); ot.append(int(j)); om.append((Tj @ np.linalg.inv(Ti)).astype(np.float32)); oi.append(ODO_INFO)
    return Window(Tcw, fixed, prior, prob.points.astype(np.float32), prob.edge_point, prob.edge_pose, prob.uv.astype(np.float32),
                  prob.info[:, 0].astype(np.float32), of, ot, np.array(om, np.float32).reshape(-1, 16),
                  np.array(oi, np.float32).reshape(-1, 36))


def window(n_kf, n_lm, seed=42, obs_per_lm=6, outlier_frac=0.05, noise=True, **kw):
    prob = synth.ba_window(n_kf, n_lm, seed=seed, obs_per_lm=obs_per_lm, outlier_frac=outlier_frac, noise=noise)
    return prob, lift(prob, **kw)


def window_params(prob, iterations=10, chi2_cut=25.0):
    return params(prob.fx, prob.cx, prob.cy, tbc_matrix(), prob.huber_delta, iterations=iterations, chi2_cut=chi2_cut)


def subset(w, keep):
    """the window with only the edges in the boolean mask keep"""
    return Window(w.Tcw, w.fixed, w.prior, w.xyz, w.edge_point[keep], w.edge_kf[keep], w.uv[keep], w.inv_sigma2[keep],
                  w.odo_from, w.odo_to, w.odo_measure, w.odo_info)


def sparse_points(seed=7):
    """every fifth point without edges, every fifth (offset one) with a single edge"""
    prob, w = window(6, 200, seed=seed)
    keep = np.ones(len(w.edge_point), bool)
    first = {}
    for e, j in enumerate(w.edge_point):
        if j % 5 == 0:
            keep[e] = False
        elif j % 5 == 1:
            keep[e] = j not in first
            first.setdefault(j, e)
    return prob, subset(w, keep)


def all_fixed(seed=10):
    """every keyframe fixed, the points free: structure only, the fixed priors and odometry still in chi2"""
    prob, w = window(4, 50, seed=seed)
    w.fixed[:] = 1
    return prob, w


# the test scenes: name -> (window factory, iterations)
SCENES = {
    "one_free_kf": (lambda: window(2, 150, seed=1), 10),
    "no_odometry": (lambda: window(6, 200, seed=2, odometry=False), 10),
    "only_ba": (lambda: window(6, 200, seed=3, with_prior=False, odometry=False), 10),
    "reference_kfs": (lambda: window(8, 300, seed=4, n_ref=2), 10),
    "reference_kfs_only_ba": (lambda: window(8, 300, seed=5, n_ref=2, with_prior=False, odometry=False), 10),
    "gross_outliers": (lambda: window(6, 300, seed=6, outlier_frac=0.25), 10),
    "sparse_points": (sparse_points, 10),
    "all_fixed": (all_fixed, 10),
    "twenty_kf": (lambda: window(20, 2000, seed=8), 10),
    "c4": (lambda: window(50, 5000, seed=9), 10),
}
