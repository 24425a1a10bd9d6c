"""Local-BA windows shaped like the reference's (Map::updateLocalGraph / loadLocalGraph) rather than like tools/synth's
default forward chain with pose 0 fixed. Every builder wraps synth.ba_window and edits its output; nothing here needs a
GPU or the oracle. Test infrastructure only."""
from __future__ import annotations

import copy
import math

import numpy as np

from tools import synth


def _copy(prob):
    q = copy.copy(prob)
    for k in ("poses", "fixed", "points", "edge_pose", "edge_point", "uv", "info", "odo_i", "odo_j", "odo_meas", "odo_info",
              "gt_poses", "gt_points"):
        v = getattr(prob, k, None)
        if v is not None:
            setattr(q, k, np.array(v, copy=True))
    return q


def _keep_edges(prob, keep):
    prob.edge_pose, prob.edge_point, prob.uv, prob.info = prob.edge_pose[keep], prob.edge_point[keep], prob.uv[keep], prob.info[keep]


def _keep_odo(prob, keep):
    prob.odo_i, prob.odo_j, prob.odo_meas, prob.odo_info = prob.odo_i[keep], prob.odo_j[keep], prob.odo_meas[keep], prob.odo_info[keep]


def _add_odo(prob, i, j, meas, info6):
    prob.odo_i = np.append(prob.odo_i, np.int32(i)).astype(np.int32)
    prob.odo_j = np.append(prob.odo_j, np.int32(j)).astype(np.int32)
    prob.odo_meas = np.vstack([prob.odo_meas, np.asarray(meas, np.float64).reshape(1, 3)])
    prob.odo_info = np.vstack([prob.odo_info, np.asarray(info6, np.float64).reshape(1, 6)])


def _info3(w):
    return np.array([[w[0], w[1], w[2]], [w[1], w[3], w[4]], [w[2], w[4], w[5]]])


def _info6(M):
    return [M[0, 0], M[0, 1], M[0, 2], M[1, 1], M[1, 2], M[2, 2]]


def _rel(gi, gj):
    """relative SE(2) of pose j in the frame of pose i (PreEdgeSE2's measurement)"""
    c, s = math.cos(gi[2]), math.sin(gi[2])
    d = gj[:2] - gi[:2]
    return np.array([c * d[0] + s * d[1], -s * d[0] + c * d[1], gj[2] - gi[2]])


def reversed_measurement(meas, info6):
    """The same constraint stated from the other end: m' = m^-1, and Omega' = A Omega A^T with A = diag(-R(m_th)^T, -1),
    the first-order map e' = A e between the two edges' errors (A is orthogonal)."""
    c, s = math.cos(meas[2]), math.sin(meas[2])
    inv = np.array([-(c * meas[0] + s * meas[1]), -(-s * meas[0] + c * meas[1]), -meas[2]])
    A = np.zeros((3, 3))
    A[:2, :2] = -np.array([[c, s], [-s, c]])
    A[2, 2] = -1.0
    return inv, _info6(A @ _info3(info6) @ A.T)


def _reorder_poses(prob, order):
    """new pose k = old pose order[k]; every edge endpoint is remapped"""
    order = np.asarray(order)
    new_of_old = np.empty(prob.P, np.int32); new_of_old[order] = np.arange(prob.P, dtype=np.int32)
    prob.poses = prob.poses[order]; prob.fixed = prob.fixed[order]
    if getattr(prob, "gt_poses", None) is not None:
        prob.gt_poses = prob.gt_poses[order]
    prob.edge_pose = new_of_old[prob.edge_pose]
    prob.odo_i = new_of_old[prob.odo_i]; prob.odo_j = new_of_old[prob.odo_j]


# ------------------------------------------------------------------------------------------------------------------------
def reference_tail(P, R, n_lm, seed=42, obs_per_lm=6, mid_fixed=True, layout="circle"):
    """P local KFs in id order, then R fixed reference KFs appended as a tail (vertex ids P .. P+R-1): the reference KFs
    are the oldest of the trajectory, observe the landmarks and carry no odometry. With mid_fixed, a second fixed pose
    sits in the middle of the local KFs (the reference fixes the KF with id 1 as well), so hidx != pose index - 1."""
    base = synth.ba_window(P + R, n_lm, seed=seed, obs_per_lm=obs_per_lm, layout=layout)
    prob = _copy(base)
    prob.fixed[:] = 0
    prob.fixed[:R] = 1                                   # the oldest R KFs become the reference KFs
    _keep_odo(prob, (prob.odo_i >= R) & (prob.odo_j >= R))
    _reorder_poses(prob, np.r_[np.arange(R, P + R), np.arange(R)])
    if mid_fixed:
        prob.fixed[P // 2] = 1
    return prob


def broken_chain(P, n_lm, seed=42, obs_per_lm=6, drop=None):
    """Forward chain with two odometry edges missing (KFs that left the covisibility set): three odometry components."""
    prob = _copy(synth.ba_window(P, n_lm, seed=seed, obs_per_lm=obs_per_lm))
    drop = drop if drop is not None else (P // 3, (2 * P) // 3)
    keep = np.ones(prob.O, bool); keep[list(drop)] = False
    _keep_odo(prob, keep)
    return prob


def reversed_odometry(P, n_lm, seed=42, obs_per_lm=6, every=2):
    """Every `every`-th odometry edge given as j -> i with its measurement and information transformed consistently, and
    a second fixed pose in the middle: the a > b branch of the odometry blocks, also next to a fixed pose."""
    prob = _copy(synth.ba_window(P, n_lm, seed=seed, obs_per_lm=obs_per_lm))
    for o in range(0, prob.O, every):
        m, w = reversed_measurement(prob.odo_meas[o], prob.odo_info[o])
        prob.odo_i[o], prob.odo_j[o] = prob.odo_j[o], prob.odo_i[o]
        prob.odo_meas[o] = m; prob.odo_info[o] = w
    prob.fixed[P // 2] = 1
    return prob


def duplicated_odometry(P, n_lm, seed=42, obs_per_lm=6):
    """A second, parallel edge on one free pair (reversed, slightly different measurement), an edge between the two fixed
    poses, and fixed <-> free edges in both directions."""
    prob = _copy(synth.ba_window(P, n_lm, seed=seed, obs_per_lm=obs_per_lm))
    rng = np.random.default_rng(seed + 1)
    mid = P // 2
    prob.fixed[mid] = 1
    gt = prob.gt_poses
    w0 = prob.odo_info[0]
    o = P // 4                                           # free pair (o, o+1)
    m, w = reversed_measurement(prob.odo_meas[o] + rng.normal(0, [0.01, 0.01, 0.005]), prob.odo_info[o])
    _add_odo(prob, o + 1, o, m, w)
    _add_odo(prob, 0, mid, _rel(gt[0], gt[mid]) + rng.normal(0, [0.01, 0.01, 0.005]), w0)          # fixed -> fixed
    m, w = reversed_measurement(_rel(gt[0], gt[1]) + rng.normal(0, [0.01, 0.01, 0.005]), w0)
    _add_odo(prob, 1, 0, m, w)                                                                       # free -> fixed
    _add_odo(prob, mid, mid + 2, _rel(gt[mid], gt[mid + 2]) + rng.normal(0, [0.01, 0.01, 0.005]), w0)  # fixed -> free
    m, w = reversed_measurement(_rel(gt[mid - 2], gt[mid]) + rng.normal(0, [0.01, 0.01, 0.005]), w0)
    _add_odo(prob, mid, mid - 2, m, w)                                                               # fixed -> free, reversed
    return prob


def loop_closure(H, n_lm, n_loop=300, seed=42, obs_per_lm=6, offset=(0.12, -0.08, 0.03)):
    """Two pose segments far apart in index, joined by `n_loop` co-observed landmarks: KFs 0..H-1 are a synth window, KFs
    H..2H-1 revisit the same places (ground truth shifted by `offset`) and re-observe the first n_loop landmarks. There is
    no odometry between the segments (the KFs in between are not in the window), so the envelope of the reduced system
    spans the whole window."""
    base = synth.ba_window(H, n_lm, seed=seed, obs_per_lm=obs_per_lm)
    prob = _copy(base)
    rng = np.random.default_rng(seed + 7)
    Rbc, tbc = synth.default_Tbc()
    Rcb = Rbc.T
    tcb = -Rcb @ tbc
    gt2 = base.gt_poses + np.asarray(offset)
    drift = np.cumsum(rng.normal(0.0, [0.02, 0.02, 0.01], (H, 3)) * 0.3, axis=0)
    init2 = (gt2 + drift + np.array([0.03, -0.02, 0.01])).astype(np.float32).astype(np.float64)
    e_pose, e_pt, e_uv, e_info = [], [], [], []
    for e in range(base.E):
        j = int(base.edge_point[e])
        if j >= n_loop:
            continue
        k = int(base.edge_pose[e])
        pose = gt2[k]
        Rcw = Rcb @ synth._rotz(-pose[2])
        lc = Rcw @ (base.gt_points[j] - np.array([pose[0], pose[1], 0.0])) + tcb
        if lc[2] <= 0.5:
            continue
        uv = np.array([prob.fx * lc[0] / lc[2] + prob.cx, prob.fx * lc[1] / lc[2] + prob.cy])
        if not (0 <= uv[0] < 640 and 0 <= uv[1] < 480):
            continue
        uv = (uv + rng.normal(0.0, 1.0, 2)).astype(np.float32).astype(np.float64)
        Om = synth.edge_information(init2[k], base.points[j], Rcb, tcb, prob.fx, 1.0)
        e_pose.append(H + k); e_pt.append(j); e_uv.append(uv); e_info.append((Om[0, 0], 0.5 * (Om[0, 1] + Om[1, 0]), Om[1, 1]))
    prob.poses = np.vstack([base.poses, init2]); prob.gt_poses = np.vstack([base.gt_poses, gt2])
    prob.fixed = np.r_[base.fixed, np.zeros(H, np.uint8)].astype(np.uint8)
    prob.edge_pose = np.r_[base.edge_pose, np.asarray(e_pose, np.int32)].astype(np.int32)
    prob.edge_point = np.r_[base.edge_point, np.asarray(e_pt, np.int32)].astype(np.int32)
    prob.uv = np.vstack([base.uv, np.asarray(e_uv).reshape(-1, 2)])
    prob.info = np.vstack([base.info, np.asarray(e_info).reshape(-1, 3)])
    oi = np.arange(H, 2 * H - 1, dtype=np.int32)
    for a in oi:                                          # odometry inside the second segment only
        _add_odo(prob, a, a + 1, _rel(gt2[a - H], gt2[a + 1 - H]) + rng.normal(0, [0.01, 0.01, 0.005]), base.odo_info[0])
    return prob


def sparse_extremes(P, n_lm, seed=42, obs_per_lm=6):
    """* pose 2 keeps its odometry but loses every EdgeSE2XYZ;
    * a second fixed pose (P // 2): the landmarks whose first observer it is keep only their fixed-pose observations;
    * one extra free pose (index P) with no edges at all: it must not move."""
    prob = _copy(synth.ba_window(P, n_lm, seed=seed, obs_per_lm=obs_per_lm))
    mid = P // 2
    prob.fixed[mid] = 1
    keep = prob.edge_pose != 2
    first = np.full(prob.L, prob.P); np.minimum.at(first, prob.edge_point, prob.edge_pose)
    only_fixed = first == mid
    keep &= ~only_fixed[prob.edge_point] | (prob.fixed[prob.edge_pose] == 1)
    _keep_edges(prob, keep)
    prob.poses = np.vstack([prob.poses, prob.poses[-1] + np.array([0.25, 0.0, 0.0])])
    prob.gt_poses = np.vstack([prob.gt_poses, prob.gt_poses[-1] + np.array([0.25, 0.0, 0.0])])
    prob.fixed = np.r_[prob.fixed, np.uint8(0)].astype(np.uint8)
    return prob


def dense_covisibility(P, n_lm, seed=42):
    """Every KF observes most landmarks (obs_per_lm = P: a landmark is seen by every KF that has it in view)."""
    return synth.ba_window(P, n_lm, seed=seed, obs_per_lm=P)


def nonpd(prob, bfac=200.0):
    """_indefinite_window's construction on any window whose odometry edge 0 joins the fixed pose 0 to a free pose: pose 0
    heading exactly 0 and an information matrix [[0, B], [B, 0]] in x, y on that edge, B = bfac * max|diag H|. The reduced
    system is not positive definite until lambda outgrows B."""
    from oracle import pyoracle
    q = _copy(prob)
    assert q.fixed[q.odo_i[0]] == 1 and q.fixed[q.odo_j[0]] == 0
    q.poses[0, 2] = 0.0
    lin = pyoracle.BAOracle(q).linearize()
    md = max(np.abs(np.diag(lin["Hpp"])).max(), np.abs(lin["Hll"][:, [0, 1, 2], [0, 1, 2]]).max())
    q.odo_info[0] = [0.0, bfac * md, 0.0, 0.0, 0.0, q.odo_info[0][5]]
    return q


def edge_permuted(prob, seed=0):
    """The same window with its XYZ and odometry edges handed over in a random order."""
    q = _copy(prob)
    rng = np.random.default_rng(seed)
    _keep_edges(q, rng.permutation(q.E))
    _keep_odo(q, rng.permutation(q.O))
    return q


# ------------------------------------------------------------------------------------------------------------------------
# Windows the GPU tests (test_ba_paths_gpu.py) hold to the strict per-step bar, with their LM iteration counts.
# test_ba_topology_oracle.py screens every one of them with the oracle alone: a random edge permutation must not move any
# per-step update by more than 1e-8 relative, otherwise the window is too ill-conditioned for that bar.
def _synth(P, obs, n_lm=1500, seed=1):
    return lambda: synth.ba_window(P, n_lm, seed=seed, obs_per_lm=obs)


STRICT = {
    # reduced-solve paths of the small-window solvers (n <= 156): twisted separator 6 / 10 / 16, w = 17 beyond the twist,
    # nf = 16 where the chain rule rejects the twist
    "twist_w6": (_synth(53, 7), 8),
    "twist_w10": (_synth(53, 11), 8),
    "twist_w16": (_synth(53, 17), 8),
    "smem_w17": (_synth(53, 18), 8),
    "chain_nf16": (_synth(17, 6), 8),
    # one generator on both sides of the shared-memory limit: nf = 52 (n = 156) and nf = 53 (n = 159)
    "smem_nf52": (_synth(53, 6), 8),
    "large_nf53": (_synth(54, 6), 8),
    # band half-width w = obs_per_lm - 1 at nf = 59; w = 11 is beyond the band solver
    **{f"band_w{w}": (_synth(60, w + 1), 8) for w in (1, 3, 4, 6, 8, 10)},
    "band_w2": (_synth(60, 3, seed=2), 8),             # seed 1 fails the conditioning screen (6e-8)
    "env_w11": (_synth(60, 12), 8),
    # nf >= 2049: comparison-sorted structure build; w = 10 at this size: the band's shared-memory budget decides p
    "sorted_w10": (lambda: reference_tail(2054, 6, 12000, seed=5, obs_per_lm=11, layout="zigzag"), 3),
    # persistent work split
    "dense_nf29": (lambda: dense_covisibility(30, 1500, seed=3), 8),
    "dense_arena": (lambda: dense_covisibility(10, 10000, seed=3), 6),
    # reference-shaped topologies
    "tail_nf23": (lambda: reference_tail(24, 4, 1500, seed=3), 8),
    "tail_nf59": (lambda: reference_tail(60, 6, 2500, seed=3), 6),
    "broken_nf29": (lambda: broken_chain(30, 1500, seed=3), 8),
    "reversed_nf28": (lambda: reversed_odometry(30, 1500, seed=3), 8),
    "duplicated_nf28": (lambda: duplicated_odometry(30, 1500, seed=3), 8),
    "loop_nf39": (lambda: loop_closure(20, 2000, 300, seed=3), 8),
    "loop_nf79": (lambda: loop_closure(40, 3000, 400, seed=3), 6),
    "sparse_nf29": (lambda: sparse_extremes(30, 1500, seed=3), 8),
}


def strict(name):
    build, iters = STRICT[name]
    return build(), iters
