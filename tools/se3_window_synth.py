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


# ---------------------------------------------------------------------------------------------------------------------
# SE(3) windows built directly, in the shapes Map::updateLocalGraph / loadLocalGraph produce (reference src/Map.cpp:285-331,
# :414-566, :568-698): an upward camera on a short arc sees a ceiling, so a point is seen by every keyframe whose image
# holds it; local keyframes come first, all with a prior, one of them fixed and not at index 0; reference keyframes come
# last, fixed and without a prior; odometry runs only from the previous keyframe of the window, with gaps.
# ---------------------------------------------------------------------------------------------------------------------
FX, CX, CY, WIDTH, HEIGHT = 520.0, 320.0, 240.0, 640, 480
MAX_OCTAVE = 7  # the deepest level of the 8-level ORB pyramid
HUBER = math.sqrt(5.991)


def up_tbc():
    """A camera looking at the ceiling: cam z -> body z, cam x -> body -x, cam y -> body -y, 0.3 m up."""
    T = np.eye(4); T[:3, :3] = np.diag([-1.0, -1.0, 1.0]); T[:3, 3] = (0.1, 0.0, 0.3)
    return T


def direct_params(iterations=10, chi2_cut=25.0):
    return params(FX, CX, CY, up_tbc(), HUBER, iterations=iterations, chi2_cut=chi2_cut)


def _rotz(a):
    c, s = math.cos(a), math.sin(a)
    return np.array([[c, -s, 0.0], [s, c, 0.0], [0.0, 0.0, 1.0]])


def _rotvec(v):
    v = np.asarray(v, float)
    th = np.linalg.norm(v)
    if th == 0:
        return np.eye(3)
    k = v / th
    K = np.array([[0, -k[2], k[1]], [k[2], 0, -k[0]], [-k[1], k[0], 0]])
    return np.eye(3) + math.sin(th) * K + (1 - math.cos(th)) * K @ K


def _se3(R, t):
    T = np.eye(4); T[:3, :3] = R; T[:3, 3] = t
    return T


def _exp_noise(rng, rot, trans):
    return _se3(_rotvec(rng.normal(0.0, rot, 3)), rng.normal(0.0, trans, 3))


def direct(seed, n_local=12, n_pt=300, *, n_ref=0, prior=True, odometry=True, yaw=0.0, arc=0.3, radius=1.0, ceiling=3.0,
           fixed_at=None, odo_gaps=(), odo_reversed=(), odo_duplicate=(), odo_antiparallel=(), n_edgeless=0, unobserved=(),
           loop=0, outlier_frac=0.05, G=None, shuffle=False, spread=0.9, odo_noise=(0.002, 0.005)):
    """One SE(3)-XYZ window; returns a Window in direct_params()'s camera.

    n_local keyframes on an arc of `arc` radians of a circle of `radius` m, heading along it; the world yaw of the arc's
    middle is `yaw`. n_pt points on a ceiling `ceiling` m up, within `spread` m of the arc's middle; each is seen by every
    keyframe whose image holds it. n_ref reference keyframes (last; fixed, no prior) near the arc see each point with
    probability 1/2. With prior (loadLocalGraph) every local keyframe has the plane-motion prior and the local keyframe at
    fixed_at (default 1) is fixed; without it (loadLocalGraphOnlyBa) there is neither prior nor odometry, and the local
    keyframe at fixed_at is fixed (default 0). odometry: a link from the previous local keyframe to each local keyframe
    but those in odo_gaps; the links into odo_reversed run backwards, those into odo_duplicate are doubled and those into
    odo_antiparallel get a second link backwards. n_edgeless points lose every edge; the local keyframes in `unobserved`
    lose theirs. loop = k > 0 makes a loop-closure window: the first k local keyframes and the rest revisit one arc (ids
    far apart, no odometry between the two), a fifth of the points (the merged ones) seen by both, the rest by one side.
    G: a 4x4 world transform applied to everything (with priors, keep it a yaw about world z). shuffle: keyframes, points,
    odometry and edges in a random order. odo_noise: the odometry's rotation and translation noise (rad, m)."""
    rng = np.random.default_rng(seed)
    Tbc = up_tbc()
    Tcb = np.linalg.inv(Tbc)
    N = n_local + n_ref
    # ground truth: body poses on the arc (a loop window revisits it), reference keyframes beside it
    gt = []
    for k in range(N):
        if k < n_local:
            i, m = (k, n_local) if not loop else ((k, loop) if k < loop else (k - loop, n_local - loop))
            a = yaw - math.pi / 2 + (i / max(m - 1, 1) - 0.5) * arc + (0.01 if loop and k >= loop else 0.0)
            p, th = radius * np.array([math.cos(a), math.sin(a)]), a + math.pi / 2
        else:
            a = yaw - math.pi / 2
            p, th = radius * np.array([math.cos(a), math.sin(a)]) + rng.uniform(-0.3, 0.3, 2), yaw + rng.uniform(-0.3, 0.3)
        gt.append(_se3(_rotz(th), [p[0], p[1], 0.0]))  # Twb
    mid = np.mean([T[:2, 3] for T in gt[:n_local]], axis=0)
    Tcw_gt = [Tcb @ np.linalg.inv(T) for T in gt]
    # points on the ceiling and their observers
    pts = np.column_stack([mid + rng.uniform(-spread, spread, (n_pt, 2)), ceiling + rng.uniform(-0.3, 0.3, n_pt)])
    side = rng.choice(3, n_pt, p=[0.4, 0.4, 0.2]) if loop else np.full(n_pt, 2)
    e_kf, e_pt, e_uv, e_w = [], [], [], []
    for j in range(n_pt):
        for k in range(N):
            if k < n_local:
                if loop and side[j] != 2 and (k < loop) != (side[j] == 0):
                    continue
            elif rng.random() < 0.5:
                continue
            pc = Tcw_gt[k][:3, :3] @ pts[j] + Tcw_gt[k][:3, 3]
            if pc[2] <= 0.5:
                continue
            uv = pc[:2] / pc[2] * FX + (CX, CY)
            if not (10 <= uv[0] < WIDTH - 10 and 10 <= uv[1] < HEIGHT - 10):
                continue
            octave = int(rng.integers(0, MAX_OCTAVE + 1))
            sigma = float(np.float32(1.2) ** octave)
            uv = uv + rng.normal(0.0, sigma, 2)
            if rng.random() < outlier_frac:
                uv = uv + rng.uniform(10, 40, 2) * rng.choice([-1.0, 1.0], 2)
            e_kf.append(k); e_pt.append(j); e_uv.append(uv); e_w.append(np.float32(1.0) / np.float32(sigma * sigma))
    e_kf, e_pt = np.array(e_kf, np.int32), np.array(e_pt, np.int32)
    keep = ~np.isin(e_kf, np.asarray(unobserved, np.int32))
    if n_edgeless:
        keep &= ~np.isin(e_pt, rng.choice(n_pt, n_edgeless, replace=False))
    # the fixed keyframes, the priors and the odometry
    fixed = np.zeros(N, np.uint8); fixed[n_local:] = 1
    fa = (1 if prior else 0) if fixed_at is None else fixed_at
    if 0 <= fa < n_local:
        fixed[fa] = 1
    pri = np.zeros(N, np.uint8)
    if prior:
        pri[:n_local] = 1
    of, ot, om = [], [], []

    def link(i, j):
        Z = _exp_noise(rng, *odo_noise) @ Tcw_gt[j] @ np.linalg.inv(Tcw_gt[i])
        of.append(i); ot.append(j); om.append(Z)

    if odometry:
        for k in range(1, n_local):
            if k in odo_gaps or k in unobserved or k - 1 in unobserved or (loop and k == loop):
                continue
            if k in odo_reversed:
                link(k, k - 1)
            else:
                link(k - 1, k)
            if k in odo_duplicate:
                link(k - 1, k)
            if k in odo_antiparallel:
                link(k, k - 1)
    # the start: free keyframes and every point perturbed (about world z only where the priors hold the plane)
    Tcw0 = []
    for k in range(N):
        T = Tcw_gt[k]
        if not fixed[k]:
            D = _se3(_rotz(rng.normal(0, 0.01)), [*rng.normal(0, 0.02, 2), 0.0]) if prior else _exp_noise(rng, 0.005, 0.02)
            T = Tcb @ np.linalg.inv(gt[k] @ D)
        Tcw0.append(T)
    depth = pts[:, 2] - 0.3
    xyz0 = pts + rng.normal(0.0, 1.0, pts.shape) * (0.03 * depth)[:, None]
    if G is not None:
        Gi = np.linalg.inv(G)
        Tcw0 = [T @ Gi for T in Tcw0]
        xyz0 = xyz0 @ G[:3, :3].T + G[:3, 3]
    w = Window(np.array(Tcw0, np.float32).reshape(N, 16), fixed, pri, xyz0.astype(np.float32), e_pt[keep], e_kf[keep],
               np.array(e_uv, np.float32).reshape(-1, 2)[keep], np.array(e_w, np.float32)[keep], of, ot,
               np.array(om, np.float32).reshape(-1, 16), np.tile(ODO_INFO.reshape(1, 36), (len(of), 1)))
    if shuffle:
        w, _ = permute(w, rng)
    return w


def permute(w, rng):
    """w with its keyframes, points, odometry links and edges in a random order; returns (window, (kf, pt, odo, edge)),
    where kf[i] is the old index of new keyframe i and so on."""
    N, O, L, E = w.sizes
    pk, pp, po, pe = rng.permutation(N), rng.permutation(L), rng.permutation(O), rng.permutation(E)
    ik, ip = np.argsort(pk).astype(np.int32), np.argsort(pp).astype(np.int32)
    w2 = Window(w.Tcw[pk], w.fixed[pk], w.prior[pk], w.xyz[pp], ip[w.edge_point[pe]], ik[w.edge_kf[pe]], w.uv[pe], w.inv_sigma2[pe],
                ik[w.odo_from[po]], ik[w.odo_to[po]], w.odo_measure[po], w.odo_info[po])
    return w2, (pk, pp, po, pe)


def yaw_G(gamma, tx=0.0, ty=0.0):
    """a world transform that keeps the plane: a yaw about world z and a shift in it"""
    return _se3(_rotz(gamma), [tx, ty, 0.0])


def aligned_G(w, k, R):
    """the world rotation under which keyframe k of w (built with G = I) has the camera rotation R"""
    Rcw = w.Tcw[k].reshape(4, 4)[:3, :3].astype(np.float64)
    return _se3(R.T @ Rcw, [0.4, -0.3, 0.2])


def n_free(w):
    """free keyframes that some edge, odometry link or prior puts in the graph"""
    active = w.prior.astype(bool).copy()
    active[w.odo_from] = True; active[w.odo_to] = True; active[w.edge_kf] = True
    return int(np.count_nonzero(active & (w.fixed == 0)))


def _only_ba_rotated(seed, R, small, **kw):
    base = dict(n_local=8 if small else 14, n_pt=40 if small else 250, n_ref=2, prior=False, odometry=False, fixed_at=-1)
    base.update(kw)
    w0 = direct(seed, **base)
    return direct(seed, G=aligned_G(w0, base["n_local"] // 2, R), **base)


def _trimmed(seed, n_items, small):
    """a window whose E + N + O is n_items: its first edges only"""
    w = direct(seed, n_local=6, n_pt=60, n_ref=1, odo_gaps=(3,))
    N, O, _, _ = w.sizes
    keep = np.zeros(len(w.edge_point), bool); keep[:n_items - N - O] = True
    return subset(w, keep)


def _points(seed, n_items, small):
    """a window whose nf + L is n_items"""
    w0 = direct(seed, n_local=4, n_pt=1, fixed_at=1)
    return direct(seed, n_local=4, n_pt=n_items - n_free(w0), fixed_at=1, spread=0.5)


# name -> (factory(small) -> Window, iterations); every window is in direct_params()'s camera. The small versions keep a
# scene's layout at a size the numpy restatement runs in seconds.
DIRECT_SCENES = {
    # loadLocalGraph: reference keyframes last, a fixed local keyframe at index 2, an odometry gap, a keyframe held only by
    # its prior, edgeless points; world yaw across 0, so the cameras' rotations lie across pi about z
    "local_graph": (lambda small: direct(31, n_local=8 if small else 14, n_pt=50 if small else 300, n_ref=3, fixed_at=2,
                                         odo_gaps=(5,), unobserved=(6,), n_edgeless=10, yaw=-0.7, G=yaw_G(0.7, 2.0, -1.0)), 10),
    # world yaw across +-pi; reversed, duplicate and antiparallel odometry
    "yaw_near_pi": (lambda small: direct(32, n_local=8 if small else 12, n_pt=50 if small else 300, n_ref=2,
                                         odo_reversed=(3,), odo_duplicate=(4,), odo_antiparallel=(6,), yaw=math.pi - 0.4,
                                         G=yaw_G(0.4, -3.0, 1.5)), 10),
    # two clusters far apart in id revisit one arc and share the merged points
    "loop_closure": (lambda small: direct(33, n_local=10 if small else 16, n_pt=60 if small else 400, loop=5 if small else 8,
                                          n_ref=2, fixed_at=3, odo_antiparallel=(2,)), 10),
    # loadLocalGraphOnlyBa under a world rotation that puts the cameras in quat_from_R's x / y branches; keyframes with no
    # edge (left out of the graph) and edgeless points
    "only_ba_x": (lambda small: _only_ba_rotated(34, _rotvec(2.95 * np.array([0.95, 0.25, 0.18]) / np.linalg.norm([0.95, 0.25, 0.18])),
                                                 small, unobserved=(2, 5), n_edgeless=8), 10),
    "only_ba_y": (lambda small: _only_ba_rotated(35, _rotvec(2.95 * np.array([0.2, 0.96, -0.2]) / np.linalg.norm([0.2, 0.96, -0.2])),
                                                 small, unobserved=(1,)), 10),
    # keyframes, points, odometry and edges in a random order
    "shuffled": (lambda small: direct(36, n_local=8 if small else 14, n_pt=50 if small else 300, n_ref=2, fixed_at=4,
                                      odo_gaps=(6,), odo_reversed=(2,), n_edgeless=5, shuffle=True), 10),
    # every free keyframe sees every point: the envelope is full and its first column has nf - 1 rows
    "dense": (lambda small: direct(37, n_local=10 if small else 50, n_pt=40 if small else 400, odo_reversed=(7,),
                                   odo_antiparallel=(4,)), 10),
    # more than 40 k edges: the natural grid is capped by the SM count
    "large": (lambda small: direct(38, n_local=12 if small else 90, n_pt=60 if small else 1700, n_ref=0 if small else 4,
                                   arc=0.4 if small else 1.3, radius=1.0 if small else 3.0, spread=0.9 if small else 2.3,
                                   odo_gaps=(5,)), 10),
    # E = 0 and L = 0: the pose graph of the priors and the odometry alone (four iterations: it has converged to rounding
    # level by the sixth)
    # noisy odometry keeps chi2 well above the rounding of the 1e6 prior informations
    "no_points": (lambda small: direct(39, n_local=6, n_pt=0, n_ref=0, odo_reversed=(2,), odo_noise=(0.03, 0.1)), 4),
    # E = 0, L > 0: every point edgeless
    "edgeless": (lambda small: direct(40, n_local=6, n_pt=30, n_edgeless=30, odo_noise=(0.03, 0.1)), 4),
    # loadLocalGraphOnlyBa with no edge: no keyframe is in the graph, no iteration runs
    "only_ba_no_edges": (lambda small: direct(41, n_local=5, n_pt=20, n_edgeless=20, prior=False, odometry=False), 10),
    # N = 1: one free keyframe with its prior, and one fixed keyframe with free points (two iterations: single-edge points
    # soon fit exactly)
    "one_kf": (lambda small: direct(42, n_local=1, n_pt=30, fixed_at=-1), 2),
    "one_kf_fixed": (lambda small: direct(43, n_local=1, n_pt=30, fixed_at=0, prior=False, odometry=False), 2),
}
for _n in (255, 256, 257):
    DIRECT_SCENES[f"items_{_n}"] = ((lambda n: lambda small: _trimmed(44 + n, n, small))(_n), 10)  # E + N + O
    DIRECT_SCENES[f"points_{_n}"] = ((lambda n: lambda small: _points(45 + n, n, small))(_n), 10)  # nf + L
