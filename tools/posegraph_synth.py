"""Seeded pose graphs for GlobalMapper::GlobalBA: a planar robot driven along a chain, a circle, a figure-eight or a circle
driven several times, seen through a camera mounted with a non-trivial Tbc.

* Keyframes every 0.3 m of travel (the circles are wide enough that a step turns less than 10 degrees).
* Odometry edges i -> i+1 by Track::calcOdoConstraintCam's formula from noisy SE(2) increments: measure = cTb bTb bTc, an
  information diag(1/dx^2, 1/dy^2, 1e-4, 1e-4, 1e-4, 1/dtheta^2) with d = |increment| * uncertainty + noise.
* Start poses by dead reckoning over the noisy increments, so LM has the drift to remove.
* Feature edges i -> i+h for a few hops h, and loop-closure edges where the path revisits a place: measure = the true
  relative camera pose times a small random perturbation, information Q diag(l) Q^T with l log-uniform inside InfoSE3's
  clamp range.
Everything is float32 as the reference holds it; a graph is dict(Tcw [N,4,4], fixed [N], edges [(from, to, measure [4,4],
info [6,6])], truth [N,4,4] (true Tcw), Tbc).
"""
from __future__ import annotations

import numpy as np

ODO_UNCERTAIN = (0.1, 0.1, 0.1)    # Config::ODO_X_UNCERTAIN, ODO_Y_UNCERTAIN, ODO_T_UNCERTAIN
ODO_NOISE = (0.01, 0.01, 0.005)    # Config::ODO_X_NOISE, ODO_Y_NOISE, ODO_T_NOISE


def default_Tbc():
    """A camera looking forward along the body x axis, pitched down 5 degrees, 0.3 m up and 0.1 m forward."""
    p = np.deg2rad(5.0)
    Rbc0 = np.array([[0, 0, 1], [-1, 0, 0], [0, -1, 0]], float)       # camera z -> body x, camera x -> -body y
    Rp = np.array([[np.cos(p), 0, np.sin(p)], [0, 1, 0], [-np.sin(p), 0, np.cos(p)]])
    T = np.eye(4)
    T[:3, :3] = Rp @ Rbc0
    T[:3, 3] = (0.1, 0.02, 0.3)
    return T.astype(np.float32)


def se2(x, y, th):
    c, s = np.cos(th), np.sin(th)
    T = np.eye(4)
    T[:2, :2] = [[c, -s], [s, c]]
    T[:2, 3] = (x, y)
    return T


def inv(T):
    R = T[:3, :3]
    out = np.eye(4)
    out[:3, :3] = R.T
    out[:3, 3] = -R.T @ T[:3, 3]
    return out


def rot(v):
    th = np.linalg.norm(v)
    if th < 1e-15:
        return np.eye(3)
    k = v / th
    K = np.array([[0, -k[2], k[1]], [k[2], 0, -k[0]], [-k[1], k[0], 0]])
    return np.eye(3) + np.sin(th) * K + (1 - np.cos(th)) * K @ K


def _steps(kind, N, laps):
    """Per-keyframe SE(2) increments (ds, dtheta) of the true path."""
    ds = 0.3
    if kind == "chain":
        return [(ds, 0.03 * np.sin(0.2 * i)) for i in range(N - 1)]
    if kind in ("loop", "revisit"):
        per_lap = max((N - 1) / laps, 8)
        return [(ds, 2 * np.pi / per_lap) for _ in range(N - 1)]
    if kind == "figure8":
        per_circle = max((N - 1) / (2 * laps), 8)
        out = []
        for i in range(N - 1):
            sign = 1 if int(i // per_circle) % 2 == 0 else -1
            out.append((ds, sign * 2 * np.pi / per_circle))
        return out
    raise ValueError(kind)


def info_matrix(rng, lo=1e-2, hi=1e4):
    Q, _ = np.linalg.qr(rng.normal(size=(6, 6)))
    lam = np.exp(rng.uniform(np.log(lo), np.log(hi), 6))
    M = ((Q * lam) @ Q.T).astype(np.float32)
    return (M + M.T) / np.float32(2)


def perturb(rng, T, sigma_t, sigma_r):
    D = np.eye(4)
    D[:3, :3] = rot(rng.normal(scale=sigma_r, size=3))
    D[:3, 3] = rng.normal(scale=sigma_t, size=3)
    return T @ D


def graph(seed=0, N=50, kind="chain", laps=1, hops=(2, 3, 4, 5), loop_radius=0.6, loop_every=3, odo_scale=1.0,
          meas_noise=(0.005, 0.002), start=(0.0, 0.0, 0.0), Tbc=None):
    rng = np.random.default_rng(seed)
    Tbc = default_Tbc() if Tbc is None else np.asarray(Tbc, np.float32)
    Tbc64 = Tbc.astype(np.float64)
    Tcb = inv(Tbc64)
    steps = _steps(kind, N, laps)
    Twb = [se2(*start)]
    for ds, dth in steps:
        Twb.append(Twb[-1] @ se2(ds, 0.0, dth))
    Twc = [T @ Tbc64 for T in Twb]
    edges = []
    est = [Twb[0]]
    for i, (ds, dth) in enumerate(steps):  # odometry: noisy SE(2) increments, calcOdoConstraintCam
        nx = ds + rng.normal(scale=ODO_NOISE[0] * odo_scale)
        ny = rng.normal(scale=ODO_NOISE[1] * odo_scale)
        nth = dth + rng.normal(scale=ODO_NOISE[2] * odo_scale)
        bTb = se2(nx, ny, nth)
        est.append(est[-1] @ bTb)
        d = [abs(v) * u + n for v, u, n in zip((nx, ny, nth), ODO_UNCERTAIN, ODO_NOISE)]
        info = np.diag(np.float32([1 / d[0] ** 2, 1 / d[1] ** 2, 1e-4, 1e-4, 1e-4, 1 / d[2] ** 2]))
        edges.append((i, i + 1, (Tcb @ bTb @ Tbc64).astype(np.float32), info.astype(np.float32)))

    def feat(i, j):
        Z = perturb(rng, inv(Twc[i]) @ Twc[j], *meas_noise)
        edges.append((i, j, Z.astype(np.float32), info_matrix(rng)))

    for i in range(N):
        for h in hops:
            if i + h < N:
                feat(i, i + h)
    pos = np.array([T[:2, 3] for T in Twb])
    n_loop = 0
    for j in range(N):
        for i in range(0, j - 10):
            if np.linalg.norm(pos[i] - pos[j]) < loop_radius and (i + j) % loop_every == 0:
                feat(i, j)
                n_loop += 1
    Tcw = np.array([inv(T @ Tbc64) for T in est], np.float32)
    truth = np.array([inv(T) for T in Twc], np.float32)
    fixed = np.zeros(N, np.uint8)
    fixed[0] = 1
    return dict(Tcw=Tcw, fixed=fixed, edges=edges, truth=truth, Tbc=Tbc, n_loop=n_loop)


def map_points(seed, g, M=200):
    """M map points: a main keyframe index and its camera-frame position (mViewMPs) each."""
    rng = np.random.default_rng(seed)
    N = len(g["Tcw"])
    kf = rng.integers(0, N, size=M).astype(np.int32)
    view = np.stack([rng.uniform(-2, 2, M), rng.uniform(-1, 1, M), rng.uniform(1, 8, M)], 1).astype(np.float32)
    return kf, view
