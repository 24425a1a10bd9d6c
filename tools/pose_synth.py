"""Seeded pose-only BA problems shaped like Localizer::DoLocalBA's graph: a camera on a planar robot (synth.default_Tbc),
map points in front of it, their keypoint observations with pixel noise and optional gross outliers, and a start pose
perturbed from the ground truth. Used by the pose-BA tests and tools/pose_ba_bench.py."""
from __future__ import annotations

import math

import numpy as np

from tools import synth

FX, CX, CY = 520.0, 320.0, 240.0
SIGMA2 = np.array([1.2 ** (2 * k) for k in range(8)], np.float32)
INV_SIGMA2 = (1.0 / SIGMA2).astype(np.float32)


def Tbc_f32():
    Rbc, tbc = synth.default_Tbc()
    T = np.eye(4); T[:3, :3] = Rbc; T[:3, 3] = tbc
    return T.astype(np.float32)


def rot(axis, th):
    c, s = math.cos(th), math.sin(th)
    i, j = [(1, 2), (2, 0), (0, 1)][axis]
    R = np.eye(3); R[i, i] = c; R[j, j] = c; R[i, j] = -s; R[j, i] = s
    return R


def planar_Tcw(x, y, yaw, roll=0.0, pitch=0.0, z=0.0):
    """Tcw = Tcb * Tbw for the body pose Twb = (x, y, z, Rz(yaw) Ry(pitch) Rx(roll)); float64 [4,4]."""
    Twb = np.eye(4); Twb[:3, :3] = rot(2, yaw) @ rot(1, pitch) @ rot(0, roll); Twb[:3, 3] = (x, y, z)
    return np.linalg.inv(Tbc_f32().astype(np.float64)) @ np.linalg.inv(Twb)


def make_problem(E, seed=0, yaw=None, noise_px=0.5, outliers=0.0, start_rot=0.01, start_trans=0.05, tilt=0.0, zero_rotation=False):
    """Returns dict(Tcw [4,4] float32 start, Tcw_gt [4,4] float64, xyz [E,3], uv [E,2], info [E] float32, octave [E])."""
    rng = np.random.default_rng(seed)
    if zero_rotation:
        gt = np.eye(4); gt[:3, 3] = rng.normal(0, 0.5, 3)
    else:
        yaw = rng.uniform(-math.pi, math.pi) if yaw is None else yaw
        gt = planar_Tcw(rng.uniform(-3, 3), rng.uniform(-3, 3), yaw)
    Twc = np.linalg.inv(gt)
    depth = rng.uniform(2.0, 12.0, E)
    u = rng.uniform(10, 630, E); v = rng.uniform(10, 470, E)
    pc = np.stack([(u - CX) / FX * depth, (v - CY) / FX * depth, depth], axis=1)
    xyz = (pc @ Twc[:3, :3].T + Twc[:3, 3]).astype(np.float32)
    pc32 = xyz.astype(np.float64) @ gt[:3, :3].T + gt[:3, 3]
    uv = np.stack([pc32[:, 0] / pc32[:, 2] * FX + CX, pc32[:, 1] / pc32[:, 2] * FX + CY], axis=1)
    uv = uv + rng.normal(0, noise_px, uv.shape) if noise_px else uv
    n_out = int(round(outliers * E))
    if n_out:
        idx = rng.choice(E, n_out, replace=False)
        uv[idx] += rng.uniform(40, 120, (n_out, 2)) * rng.choice([-1, 1], (n_out, 2))
    octave = rng.integers(0, 8, E).astype(np.int32)
    info = INV_SIGMA2[octave]
    if zero_rotation:
        start = gt.copy(); start[:3, 3] += rng.normal(0, start_trans, 3)
    else:
        d = np.eye(4)
        d[:3, :3] = rot(0, rng.normal(0, start_rot) + tilt) @ rot(1, rng.normal(0, start_rot)) @ rot(2, rng.normal(0, start_rot))
        d[:3, 3] = rng.normal(0, start_trans, 3)
        start = d @ gt
    return dict(Tcw=start.astype(np.float32), Tcw_gt=gt, xyz=xyz, uv=uv.astype(np.float32), info=info.astype(np.float32),
                octave=octave)


def batch(problems):
    """CSR concatenation: (Tcw [B,16], edge_ptr [B+1], xyz [E,3], uv [E,2], info [E])."""
    ptr = np.zeros(len(problems) + 1, np.int32)
    ptr[1:] = np.cumsum([len(p["xyz"]) for p in problems])

    def cat(key, width):
        return np.concatenate([np.asarray(p[key], np.float32).reshape(-1, width) for p in problems] + [np.zeros((0, width), np.float32)])
    return (np.stack([p["Tcw"].reshape(16) for p in problems]).astype(np.float32), ptr, cat("xyz", 3), cat("uv", 2),
            cat("info", 1).reshape(-1))
