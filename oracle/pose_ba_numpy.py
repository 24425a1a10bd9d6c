"""Independent numpy restatement of the pose-only BA oracle (oracle/pose_ba_oracle.cpp) — TEST INFRASTRUCTURE ONLY.

Written separately from the C++ oracle to check it: poses are rotation matrices + translations (g2o's quaternion state is
kept only where g2o's arithmetic depends on it: normalisation after every product), the projection edge's pose Jacobian
is a central difference through exp-oplus, the prior's Jacobian is g2o's constant -I, and edge sums are vectorised.
"""
from __future__ import annotations

import math

import numpy as np


def skew(v):
    return np.array([[0.0, -v[2], v[1]], [v[2], 0.0, -v[0]], [-v[1], v[0], 0.0]])


def quat_of(R):
    """Unit quaternion (x, y, z, w) with w >= 0 of a 3x3 matrix (Eigen's branch on the trace), normalised like g2o."""
    t = np.trace(R)
    if t > 0:
        s = math.sqrt(t + 1.0)
        w = 0.5 * s; s = 0.5 / s
        q = np.array([(R[2, 1] - R[1, 2]) * s, (R[0, 2] - R[2, 0]) * s, (R[1, 0] - R[0, 1]) * s, w])
    else:
        if R[1, 1] > R[0, 0]:
            i = 1 if R[2, 2] <= R[1, 1] else 2
        else:
            i = 0 if R[2, 2] <= R[0, 0] else 2
        j, k = (i + 1) % 3, (i + 2) % 3
        s = math.sqrt(R[i, i] - R[j, j] - R[k, k] + 1.0)
        v = np.zeros(3); v[i] = 0.5 * s; s = 0.5 / s
        w = (R[k, j] - R[j, k]) * s
        v[j] = (R[j, i] + R[i, j]) * s; v[k] = (R[k, i] + R[i, k]) * s
        q = np.array([v[0], v[1], v[2], w])
    if q[3] < 0:
        q = -q
    return q / np.linalg.norm(q)


def rot_of(q):
    x, y, z, w = q
    return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)],
                     [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
                     [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]])


class Pose:
    """g2o SE3Quat as (unit quaternion, t); R is derived."""

    def __init__(self, q, t):
        self.q = np.asarray(q, float); self.t = np.asarray(t, float)

    @staticmethod
    def from_Rt(R, t):
        return Pose(quat_of(np.asarray(R, float)), t)

    @property
    def R(self):
        return rot_of(self.q)

    def __mul__(self, o):
        return Pose.from_Rt(self.R @ o.R, self.R @ o.t + self.t)

    def inv(self):
        return Pose.from_Rt(self.R.T, -(self.R.T @ self.t))

    def vec(self):
        return np.concatenate([self.q, self.t])


def exp(u):
    w, v = np.asarray(u[:3], float), np.asarray(u[3:], float)
    th = np.linalg.norm(w)
    W = skew(w)
    if th < 1e-5:
        R = np.eye(3) + W + W @ W
        V = R
    else:
        R = np.eye(3) + math.sin(th) / th * W + (1 - math.cos(th)) / th ** 2 * W @ W
        V = np.eye(3) + (1 - math.cos(th)) / th ** 2 * W + (th - math.sin(th)) / th ** 3 * W @ W
    return Pose.from_Rt(R, V @ v)


def log(T):
    R = T.R
    d = 0.5 * (np.trace(R) - 1)
    dR = np.array([R[2, 1] - R[1, 2], R[0, 2] - R[2, 0], R[1, 0] - R[0, 1]])
    if d > 0.99999:
        w = 0.5 * dR
        W = skew(w)
        Vinv = np.eye(3) - 0.5 * W + W @ W / 12.0
    else:
        th = math.acos(d)
        w = th / (2 * math.sqrt(1 - d * d)) * dR
        W = skew(w)
        Vinv = np.eye(3) - 0.5 * W + (1 - th / (2 * math.tan(th / 2))) / th ** 2 * W @ W
    return np.concatenate([w, Vinv @ T.t])


def from_f32(T):
    T = np.asarray(T, np.float32).astype(float).reshape(4, 4)
    return Pose.from_Rt(T[:3, :3], T[:3, 3])


def plane_prior(pose, Tbc, xrot=1e6, yrot=1e6, zinfo=1.0):
    """addPlaneMotionSE3Expmap: keep only the body yaw (angle * axis.z of the body rotation) and zero the body height."""
    Tbc = from_f32(Tbc)
    Tbw = Tbc * pose
    q = Tbw.q                                                  # AngleAxisd(q): angle 2 atan2(|v|, |w|), axis v / (+-|v|)
    n = np.linalg.norm(q[:3])
    yaw = 2 * math.atan2(n, abs(q[3])) * (q[2] / (n if q[3] >= 0 else -n)) if n else 0.0
    Rz = np.array([[math.cos(yaw), -math.sin(yaw), 0], [math.sin(yaw), math.cos(yaw), 0], [0, 0, 1.0]])
    meas = Tbc.inv() * Pose(quat_of(Rz), np.array([Tbw.t[0], Tbw.t[1], 0.0]))
    A = np.zeros((6, 6)); A[:3, :3] = Tbc.R; A[3:, 3:] = Tbc.R; A[3:, :3] = skew(Tbc.t) @ Tbc.R
    info = A.T @ np.diag([float(np.float32(xrot)), float(np.float32(yrot)), 1e-4, 1e-4, 1e-4, float(np.float32(zinfo))]) @ A
    info = np.triu(info) + np.triu(info, 1).T
    return meas, info


def proj_errors(T, xyz, uv, fx, cx, cy):
    pc = xyz @ T.R.T + T.t
    return uv - (pc[:, :2] / pc[:, 2:3] * fx + np.array([cx, cy]))


def numeric_jacobian(T, xyz, uv, fx, cx, cy, h=1e-3):
    """d error / d delta through exp(delta) * T by five-point central differences: [E, 2, 6]."""
    J = np.zeros((len(xyz), 2, 6))
    f = lambda d: proj_errors(exp(d) * T, xyz, uv, fx, cx, cy)
    for k in range(6):
        d = np.zeros(6); d[k] = h
        J[:, :, k] = (8 * (f(d) - f(-d)) - (f(2 * d) - f(-2 * d))) / (12 * h)
    return J


def run(Tcw, xyz, uv, info, fx, cx, cy, Tbc, delta, xrot=1e6, yrot=1e6, zinfo=1.0, iterations=30):
    """Same contract as oracle.pypose.run (stats as a list of dicts)."""
    xyz = np.asarray(xyz, np.float32).astype(float).reshape(-1, 3)
    uv = np.asarray(uv, np.float32).astype(float).reshape(-1, 2)
    w = np.asarray(info, np.float32).astype(float)
    fx, cx, cy, delta = (float(np.float32(v)) for v in (fx, cx, cy, delta))
    est = from_f32(Tcw)
    if len(xyz) == 0:
        return dict(pose=est.vec(), iterations=0, status=1, stats=[], trace=np.zeros((0, 7)))
    meas, Op = plane_prior(est, Tbc, xrot, yrot, zinfo)

    def chi2(T):
        e = proj_errors(T, xyz, uv, fx, cx, cy)
        c2 = (e * e).sum(1) * w
        rob = np.where(c2 <= delta ** 2, c2, 2 * np.sqrt(c2) * delta - delta ** 2)
        ep = log(meas * T.inv())
        return ep @ Op @ ep + rob.sum()

    stats, trace, status = [], [], 0
    lam = ni = 0.0
    for it in range(iterations):
        cur = chi2(est)
        e = proj_errors(est, xyz, uv, fx, cx, cy)
        c2 = (e * e).sum(1) * w
        rho1 = np.where(c2 <= delta ** 2, 1.0, delta / np.sqrt(np.maximum(c2, 1e-300)))
        J = numeric_jacobian(est, xyz, uv, fx, cx, cy)
        Wt = (rho1 * w)[:, None, None]
        H = Op + np.einsum("eik,eil->kl", J * Wt, J)
        ep = log(meas * est.inv())
        b = Op @ ep - np.einsum("eik,ei->k", J * Wt, e)      # J_prior = -I
        if it == 0:
            lam, ni = 1e-5 * np.abs(np.diag(H)).max(), 2.0
        q = failed = 0; acc = 0; rho = 0.0
        while True:
            A = H + lam * np.eye(6)
            try:
                L = np.linalg.cholesky(A)
                ok = True
            except np.linalg.LinAlgError:
                ok = False
            if ok:
                x = np.linalg.solve(L.T, np.linalg.solve(L, b))
                trial = exp(x) * est
                tmp = chi2(trial)
                scale = x @ (lam * x + b) + 1e-3
            else:
                failed += 1
                tmp, scale = np.finfo(float).max, 1e-3
            rho = (cur - tmp) / scale
            if rho > 0 and np.isfinite(tmp):
                lam *= max(1 / 3, min(1 - (2 * rho - 1) ** 3, 2 / 3))
                ni = 2.0; cur = tmp; est = trial; acc = 1
            else:
                lam *= ni; ni *= 2
            q += 1
            if not (rho < 0 and q < 10):
                break
        term = int(q == 10 or rho == 0)
        stats.append(dict(chi2_after=cur, lambda_=lam, trials=q, accepted=acc, terminate=term))
        trace.append(est.vec())
        if term:
            if failed == q:
                status = 2
            break
    return dict(pose=est.vec(), iterations=len(stats), status=status, stats=stats, trace=np.array(trace))
