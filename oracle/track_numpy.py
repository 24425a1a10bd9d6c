"""numpy restatement of the host part of Track (updateFramePose with the pre-integration, needNewKF) — TEST
INFRASTRUCTURE ONLY. It checks oracle/track_oracle.cpp independently; float cos / sin come from glibc through the oracle
library's cosf / sinf, because numpy's float32 trig is not glibc's."""
from __future__ import annotations

import math

import numpy as np

from oracle import pytrack

F = np.float32


def _cos(x):
    return F(pytrack.lib().track_oracle_cosf(float(x)))


def _sin(x):
    return F(pytrack.lib().track_oracle_sinf(float(x)))


def _norm_angle(t):
    t = float(t)
    if -math.pi <= t < math.pi:
        return t
    t = t - math.floor(t / (2 * math.pi)) * 2 * math.pi
    if t >= math.pi:
        t -= 2 * math.pi
    if t < -math.pi:
        t += 2 * math.pi
    return t


def se2(x, y, th):
    return (F(x), F(y), F(_norm_angle(F(th))))


def minus(a, b):
    dx, dy = F(a[0] - b[0]), F(a[1] - b[1])
    dth = F(_norm_angle(F(a[2] - b[2])))
    c, s = _cos(b[2]), _sin(b[2])
    return se2(F(F(c * dx) + F(s * dy)), F(F(F(-s) * dx) + F(c * dy)), dth)


def mat(a):
    c, s = _cos(a[2]), _sin(a[2])
    return np.array([[c, -s, 0, a[0]], [s, c, 0, a[1]], [0, 0, 1, 0], [0, 0, 0, 1]], np.float32)


def gemm4(A, B):
    D = np.zeros((4, 4), np.float32)
    for i in range(4):
        for j in range(4):
            t = F(A[i, 0] * B[0, j])
            for k in range(1, 4):
                t = F(t + F(A[i, k] * B[k, j]))
            D[i, j] = F(float(t) * 1.0 + 0.0)
    return D


def cam(cfg, d):
    return gemm4(gemm4(np.asarray(cfg["cTb"], np.float32), mat(d)), np.asarray(cfg["bTc"], np.float32))


def pose(cfg, odom, kf_odom, last_odom, meas, cov):
    fr, kf, last = se2(*odom), se2(*kf_odom), se2(*last_odom)
    Tcr = cam(cfg, minus(kf, fr))
    ok = minus(fr, last)
    ox, oy = float(ok[0]), float(ok[1])
    meas = [float(v) for v in meas]
    c, s = math.cos(meas[2]), math.sin(meas[2])
    meas[0] += c * ox + -s * oy
    meas[1] += s * ox + c * oy
    meas[2] += float(ok[2])
    A, Bk, V = np.eye(3), np.eye(3), np.zeros((3, 3))
    A[0, 2] = c * -oy + -s * ox
    A[1, 2] = s * -oy + c * ox
    Bk[:2, :2] = [[c, -s], [s, c]]
    for k in range(3):
        V[k, k] = float(F(F(cfg["odo_noise"][k]) * F(cfg["odo_noise"][k])))
    S = np.asarray(cov, np.float64).reshape(3, 3, order="F")

    def mul(X, Y):
        R = np.zeros((3, 3))
        for i in range(3):
            for j in range(3):
                R[i, j] = X[i, 0] * Y[0, j] + (X[i, 1] * Y[1, j] + X[i, 2] * Y[2, j])
        return R
    out = mul(mul(A, S), A.T) + mul(mul(Bk, V), Bk.T)
    return Tcr, np.array(meas), out.ravel(order="F")


def decide(cfg, dframes, n_tracked_old, n_obs_mp, n_good_prl, n_inlier, odom, kf_odom, accept):
    c0 = dframes > cfg["min_frames"]
    c1 = F(n_tracked_old) <= F(F(n_obs_mp) * F(0.5))
    c2 = n_good_prl > 40
    c3 = dframes > cfg["max_frames"]
    c4 = F(n_inlier) < F(F(0.1) * F(cfg["nfeatures"])) or n_inlier < 20
    need = c0 and ((c1 and c2) or c3 or c4)
    d = minus(se2(*odom), se2(*kf_odom))
    c5 = abs(d[2]) >= F(0.0349)
    T = cam(cfg, se2(*d))
    sq = 0.0
    for k in range(3):
        sq += float(T[k, 3]) * float(T[k, 3])
    c6 = math.sqrt(sq) >= float(F(F(F(0.0523) * F(cfg["upper_depth"])) * F(0.1)))
    by_odo = c5 or c6
    need = need and by_odo
    if accept:
        return bool(need), False
    return False, bool(c0 and (c4 or c3) and by_odo)
