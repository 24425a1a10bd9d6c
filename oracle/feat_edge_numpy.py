"""Independent numpy restatement of the feature-graph constraint (GlobalMapper::CreateFeatEdge + Sparsifier) — TEST
INFRASTRUCTURE ONLY. It shares no code and no derivation with oracle/feat_edge_oracle.cpp: poses are 4 x 4 matrices,
rotations go through scipy.spatial.transform.Rotation, every edge Jacobian (point edges and priors alike) is a central
difference through oplus, the damped system is solved whole (poses and points together, numpy.linalg.solve; the Schur
complement of the C++ oracle is the same linear system), the marginalisation forms the dense (12 + 3N)^2 matrix the
reference allocates and solves with it, and the clamp is a real numpy.linalg.svd. tests/test_feat_edge_oracle.py holds the
C++ oracle's LM trajectory and final constraint to it.
"""
from __future__ import annotations

import numpy as np
from scipy.spatial.transform import Rotation

H_NUM = 1e-6


def skew(v):
    return np.array([[0, -v[2], v[1]], [v[2], 0, -v[0]], [-v[1], v[0], 0.0]])


def quat_vec(R):
    """toCompactQuaternion: the vector part of the unit quaternion with w >= 0."""
    q = Rotation.from_matrix(R).as_quat()
    return -q[:3] if q[3] < 0 else q[:3]


def from_mqt(d):
    """fromVectorMQT: (t, qx, qy, qz) -> 4 x 4."""
    v = np.asarray(d[3:6], float)
    n2 = v @ v
    q = np.append(v, np.sqrt(1 - n2)) if n2 <= 1 else np.append(v / np.sqrt(n2), 0.0)
    T = np.eye(4)
    T[:3, :3] = Rotation.from_quat(q).as_matrix()
    T[:3, 3] = d[:3]
    return T


def oplus(X, d):
    return X @ from_mqt(d)


def plane_motion_prior(Twc, Tbc, xrot, yrot, zinfo):
    """addVertexSE3PlaneMotion: (measurement 4 x 4, information 6 x 6)."""
    Tbc = np.asarray(Tbc, float)
    Twb = Twc @ np.linalg.inv(Tbc)
    yaw = Rotation.from_matrix(Twb[:3, :3]).as_rotvec()[2]
    P = np.eye(4)
    P[:3, :3] = Rotation.from_rotvec([0, 0, yaw]).as_matrix()
    P[:2, 3] = Twb[:2, 3]
    R, t = Tbc[:3, :3], Tbc[:3, 3]
    A = np.block([[R, skew(t) @ R], [np.zeros((3, 3)), R]])
    return P @ Tbc, A.T @ np.diag([1e-4, 1e-4, zinfo, xrot, yrot, 1e-4]) @ A


def prior_error(Zinv, X):
    E = Zinv @ X
    return np.concatenate([E[:3, 3], quat_vec(E[:3, :3])])


def edge_error(X, p, z):
    return np.linalg.inv(X)[:3] @ np.append(p, 1.0) - z


def num_jac(f, n):
    cols = []
    for i in range(n):
        d = np.zeros(n); d[i] = H_NUM
        cols.append((f(d) - f(-d)) / (2 * H_NUM))
    return np.stack(cols, axis=1)


def huber(c2, delta):
    if c2 <= delta * delta:
        return c2, 1.0
    s = np.sqrt(c2)
    return 2 * s * delta - delta * delta, delta / s


class Pair:
    def __init__(self, mode, Tcw0, Tcw1, xyz, z0, z1, info0, info1, Tbc, xrot=1e6, yrot=1e6, zinfo=1.0, delta=5.99):
        self.mode = mode
        self.X = [np.linalg.inv(np.asarray(T, np.float32).astype(float).reshape(4, 4)) for T in (Tcw0, Tcw1)]
        self.p = np.asarray(xyz, np.float32).astype(float).reshape(-1, 3)
        self.z = [np.asarray(z, np.float32).astype(float).reshape(-1, 3) for z in (z0, z1)]
        self.om = [np.asarray(o, float).reshape(-1, 3, 3) for o in (info0, info1)]
        self.free = [1] if mode == 0 else [0, 1]
        self.delta = delta
        self.prior = {}
        for k in self.free:
            Z, Om = plane_motion_prior(self.X[k], np.asarray(Tbc, np.float32).astype(float).reshape(4, 4), xrot, yrot, zinfo)
            self.prior[k] = (np.linalg.inv(Z), Om)
        self.last = (list(self.X), self.p.copy())

    def chi2(self, X, p):
        c = sum(prior_error(Zi, X[k]) @ Om @ prior_error(Zi, X[k]) for k, (Zi, Om) in self.prior.items())
        for j in range(len(p)):
            for k in (0, 1):
                e = edge_error(X[k], p[j], self.z[k][j])
                c += huber(e @ self.om[k][j] @ e, self.delta)[0]
        return c

    def build(self):
        """Dense H and b over (free poses, points)."""
        nf, N = len(self.free), len(self.p)
        n = 6 * nf + 3 * N
        H = np.zeros((n, n)); b = np.zeros(n)
        col = {k: 6 * i for i, k in enumerate(self.free)}
        for k, (Zi, Om) in self.prior.items():
            e = prior_error(Zi, self.X[k])
            J = num_jac(lambda d: prior_error(Zi, oplus(self.X[k], d)), 6)
            s = slice(col[k], col[k] + 6)
            H[s, s] += J.T @ Om @ J
            b[s] -= J.T @ Om @ e
        for j in range(N):
            sl = slice(6 * nf + 3 * j, 6 * nf + 3 * j + 3)
            for k in (0, 1):
                e = edge_error(self.X[k], self.p[j], self.z[k][j])
                W = huber(e @ self.om[k][j] @ e, self.delta)[1] * self.om[k][j]
                Jl = num_jac(lambda d: edge_error(self.X[k], self.p[j] + d, self.z[k][j]), 3)
                H[sl, sl] += Jl.T @ W @ Jl
                b[sl] -= Jl.T @ W @ e
                if k in col:
                    Jp = num_jac(lambda d: edge_error(oplus(self.X[k], d), self.p[j], self.z[k][j]), 6)
                    sp = slice(col[k], col[k] + 6)
                    H[sp, sp] += Jp.T @ W @ Jp
                    H[sp, sl] += Jp.T @ W @ Jl
                    H[sl, sp] += Jl.T @ W @ Jp
                    b[sp] -= Jp.T @ W @ e
        return H, b

    def optimize(self, iterations):
        stats = []
        lam, ni = 0.0, 2.0
        nf = len(self.free)
        for it in range(iterations):
            cur = self.chi2(self.X, self.p)
            self.last = (list(self.X), self.p.copy())
            before = cur
            H, b = self.build()
            if it == 0:
                lam, ni = 1e-5 * np.abs(np.diag(H)).max(), 2.0
            trials, accepted, rho = 0, 0, 0.0
            while True:
                Hd = H + lam * np.eye(len(b))
                try:
                    np.linalg.cholesky(Hd)
                    x = np.linalg.solve(Hd, b)
                    ok2 = True
                except np.linalg.LinAlgError:
                    ok2 = False
                temp, scale = np.finfo(float).max, 0.0
                if ok2:
                    Xt = list(self.X)
                    for i, k in enumerate(self.free):
                        Xt[k] = oplus(self.X[k], x[6 * i:6 * i + 6])
                    pt = self.p + x[6 * nf:].reshape(-1, 3)
                    temp = self.chi2(Xt, pt)
                    self.last = (Xt, pt)
                    scale = x @ (lam * x + b)
                rho = (cur - temp) / (scale + 1e-3)
                if rho > 0 and np.isfinite(temp):
                    lam *= max(1 / 3, min(1 - (2 * rho - 1) ** 3, 2 / 3)); ni = 2.0
                    cur = temp; self.X, self.p = Xt, pt; accepted = 1
                else:
                    lam *= ni; ni *= 2
                trials += 1
                if not (rho < 0 and trials < 10):
                    break
            term = int(trials == 10 or rho == 0)
            stats.append(dict(chi2_before=before, chi2_after=cur, lam=lam, trials=trials, accepted=accepted, terminate=term))
            if term:
                break
        return stats


def se3_min(T):
    return np.concatenate([T[:3, 3], quat_vec(T[:3, :3])])


def se3_from_min(v):
    w = 1 - v[3:] @ v[3:]
    q = np.append(v[3:], np.sqrt(w)) if w > 0 else np.append(-v[3:], 0.0)
    T = np.eye(4)
    T[:3, :3] = Rotation.from_quat(q).as_matrix()
    T[:3, 3] = v[:3]
    return T


def marginalize(KF, pts, z_info):
    """Sparsifier::DoMarginalizeSE3XYZ + InfoSE3 with the dense matrix. z_info[k] [N,3,3]. Returns (measure 4 x 4, info 6 x 6,
    the matrix handed to the SVD)."""
    d, N = 1e-6, len(pts)
    H = np.zeros((12 + 3 * N, 12 + 3 * N))
    f = lambda T, p: np.linalg.inv(T)[:3] @ np.append(p, 1.0)
    for j in range(N):
        for k in (0, 1):
            ref, v = f(KF[k], pts[j]), se3_min(KF[k])
            J = np.zeros((3, 9))
            for i in range(6):
                vd = v.copy(); vd[i] += d
                J[:, i] = (f(se3_from_min(vd), pts[j]) - ref) / d
            for i in range(3):
                pd = pts[j].copy(); pd[i] += d
                J[:, 6 + i] = (f(KF[k], pd) - ref) / d
            idx = np.r_[6 * k:6 * k + 6, 12 + 3 * j:12 + 3 * j + 3]
            H[np.ix_(idx, idx)] += J.T @ z_info[k][j] @ J
    H[:12, :12] += 1e-6 * np.eye(12)
    Hm = H[:12, :12] - H[:12, 12:] @ np.linalg.solve(H[12:, 12:], H[12:, :12])
    rel = lambda A, B: se3_min(np.linalg.inv(A) @ B)
    ref, v = rel(KF[0], KF[1]), [se3_min(KF[0]), se3_min(KF[1])]
    J = np.zeros((6, 12))
    for i in range(12):
        vd = v[i // 6].copy(); vd[i % 6] += d
        J[:, i] = ((rel(se3_from_min(vd), KF[1]) if i < 6 else rel(KF[0], se3_from_min(vd))) - ref) / d
    I = np.linalg.inv(J @ np.linalg.inv(Hm) @ J.T)
    I = (I + I.T) / 2
    return np.linalg.inv(KF[0]) @ KF[1], clamp_svd(I), I


def clamp_svd(I):
    U, s, Vt = np.linalg.svd(I)
    for i in range(6):
        s[i] = min(max(s[i], 1e-6), 1e4) if U[:, i] @ Vt[i] >= 0 else -1e-6
    I = U @ np.diag(s) @ Vt
    return (I + I.T) / 2


def run(mode, Tcw0, Tcw1, xyz, z0, z1, info0, info1, Tbc, iterations=(15, 30), chi2_cut=5.0, cut=True, **kw):
    """One keyframe pair: dict(stats, measure, info, outlier, X, points)."""
    pr = Pair(mode, Tcw0, Tcw1, xyz, z0, z1, info0, info1, Tbc, **kw)
    stats = pr.optimize(iterations[mode])
    N = len(pr.p)
    out = np.zeros(N, bool)
    if mode == 1 and cut:
        Xl, pl = pr.last
        for j in range(N):
            for k in (0, 1):
                e = edge_error(Xl[k], pl[j], pr.z[k][j])
                out[j] |= e @ pr.om[k][j] @ e > chi2_cut
    keep = ~out
    measure, info, pre = marginalize(pr.X, pr.p[keep], [pr.om[0][keep], pr.om[1][keep]])
    return dict(stats=stats, measure=measure, info=info, pre_clamp=pre, outlier=out, X=pr.X, points=pr.p)
