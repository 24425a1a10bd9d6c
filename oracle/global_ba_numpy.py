"""Independent numpy restatement of GlobalMapper::GlobalBA — TEST INFRASTRUCTURE ONLY. It shares no derivation with
oracle/global_ba_oracle.cpp: poses are 4 x 4 matrices, oplus and the priors go through scipy.spatial.transform.Rotation
(the helpers of oracle/feat_edge_numpy.py), every Jacobian is a five-point central difference through oplus, and the damped system
is solved dense with numpy.linalg.solve. Only the conversions that are the specification itself — toIsometry3D's
un-normalised Eigen quaternion and cvu::inv's float rigid inverse — are restated as the reference has them.
tests/test_global_ba_oracle.py holds the C++ oracle's LM trajectory and poses to it on small graphs.
"""
from __future__ import annotations

import numpy as np

from oracle.feat_edge_numpy import oplus, plane_motion_prior, prior_error

H_NUM = 1e-3


def num_jac(f, n):
    """Five-point central differences with step H_NUM: truncation error ~ H_NUM^4 / 30 * f^(5), rounding ~ 1e-16 / H_NUM."""
    cols = []
    for i in range(n):
        d = np.zeros(n)
        d[i] = H_NUM
        cols.append((-f(2 * d) + 8 * f(d) - 8 * f(-d) + f(-2 * d)) / (12 * H_NUM))
    return np.stack(cols, axis=1)


def eigen_quat(m):
    """Eigen Quaterniond(const Matrix3d&) as (x, y, z, w), not normalised."""
    t = m[0, 0] + m[1, 1] + m[2, 2]
    if t > 0:
        s = np.sqrt(t + 1.0)
        w, s = 0.5 * s, 0.5 / s
        return np.array([(m[2, 1] - m[1, 2]) * s, (m[0, 2] - m[2, 0]) * s, (m[1, 0] - m[0, 1]) * s, w])
    i = 0
    if m[1, 1] > m[0, 0]:
        i = 1
    if m[2, 2] > m[i, i]:
        i = 2
    j, k = (i + 1) % 3, (i + 2) % 3
    s = np.sqrt(m[i, i] - m[j, j] - m[k, k] + 1.0)
    c = np.zeros(3)
    c[i] = 0.5 * s
    s = 0.5 / s
    c[j] = (m[j, i] + m[i, j]) * s
    c[k] = (m[k, i] + m[i, k]) * s
    return np.array([c[0], c[1], c[2], (m[k, j] - m[j, k]) * s])


def quat_matrix(q):
    """Eigen toRotationMatrix of a possibly non-unit quaternion (x, y, z, w)."""
    x, y, z, w = q
    return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)],
                     [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
                     [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]])


def to_iso(T):
    """converter.cpp toIsometry3D(cv::Mat) of a float 4 x 4."""
    T = np.asarray(T, np.float32).astype(float).reshape(4, 4)
    X = np.eye(4)
    X[:3, :3] = quat_matrix(eigen_quat(T[:3, :3]))
    X[:3, 3] = T[:3, 3]
    return X


def cv_inv(T):
    """cvu::inv of a float 4 x 4: R^T and -R^T t accumulated in double, rounded to float."""
    T = np.asarray(T, np.float32).reshape(4, 4)
    out = np.eye(4, dtype=np.float32)
    R = T[:3, :3].astype(float)
    out[:3, :3] = T[:3, :3].T
    out[:3, 3] = (-(R.T @ T[:3, 3].astype(float))).astype(np.float32)
    return out


def iso_inv(X):
    out = np.eye(4)
    out[:3, :3] = X[:3, :3].T
    out[:3, 3] = -X[:3, :3].T @ X[:3, 3]
    return out


def mqt_vec(R):
    """toCompactQuaternion: Eigen's quaternion of R, normalised, with w >= 0. E's rotation is not orthogonal to double
    precision (toIsometry3D keeps the un-normalised quaternion of the float measurement), so scipy's orthogonalising
    from_matrix would answer a different question."""
    q = eigen_quat(R)
    q = q / np.linalg.norm(q)
    return -q[:3] if q[3] < 0 else q[:3]


def edge_error(Zinv, Xi, Xj):
    E = Zinv @ iso_inv(Xi) @ Xj
    return np.concatenate([E[:3, 3], mqt_vec(E[:3, :3])])


class Graph:
    def __init__(self, g, Tbc, xrot=1e6, yrot=1e6, zinfo=1.0):
        self.X = [to_iso(cv_inv(T)) for T in np.asarray(g["Tcw"], np.float32).reshape(-1, 4, 4)]
        self.free = [v for v in range(len(self.X)) if not g["fixed"][v]]
        self.edges = [(i, j, iso_inv(to_iso(Z)), np.asarray(O, np.float32).astype(float).reshape(6, 6)) for i, j, Z, O in g["edges"]]
        # addVertexSE3PlaneMotion takes Config::bTc through toSE3Quat, whose quaternion is normalised
        Tbc = np.asarray(Tbc, np.float32).astype(float).reshape(4, 4)
        q = eigen_quat(Tbc[:3, :3])
        Tbc[:3, :3] = quat_matrix(q / np.linalg.norm(q))
        self.prior = []
        for X in self.X:
            Z, Om = plane_motion_prior(X, Tbc, xrot, yrot, zinfo)
            self.prior.append((iso_inv(Z), Om))

    def chi2(self, X):
        c = 0.0
        for v, (Zi, Om) in enumerate(self.prior):
            e = prior_error(Zi, X[v])
            c += e @ Om @ e
        for i, j, Zi, Om in self.edges:
            e = edge_error(Zi, X[i], X[j])
            c += e @ Om @ e
        return c

    def build(self):
        n = 6 * len(self.free)
        idx = {v: k for k, v in enumerate(self.free)}
        H, b = np.zeros((n, n)), np.zeros(n)
        for v in self.free:
            Zi, Om = self.prior[v]
            e = prior_error(Zi, self.X[v])
            J = num_jac(lambda d: prior_error(Zi, oplus(self.X[v], d)), 6)
            s = slice(6 * idx[v], 6 * idx[v] + 6)
            H[s, s] += J.T @ Om @ J
            b[s] -= J.T @ Om @ e
        for i, j, Zi, Om in self.edges:
            e = edge_error(Zi, self.X[i], self.X[j])
            Js = {i: num_jac(lambda d: edge_error(Zi, oplus(self.X[i], d), self.X[j]), 6),
                  j: num_jac(lambda d: edge_error(Zi, self.X[i], oplus(self.X[j], d)), 6)}
            for a in (i, j):
                if a not in idx:
                    continue
                sa = slice(6 * idx[a], 6 * idx[a] + 6)
                b[sa] -= Js[a].T @ Om @ e
                for c in (i, j):
                    if c in idx:
                        sc = slice(6 * idx[c], 6 * idx[c] + 6)
                        H[sa, sc] += Js[a].T @ Om @ Js[c]
        return H, b

    def optimize(self, iterations):
        """OptimizationAlgorithmLevenberg::solve, iteration by iteration. Returns the per-iteration stats as dicts."""
        stats = []
        if not self.free:
            return stats
        cur = self.chi2(self.X)
        lam, ni = 0.0, 2.0
        for it in range(iterations):
            H, b = self.build()
            if it == 0:
                lam, ni = 1e-5 * np.max(np.abs(np.diag(H))), 2.0
            st = dict(chi2_before=cur, accepted=0)
            q = 0
            while True:
                A = H + lam * np.eye(len(b))
                try:
                    np.linalg.cholesky(A)
                    dx = np.linalg.solve(A, b)
                    Xt = list(self.X)
                    for k, v in enumerate(self.free):
                        Xt[v] = oplus(self.X[v], dx[6 * k:6 * k + 6])
                    temp, scale = self.chi2(Xt), dx @ (lam * dx + b)
                except np.linalg.LinAlgError:
                    temp, scale, Xt = np.finfo(float).max, 0.0, None
                rho = (cur - temp) / (scale + 1e-3)
                if rho > 0 and np.isfinite(temp):
                    alpha = min(1 - (2 * rho - 1) ** 3, 2 / 3)
                    lam *= max(1 / 3, alpha)
                    ni = 2.0
                    cur = temp
                    self.X = Xt
                    st["accepted"] = 1
                else:
                    lam *= ni
                    ni *= 2
                q += 1
                if not (rho < 0 and q < 10):
                    break
            st.update(chi2_after=cur, **{"lambda": lam}, rho=rho, trials=q, terminate=int(q == 10 or rho == 0))
            stats.append(st)
            if st["terminate"]:
                break
        return stats
