"""An independent restatement of the SE(3)-XYZ window BA (se2gpu_se3_ba, DESIGN.md section 12) in numpy, with scipy
rotations: g2o's SE3Quat, EdgeProjectXYZ2UV, EdgeSE3Expmap and the plane-motion EdgeSE3ExpmapPrior, and
OptimizationAlgorithmLevenberg over the free keyframes and the marginalised points, solved by the Schur complement with
a dense Cholesky of the reduced system. Test infrastructure only."""
from __future__ import annotations

import numpy as np
import scipy.sparse as sp
from scipy.spatial.transform import Rotation

DBL_MAX = np.finfo(np.float64).max


def skew(v):
    return np.array([[0, -v[2], v[1]], [v[2], 0, -v[0]], [-v[1], v[0], 0]])


class SE3:
    """SE3Quat as (R, t); the rotation is re-normalised through a quaternion after every product, as g2o does."""

    def __init__(self, R, t):
        self.R = Rotation.from_matrix(R).as_matrix() if R is not None else np.eye(3)
        self.t = np.asarray(t, float).copy()

    def __mul__(self, o):
        return SE3(self.R @ o.R, self.t + self.R @ o.t)

    def inv(self):
        return SE3(self.R.T, -self.R.T @ self.t)

    def adj(self):
        A = np.zeros((6, 6))
        A[:3, :3] = self.R; A[3:, 3:] = self.R; A[3:, :3] = skew(self.t) @ self.R
        return A

    def quat_t(self):
        q = Rotation.from_matrix(self.R).as_quat()
        if q[3] < 0:
            q = -q
        return np.concatenate([q, self.t])

    @staticmethod
    def from_f32(T):
        """converter.cpp toSE3Quat: the float matrix widened, through Eigen's Quaterniond(Matrix3d), which projects a
        matrix that float rounding left slightly off SO(3) differently from scipy's from_matrix"""
        T = np.asarray(T, np.float64).reshape(4, 4)
        return SE3(Rotation.from_quat(eigen_quat(T[:3, :3])).as_matrix(), T[:3, 3])


def eigen_quat(m):
    """Eigen's Quaterniond(const Matrix3d&), (x, y, z, w) before normalisation: the w branch while the trace is positive,
    else the branch of the largest diagonal entry"""
    t = m[0, 0] + m[1, 1] + m[2, 2]
    if t > 0:
        t = np.sqrt(t + 1.0)
        w, t = 0.5 * t, 0.5 / t
        return np.array([(m[2, 1] - m[1, 2]) * t, (m[0, 2] - m[2, 0]) * t, (m[1, 0] - m[0, 1]) * t, w])
    i = 0
    if m[1, 1] > m[0, 0]:
        i = 1
    if m[2, 2] > m[i, i]:
        i = 2
    j, k = (i + 1) % 3, (i + 2) % 3
    q = np.zeros(4)
    t = np.sqrt(m[i, i] - m[j, j] - m[k, k] + 1.0)
    q[i], t = 0.5 * t, 0.5 / t
    q[3] = (m[k, j] - m[j, k]) * t
    q[j] = (m[j, i] + m[i, j]) * t
    q[k] = (m[k, i] + m[i, k]) * t
    return q


def se3_exp(u):
    w, v = u[:3], u[3:]
    th = np.linalg.norm(w)
    O = skew(w)
    if th < 1e-5:
        V = np.eye(3) + O + O @ O
    else:
        V = np.eye(3) + (1 - np.cos(th)) / th ** 2 * O + (th - np.sin(th)) / th ** 3 * O @ O
    return SE3(Rotation.from_rotvec(w).as_matrix(), V @ v)


def se3_log(T):
    w = Rotation.from_matrix(T.R).as_rotvec()
    th = np.linalg.norm(w)
    O = skew(w)
    f = 1.0 / 12.0 if th < 1e-5 else (1 - th / (2 * np.tan(th / 2))) / th ** 2
    Vinv = np.eye(3) - 0.5 * O + f * O @ O
    return np.concatenate([w, Vinv @ T.t])


def permute_info(info):
    """addEdgeSE3Expmap (src/optimizer.cpp:489-494): [trans rot] -> [rot trans], block for block."""
    I = np.asarray(info, float).reshape(6, 6)
    N = np.zeros((6, 6))
    N[:3, :3] = I[3:, 3:]; N[3:, :3] = I[:3, 3:]; N[:3, 3:] = I[3:, :3]; N[3:, 3:] = I[:3, :3]
    return N


def plane_motion_prior(T, Tbc, xrot, yrot, zinfo):
    """addPlaneMotionSE3Expmap: (measurement, information) of the prior of pose T (camera from world)."""
    Tbc = SE3.from_f32(Tbc)
    Tbw = Tbc * T
    yaw = Rotation.from_matrix(Tbw.R).as_rotvec()[2]
    m = SE3(Rotation.from_euler("z", yaw).as_matrix(), np.array([Tbw.t[0], Tbw.t[1], 0.0]))
    J = Tbc.adj()
    info = J.T @ np.diag([xrot, yrot, 1e-4, 1e-4, 1e-4, zinfo]) @ J
    return Tbc.inv() * m, info


def prior_error(meas, T):
    return se3_log(meas * T.inv())


def proj(T, X, uv, fx, cx, cy):
    """EdgeProjectXYZ2UV's error and its Jacobians: (e [2], Jpose [2,6], Jpoint [2,3])."""
    pc = T.R @ X + T.t
    x, y, z = pc
    e = np.asarray(uv, float) - (pc[:2] / z * fx + np.array([cx, cy]))
    Jp = np.array([[x * y / z ** 2 * fx, -(1 + x * x / z ** 2) * fx, y / z * fx, -fx / z, 0, x / z ** 2 * fx],
                   [(1 + y * y / z ** 2) * fx, -x * y / z ** 2 * fx, -x / z * fx, 0, -fx / z, y / z ** 2 * fx]])
    Jl = -1.0 / z * np.array([[fx, 0, -x / z * fx], [0, fx, -y / z * fx]]) @ T.R
    return e, Jp, Jl


def odo_error(Z, Ti, Tj):
    """EdgeSE3Expmap: e = log(Tj^-1 Z Ti) and g2o's Jacobians Adj(Tj^-1 Z), -Adj(Ti^-1 Z^-1)."""
    e = se3_log(Tj.inv() * Z * Ti)
    return e, (Tj.inv() * Z).adj(), -(Ti.inv() * Z.inv()).adj()


def huber(c2, delta):
    if c2 <= delta * delta:
        return c2, 1.0
    s = np.sqrt(c2)
    return 2 * s * delta - delta * delta, delta / s


class Oracle:
    """w: se2lam_b200.se3ba.Window; prm: the params (fx, cx, cy, Tbc, huber_delta, x/yrot_info, z_info, iterations,
    chi2_cut) as attributes."""

    def __init__(self, w, prm):
        self.w, self.p = w, prm
        N, O, L, E = w.sizes
        self.N, self.O, self.L, self.E = N, O, L, E
        self.T = [SE3.from_f32(w.Tcw[k]) for k in range(N)]
        self.X = w.xyz.astype(np.float64).copy()
        Tbc = np.array(prm.Tbc[:], np.float64)
        self.prior = {k: plane_motion_prior(self.T[k], Tbc, prm.xrot_info, prm.yrot_info, prm.z_info)
                      for k in range(N) if w.prior[k]}
        self.Z = [SE3.from_f32(w.odo_measure[o]) for o in range(O)]
        self.Om = [permute_info(w.odo_info[o]) for o in range(O)]
        active = np.array([bool(w.prior[k]) for k in range(N)])
        active[w.odo_from] = True; active[w.odo_to] = True; active[w.edge_kf] = True
        self.free = [k for k in range(N) if active[k] and not w.fixed[k]]
        self.fpos = {k: i for i, k in enumerate(self.free)}
        self.pts = sorted(set(int(j) for j in w.edge_point))
        self.ppos = {j: i for i, j in enumerate(self.pts)}

    def chi2(self, T, X, robust=True):
        w, p = self.w, self.p
        out = []
        for e in range(self.E):
            k, j = w.edge_kf[e], w.edge_point[e]
            r, _, _ = proj(T[k], X[j], w.uv[e], p.fx, p.cx, p.cy)
            c2 = float(r @ r) * float(w.inv_sigma2[e])
            out.append(huber(c2, p.huber_delta)[0] if robust else c2)
        if not robust:
            return np.array(out)
        s = sum(out)
        for k, (m, I) in self.prior.items():
            e = prior_error(m, T[k]); s += e @ I @ e
        for o in range(self.O):
            e, _, _ = odo_error(self.Z[o], T[self.w.odo_from[o]], T[self.w.odo_to[o]]); s += e @ self.Om[o] @ e
        return float(s)

    def linearise(self, T, X):
        w, p = self.w, self.p
        nf, nl = len(self.free), len(self.pts)
        Hpp = np.zeros((6 * nf, 6 * nf)); bp = np.zeros(6 * nf)
        Hll = np.zeros((nl, 3, 3)); bl = np.zeros((nl, 3))
        rows, cols, vals = [], [], []
        for e in range(self.E):
            k, j = int(w.edge_kf[e]), int(w.edge_point[e])
            r, Jp, Jl = proj(T[k], X[j], w.uv[e], p.fx, p.cx, p.cy)
            wt = float(w.inv_sigma2[e])
            _, rho1 = huber(float(r @ r) * wt, p.huber_delta)
            W = rho1 * wt
            q = self.ppos[j]
            Hll[q] += W * Jl.T @ Jl; bl[q] -= W * Jl.T @ r
            if k in self.fpos:
                f = self.fpos[k]
                Hpp[6 * f:6 * f + 6, 6 * f:6 * f + 6] += W * Jp.T @ Jp; bp[6 * f:6 * f + 6] -= W * Jp.T @ r
                blk = W * Jp.T @ Jl
                for a in range(6):
                    for c in range(3):
                        rows.append(6 * f + a); cols.append(3 * q + c); vals.append(blk[a, c])
        for k, (m, I) in self.prior.items():
            if k in self.fpos:
                f = self.fpos[k]
                e = prior_error(m, T[k])
                Hpp[6 * f:6 * f + 6, 6 * f:6 * f + 6] += I; bp[6 * f:6 * f + 6] += I @ e  # J = -I
        for o in range(self.O):
            i, j = int(w.odo_from[o]), int(w.odo_to[o])
            e, Ji, Jj = odo_error(self.Z[o], T[i], T[j])
            Om = self.Om[o]
            for a, Ja in ((i, Ji), (j, Jj)):
                if a not in self.fpos:
                    continue
                fa = self.fpos[a]
                bp[6 * fa:6 * fa + 6] -= Ja.T @ Om @ e
                for c, Jc in ((i, Ji), (j, Jj)):
                    if c in self.fpos:
                        fc = self.fpos[c]
                        Hpp[6 * fa:6 * fa + 6, 6 * fc:6 * fc + 6] += Ja.T @ Om @ Jc
        Hpl = sp.csr_matrix((vals, (rows, cols)), shape=(6 * nf, 3 * nl))
        return Hpp, bp, Hll, bl, Hpl

    def optimize(self, iterations=None):
        iterations = self.p.iterations if iterations is None else iterations
        T, X = list(self.T), self.X.copy()
        nf, nl = len(self.free), len(self.pts)
        if nf == 0 and self.E == 0:
            iterations = 0
        cur = self.chi2(T, X)
        stats, trace, lam, ni, last_failed, it = [], [], 0.0, 2.0, False, 0
        for it in range(iterations):
            Hpp, bp, Hll, bl, Hpl = self.linearise(T, X)
            if it == 0:
                d = [np.abs(np.diag(Hpp)).max() if nf else 0.0, np.abs(np.diagonal(Hll, axis1=1, axis2=2)).max() if nl else 0.0]
                lam, ni = 1e-5 * max(d), 2.0
            before, q, failed, accepted, rho = cur, 0, 0, 0, 0.0
            while True:
                D = np.linalg.inv(Hll + lam * np.eye(3)) if nl else np.zeros((0, 3, 3))
                Dm = sp.block_diag([sp.csr_matrix(d) for d in D], format="csr") if nl else sp.csr_matrix((0, 0))
                blv = bl.reshape(-1)
                S = Hpp + lam * np.eye(6 * nf) - (Hpl @ Dm @ Hpl.T).toarray() if nl else Hpp + lam * np.eye(6 * nf)
                rs = bp - Hpl @ (Dm @ blv) if nl else bp
                ok = True
                try:
                    Lc = np.linalg.cholesky(S) if nf else np.zeros((0, 0))
                except np.linalg.LinAlgError:
                    ok = False
                temp, scale = DBL_MAX, 0.0
                if ok:
                    dp = np.linalg.solve(Lc.T, np.linalg.solve(Lc, rs)) if nf else np.zeros(0)
                    dl = Dm @ (blv - Hpl.T @ dp) if nl else np.zeros(0)
                    Tt, Xt = list(T), X.copy()
                    for f, k in enumerate(self.free):
                        Tt[k] = se3_exp(dp[6 * f:6 * f + 6]) * T[k]
                    for q2, j in enumerate(self.pts):
                        Xt[j] = X[j] + dl[3 * q2:3 * q2 + 3]
                    scale = float(dp @ (lam * dp + bp) + dl @ (lam * dl + blv))
                    temp = self.chi2(Tt, Xt)
                else:
                    failed += 1
                    temp, scale = DBL_MAX, 0.0
                scale += 1e-3
                rho = (cur - temp) / scale
                if rho > 0 and np.isfinite(temp):
                    alpha = min(1 - (2 * rho - 1) ** 3, 2.0 / 3.0)
                    lam *= max(1.0 / 3.0, alpha); ni = 2.0; cur = temp; T, X = Tt, Xt; accepted = 1
                else:
                    lam *= ni; ni *= 2
                q += 1
                if not (rho < 0 and q < 10):
                    break
            term = q == 10 or rho == 0
            stats.append((before, cur, lam, rho, q, accepted, int(term)))
            trace.append(np.concatenate([np.concatenate([T[k].quat_t() for k in range(self.N)]), X.reshape(-1)]))
            last_failed = term and failed == q
            if term:
                it += 1
                break
        else:
            it = iterations
        raw = self.chi2(T, X, robust=False) if self.E else np.zeros(0)
        return dict(iterations=len(stats), stats=stats, trace=trace, poses=np.array([t.quat_t() for t in T]), points=X,
                    chi2=raw, outlier=raw > self.p.chi2_cut, status=2 if last_failed else 0)
