"""CPU checks of the SE(3)-XYZ window BA's restatement (oracle/se3_ba_numpy.py): the EdgeProjectXYZ2UV point Jacobian, g2o's
adjoint EdgeSE3Expmap Jacobians, the odometry information permutation, and the recovery of noise-free windows."""
from __future__ import annotations

import numpy as np
from scipy.spatial.transform import Rotation

from oracle.se3_ba_numpy import SE3, Oracle, odo_error, permute_info, proj, se3_exp
from tools import se3_window_synth as S


def five_point(f, x, h):
    J = []
    for k in range(len(x)):
        d = np.zeros(len(x)); d[k] = h
        J.append((-f(x + 2 * d) + 8 * f(x + d) - 8 * f(x - d) + f(x - 2 * d)) / (12 * h))
    return np.array(J).T


def pose(rng, scale=0.3):
    return SE3(Rotation.from_rotvec(rng.normal(0, scale, 3)).as_matrix(), rng.normal(0, 1, 3))


def test_point_jacobian_matches_central_differences():
    rng = np.random.default_rng(0)
    for _ in range(20):
        T = pose(rng)
        X = T.inv().R @ np.array([rng.uniform(-1, 1), rng.uniform(-1, 1), rng.uniform(3, 8)]) + T.inv().t
        uv = rng.uniform(100, 500, 2)
        _, _, Jl = proj(T, X, uv, 520.0, 320.0, 240.0)
        Jn = five_point(lambda x: proj(T, x, uv, 520.0, 320.0, 240.0)[0], X, 1e-4)
        assert np.abs(Jl - Jn).max() <= 1e-6 * max(1.0, np.abs(Jl).max())


def odo_jacobians_numeric(Z, Ti, Tj, h=1e-6):
    fi = lambda d: odo_error(Z, se3_exp(d) * Ti, Tj)[0]  # noqa: E731
    fj = lambda d: odo_error(Z, Ti, se3_exp(d) * Tj)[0]  # noqa: E731
    return five_point(fi, np.zeros(6), h), five_point(fj, np.zeros(6), h)


def test_expmap_edge_jacobians_exact_at_zero_error_only():
    rng = np.random.default_rng(1)
    for _ in range(10):
        Ti, Tj = pose(rng), pose(rng)
        Z = Tj * Ti.inv()  # e = log(Tj^-1 Z Ti) = 0
        e, Ji, Jj = odo_error(Z, Ti, Tj)
        assert np.abs(e).max() < 1e-12
        Ni, Nj = odo_jacobians_numeric(Z, Ti, Tj)
        assert np.abs(Ji - Ni).max() < 1e-6 and np.abs(Jj - Nj).max() < 1e-6
        # away from zero error the adjoints are g2o's approximation: they differ at first order in the error
        gaps = []
        for eps in (1e-2, 2e-2):
            Ze = se3_exp(np.full(6, eps)) * Z
            _, Ji, Jj = odo_error(Ze, Ti, Tj)
            Ni, Nj = odo_jacobians_numeric(Ze, Ti, Tj)
            gaps.append(max(np.abs(Ji - Ni).max(), np.abs(Jj - Nj).max()))
        assert gaps[0] > 1e-4 and 1.6 < gaps[1] / gaps[0] < 2.4


def test_info_permutation_matches_add_edge_se3_expmap():
    I = np.arange(36, dtype=float).reshape(6, 6)  # not symmetric, so every block's source is visible
    N = permute_info(I)
    assert np.array_equal(N[:3, :3], I[3:, 3:]) and np.array_equal(N[3:, 3:], I[:3, :3])
    assert np.array_equal(N[3:, :3], I[:3, 3:]) and np.array_equal(N[:3, 3:], I[3:, :3])
    P = np.zeros((6, 6)); P[:3, 3:] = np.eye(3); P[3:, :3] = np.eye(3)
    Sym = I + I.T
    assert np.array_equal(permute_info(Sym), P @ Sym @ P.T)


def test_noise_free_window_is_recovered_from_a_perturbed_start():
    # loadLocalGraph: the priors are measured at the start poses, so only the points start perturbed; loadLocalGraphOnlyBa
    # with two reference keyframes (which fix the monocular scale): poses and points start perturbed
    for kw, move_poses in (({}, False), (dict(with_prior=False, odometry=False, n_ref=2), True)):
        prob, w = S.window(5, 120, seed=21, outlier_frac=0.0, noise=False, **kw)
        gt = w.Tcw.copy()
        rng = np.random.default_rng(2)
        free = np.nonzero(w.fixed == 0)[0]
        if move_poses:
            for k in free:
                T = gt[k].reshape(4, 4).astype(np.float64).copy()
                T[:3, 3] += rng.normal(0, 0.01, 3)
                w.Tcw[k] = T.reshape(16).astype(np.float32)
        pts_gt = w.xyz.copy()
        w.xyz = (w.xyz + rng.normal(0, 0.02, w.xyz.shape)).astype(np.float32)
        r = Oracle(w, S.window_params(prob, iterations=20)).optimize()
        assert r["stats"][-1][1] < 1e-4 * r["stats"][0][0]
        for k in free:
            assert np.abs(r["poses"][k][4:] - gt[k].reshape(4, 4)[:3, 3]).max() < 1e-3
        # depth along a short baseline is weakly observed: hold 95 % of the points tightly
        assert np.quantile(np.abs(r["points"] - pts_gt).max(axis=1), 0.95) < 1e-4
