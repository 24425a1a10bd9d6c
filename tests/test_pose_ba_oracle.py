"""Self-consistency of the pose-only BA oracle (oracle/pose_ba_oracle.cpp, Localizer::DoLocalBA's g2o graph): Jacobians
against central differences, SE3Quat exp / log on both sides of their branch points, the plane-motion prior against a
scipy construction, the LM trajectory against the independent numpy restatement, and convergence on synthetic data."""
import math
import os
import subprocess

import numpy as np
import pytest
from scipy.spatial.transform import Rotation

from oracle import pose_ba_numpy as pn
from oracle import pypose
from se2lam_b200 import build
from tools import pose_synth as ps

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DELTA = math.sqrt(5.991)


def run(p, iterations=30, delta=DELTA):
    return pypose.run(p["Tcw"], p["xyz"], p["uv"], p["info"], ps.FX, ps.CX, ps.CY, ps.Tbc_f32(), delta, iterations=iterations)


def pose_matrix(p7):
    T = np.eye(4)
    T[:3, :3] = Rotation.from_quat(p7[:4]).as_matrix(); T[:3, 3] = p7[4:]
    return T


@pytest.mark.parametrize("seed", range(4))
def test_projection_jacobian_equals_central_differences(seed):
    rng = np.random.default_rng(seed)
    pose = pypose.se3_exp(np.concatenate([rng.normal(0, 0.5, 3), rng.normal(0, 1, 3)]))
    for _ in range(5):
        xyz = pose_matrix(pose)
        pc = np.array([rng.uniform(-2, 2), rng.uniform(-2, 2), rng.uniform(2, 8)])
        X = np.linalg.solve(xyz[:3, :3], pc - xyz[:3, 3])
        uv = rng.uniform(0, 600, 2)
        _, J = pypose.edge(pose, X, uv, ps.FX, ps.CX, ps.CY)
        h = 1e-4
        Jn = np.zeros((2, 6))
        for k in range(6):
            d = np.zeros(6); d[k] = h
            ep = pypose.edge(pypose.se3_mul(pypose.se3_exp(d), pose), X, uv, ps.FX, ps.CX, ps.CY)[0]
            em = pypose.edge(pypose.se3_mul(pypose.se3_exp(-d), pose), X, uv, ps.FX, ps.CX, ps.CY)[0]
            e2p = pypose.edge(pypose.se3_mul(pypose.se3_exp(2 * d), pose), X, uv, ps.FX, ps.CX, ps.CY)[0]
            e2m = pypose.edge(pypose.se3_mul(pypose.se3_exp(-2 * d), pose), X, uv, ps.FX, ps.CX, ps.CY)[0]
            Jn[:, k] = (8 * (ep - em) - (e2p - e2m)) / (12 * h)
        assert np.abs(J - Jn).max() <= 1e-6 * np.abs(J).max()
        # and the numpy restatement's numeric Jacobian
        T = pn.Pose(pose[:4], pose[4:])
        Jp = pn.numeric_jacobian(T, X[None], uv[None], ps.FX, ps.CX, ps.CY)[0]
        assert np.abs(J - Jp).max() <= 1e-6 * np.abs(J).max()


@pytest.mark.parametrize("theta", [0.0, 1e-7, 9.9e-6, 1.01e-5, 1e-3, 0.3, 2.0, math.pi - 1e-3])
def test_exp_log_round_trip_on_both_sides_of_the_branches(theta):
    rng = np.random.default_rng(int(theta * 1e6) % 1000)
    axis = rng.normal(size=3); axis /= np.linalg.norm(axis)
    u = np.concatenate([theta * axis, rng.normal(0, 1, 3)])
    T = pypose.se3_exp(u)
    # exp agrees with the numpy restatement and with scipy's rotation vector
    assert np.abs(T - pn.exp(u).vec()).max() < 1e-14
    if theta >= 1e-5:
        assert np.abs(Rotation.from_quat(T[:4]).as_rotvec() - u[:3]).max() < 1e-12
    back = pypose.se3_log(T)
    d = 0.5 * (np.trace(pose_matrix(T)[:3, :3]) - 1)
    # g2o's branches are series: below theta = 1e-5 exp takes V = R = I + Omega + Omega^2 (first order in theta), and above
    # d = 0.99999 log takes omega = dR / 2 (third order); the round trip holds to those orders and exactly elsewhere
    rot_tol = theta ** 3 if d > 0.99999 else (1e-12 if theta < 3 else 1e-9)     # acos loses digits near pi
    trans_tol = theta * np.abs(u[3:]).max() if theta < 1e-5 else (theta ** 2 if d > 0.99999 else 1e-10) * max(1.0, np.abs(u).max())
    assert np.abs(back[:3] - u[:3]).max() <= max(rot_tol, 1e-15)
    assert np.abs(back[3:] - u[3:]).max() <= max(trans_tol, 1e-15)
    assert np.abs(back - pn.log(pn.Pose(T[:4], T[4:]))).max() < 1e-12


def test_log_branch_point():
    """d = 0.99999 is theta = acos(0.99999) ~ 4.47e-3: log is exact above the angle and within the series' theta^3 below."""
    th0 = math.acos(0.99999)
    out = []
    for th in (th0 * (1 - 1e-6), th0 * (1 + 1e-6)):
        u = np.array([0, 0, th, 0.1, 0.2, 0.3])
        out.append(pypose.se3_log(pypose.se3_exp(u)) - u)
    assert np.abs(out[0]).max() < th0 ** 3 and np.abs(out[1]).max() < 1e-12


@pytest.mark.parametrize("seed", range(5))
def test_plane_motion_prior_equals_scipy_construction(seed):
    rng = np.random.default_rng(seed)
    Tcw = ps.planar_Tcw(rng.uniform(-5, 5), rng.uniform(-5, 5), rng.uniform(-3, 3), roll=rng.normal(0, 0.05),
                        pitch=rng.normal(0, 0.05), z=rng.normal(0, 0.2)).astype(np.float32)
    pose = pypose.from_f32(Tcw)
    Tbc = ps.Tbc_f32().astype(np.float64)
    meas, info = pypose.prior(pose, ps.Tbc_f32(), 1e6, 2e6, 3.0)
    Tbw = Tbc @ pose_matrix(pose)
    yaw = Rotation.from_matrix(Tbw[:3, :3]).as_rotvec()[2]
    Tp = np.eye(4); Tp[:3, :3] = Rotation.from_rotvec([0, 0, yaw]).as_matrix(); Tp[:2, 3] = Tbw[:2, 3]
    ref = np.linalg.inv(Tbc) @ Tp
    assert np.abs(pose_matrix(meas) - ref).max() < 1e-12
    A = np.zeros((6, 6)); R, t = Tbc[:3, :3], Tbc[:3, 3]
    A[:3, :3] = R; A[3:, 3:] = R; A[3:, :3] = np.cross(np.eye(3), t) @ R                # rows e_i x t: skew(t)
    ref_info = A.T @ np.diag([1e6, 2e6, 1e-4, 1e-4, 1e-4, 3.0]) @ A
    np.testing.assert_allclose(info, ref_info, rtol=1e-12, atol=1e-6)
    assert np.array_equal(info, info.T)


def same_decisions(a, b):
    n = min(len(a), len(b))
    for k in range(n):
        if (a[k]["trials"], a[k]["accepted"], a[k]["terminate"]) != (b[k]["trials"], b[k]["accepted"], b[k]["terminate"]):
            return k
    return n


def decisive_prefix(st):
    """Leading iterations that accepted a step lowering chi2 by more than 1e-10 of it: past them LM's decisions hinge on
    rounding-level chi2 differences, where implementations summing in different orders legitimately part ways."""
    for k in range(len(st)):
        if not (st["accepted"][k] and st["chi2_before"][k] - st["chi2_after"][k] > 1e-10 * st["chi2_before"][k]):
            return k
    return len(st)


@pytest.mark.parametrize("kw", [dict(E=300, seed=1), dict(E=31, seed=5), dict(E=300, seed=2, outliers=0.2),
                                dict(E=300, seed=7, tilt=0.05), dict(E=1000, seed=3), dict(E=300, seed=9, zero_rotation=True)],
                         ids=["E300", "E31", "outliers", "tilted", "E1000", "zero_rotation"])
def test_oracle_trajectory_equals_numpy_restatement(kw):
    """Identical trials / accept / terminate over the decisive iterations, chi2 to 1e-10 and the same pose there, and the
    same result."""
    p = ps.make_problem(**kw)
    o = run(p)
    n = pn.run(p["Tcw"], p["xyz"], p["uv"], p["info"], ps.FX, ps.CX, ps.CY, ps.Tbc_f32(), DELTA)
    so = [dict(trials=s["trials"], accepted=s["accepted"], terminate=s["terminate"]) for s in o["stats"]]
    P = decisive_prefix(o["stats"])
    assert P >= 3
    assert same_decisions(so[:P], n["stats"][:P]) == P
    if P == o["iterations"]:
        assert n["iterations"] == P
    for k in range(P):
        assert abs(n["stats"][k]["chi2_after"] - o["stats"]["chi2_after"][k]) <= 1e-10 * o["stats"]["chi2_after"][k]
        assert abs(n["stats"][k]["lambda_"] - o["stats"]["lambda"][k]) <= 1e-8 * o["stats"]["lambda"][k]
        assert np.abs(n["trace"][k] - o["trace"][k]).max() <= 1e-9
    assert np.abs(n["pose"] - o["pose"]).max() < 1e-8


def test_noise_free_planar_pose_is_recovered():
    p = ps.make_problem(E=300, seed=30, noise_px=0.0, start_rot=0.02, start_trans=0.1)
    o = run(p)
    assert o["status"] == 0 and o["stats"]["chi2_after"][-1] < 1e-9 * o["stats"]["chi2_before"][0]   # float32 inputs
    np.testing.assert_allclose(o["Tcw"], p["Tcw_gt"], atol=2e-5)


def test_huber_kernel_keeps_the_pose_under_gross_outliers():
    p = ps.make_problem(E=300, seed=31, noise_px=0.5, outliers=0.2, start_rot=0.01, start_trans=0.05)
    gt = p["Tcw_gt"]
    robust = run(p)
    plain = run(p, delta=1e6)                                  # a delta no error reaches: no robust kernel
    err = lambda T: max(np.abs(T[:3, :3] - gt[:3, :3]).max(), np.abs(T[:3, 3] - gt[:3, 3]).max())
    assert err(robust["Tcw"]) < 1e-2
    assert err(plain["Tcw"]) > 10 * err(robust["Tcw"]) and err(plain["Tcw"]) > 0.05


def test_no_edges_is_reported_and_leaves_the_pose():
    p = ps.make_problem(E=0, seed=1)
    o = run(p)
    assert o["iterations"] == 0 and o["status"] == 1 and o["Tcw"].tobytes() == p["Tcw"].tobytes()


def test_localizer_ba_forwarder_compiles_and_links(tmp_path):
    build.build_lib()
    exe = str(tmp_path / "localizer_ba_demo")
    libdir = os.path.dirname(build.LIB_PATH)
    cmd = ["g++", "-O1", "-std=c++14", "-Wall", "-I", os.path.join(ROOT, "include"), "-I", os.path.join(ROOT, "tests", "native", "stub"),
           os.path.join(ROOT, "tests", "native", "localizer_ba_demo.cpp"), "-o", exe, "-L", libdir, "-lse2gpu", f"-Wl,-rpath,{libdir}"]
    res = subprocess.run(cmd, capture_output=True, text=True)
    assert res.returncode == 0, res.stderr
