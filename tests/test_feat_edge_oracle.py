"""Self-consistency of the feature-graph constraint oracle (oracle/feat_edge_oracle.cpp): no GPU."""
import numpy as np
import pytest

from scipy.spatial.transform import Rotation

from oracle import feat_edge_numpy as fnp
from oracle import pyfeat
from tools import featgraph_synth as S


def iso(yaw, t=(0.3, -0.2, 0.1), tilt=0.0):
    c, s = np.cos(yaw), np.sin(yaw)
    Rz = np.array([[c, -s, 0], [s, c, 0], [0, 0, 1.0]])
    ct, st = np.cos(tilt), np.sin(tilt)
    Rx = np.array([[1, 0, 0], [0, ct, -st], [0, st, ct]])
    return np.concatenate([(Rz @ Rx).ravel(), np.asarray(t, float)])


def central5(f, n, h=1e-3):
    """Five-point central differences of f at 0 along each of n coordinates."""
    cols = []
    for i in range(n):
        d = np.zeros(n); d[i] = h
        cols.append((-f(2 * d) + 8 * f(d) - 8 * f(-d) + f(-2 * d)) / (12 * h))
    return np.stack(cols, axis=1)


POSES = [iso(0.0, (0, 0, 0)), iso(0.7, tilt=0.4), iso(np.pi - 1e-3, tilt=0.1), iso(-np.pi + 1e-3)]


@pytest.mark.parametrize("X", POSES)
def test_edge_jacobians_equal_central_differences_through_oplus(X):
    p = np.array([1.5, -0.7, 4.0]); z = np.array([0.2, 0.1, 3.0])
    e, Jp, Jl = pyfeat.xyz_edge(X, p, z)
    np.testing.assert_allclose(Jp, central5(lambda d: pyfeat.xyz_edge(pyfeat.oplus(X, d), p, z)[0], 6), atol=1e-6)
    np.testing.assert_allclose(Jl, central5(lambda d: pyfeat.xyz_edge(X, p + d, z)[0], 3), atol=1e-6)


@pytest.mark.parametrize("X", POSES)
def test_prior_jacobian_equals_central_differences_through_oplus(X):
    prm = pyfeat.params(Tbc=S.TBC)
    X0 = pyfeat.oplus(X, np.array([0.05, -0.02, 0.03, 0.01, -0.02, 0.015]))   # the prior is built off another pose
    _, info, e, J = pyfeat.prior(X0, X, prm)
    np.testing.assert_allclose(J, central5(lambda d: pyfeat.prior(X0, pyfeat.oplus(X, d), prm)[2], 6), atol=1e-6)
    np.testing.assert_allclose(info, info.T, rtol=1e-12)


def test_a_planar_pose_has_zero_prior_error():
    s = S.scene(1, 12)
    prm = pyfeat.params(Tbc=s["Tbc"])
    X = pyfeat.from_Tcw(s["Tcw0"])
    meas, info, e, _ = pyfeat.prior(X, X, prm)
    np.testing.assert_allclose(e, 0, atol=1e-6)          # float Tcw: planar to float rounding
    np.testing.assert_allclose(meas, X, atol=1e-6)


def test_the_eigenvalue_form_of_the_clamp_equals_the_svd_form():
    rng = np.random.default_rng(5)
    Q, _ = np.linalg.qr(rng.standard_normal((6, 6)))
    lam = np.array([-3.0, 1e-9, 5e6, 2.0, 2.0, 40.0])     # negative, tiny, huge, repeated
    A = Q @ np.diag(lam) @ Q.T
    f = np.where(lam >= 0, np.clip(lam, 1e-6, 1e4), 1e-6)
    np.testing.assert_allclose(pyfeat.clamp(A), Q @ np.diag(f) @ Q.T, rtol=1e-9, atol=1e-9)


@pytest.mark.parametrize("mode", [0, 1])
def test_noise_free_data_gives_the_true_relative_pose(mode):
    s = S.scene(2, 40, noise=0.0)
    prm = pyfeat.params(Tbc=s["Tbc"])
    r = pyfeat.run(mode, s["Tcw0"], s["Tcw1"], s["xyz"], s["z0"], s["z1"], s["info0"], s["info1"], prm)
    assert r["status"] == 0 and r["stats"]["chi2_after"][-1] < 1e-6 * r["stats"]["chi2_before"][0]
    np.testing.assert_allclose(r["measure"], s["Tc0c1_true"], atol=1e-5)
    ev = np.linalg.eigvalsh(r["info"].astype(np.float64))
    assert ev.min() >= 0.99e-6 and ev.max() <= 1.01e4
    assert not r["outlier"].any()


def test_too_few_points_return_the_status_and_nothing_else():
    s = S.scene(3, 9)
    prm = pyfeat.params(Tbc=s["Tbc"])
    r = pyfeat.run(0, s["Tcw0"], s["Tcw1"], s["xyz"], s["z0"], s["z1"], s["info0"], s["info1"], prm)
    assert r["status"] == 1 and r["iterations"] == 0 and r["measure"] is None
    r = pyfeat.run(1, s["Tcw0"], s["Tcw1"], s["xyz"][:2], s["z0"][:2], s["z1"][:2], s["info0"][:2], s["info1"][:2], prm)
    assert r["status"] == 1 and r["measure"] is None


def test_the_fixed_keyframe_of_mode_0_never_moves():
    s = S.scene(4, 30)
    prm = pyfeat.params(Tbc=s["Tbc"])
    r = pyfeat.run(0, s["Tcw0"], s["Tcw1"], s["xyz"], s["z0"], s["z1"], s["info0"], s["info1"], prm)
    X0 = pyfeat.from_Tcw(s["Tcw0"])
    assert all(np.array_equal(r["trace"][k, 0], X0) for k in range(r["iterations"]))
    assert not np.array_equal(r["trace"][-1, 1], pyfeat.from_Tcw(s["Tcw1"]))


def rot_deg(A, B):
    return np.degrees(np.linalg.norm(Rotation.from_matrix(np.asarray(A, float)[:3, :3].T @ np.asarray(B, float)[:3, :3]).as_rotvec()))


def test_the_outlier_cut_flags_the_planted_points_and_keeps_the_constraint():
    """With the cut the constraint stays within 5 cm and 1.5 degrees of the truth; fed the same LM result without the cut
    (chi2_cut out of reach) the marginalisation keeps the planted points and the information it reports for the pair changes."""
    kw = dict(seed=32, n_points=60, noise=0.3, outlier_share=0.2, outlier_size=(0.2, 0.4))
    s = S.scene(**kw)
    args = (s["Tcw0"], s["Tcw1"], s["xyz"], s["z0"], s["z1"], s["info0"], s["info1"])
    r = pyfeat.run(1, *args, pyfeat.params(Tbc=s["Tbc"]))
    assert np.array_equal(r["outlier"] != 0, s["planted"])
    assert np.abs(r["measure"][:3, 3] - s["Tc0c1_true"][:3, 3]).max() < 0.05
    assert rot_deg(r["measure"], s["Tc0c1_true"]) < 1.5
    nocut = pyfeat.run(1, *args, pyfeat.params(Tbc=s["Tbc"], chi2_cut=1e30))
    assert not nocut["outlier"].any()
    assert np.array_equal(nocut["measure"], r["measure"])       # the cut comes after LM: the relative pose is LM's either way
    assert np.abs(nocut["Hm"] - r["Hm"]).max() > 1e-2 * np.abs(r["Hm"]).max()   # but the planted edges stay in H_marginal


def test_gross_outliers_pull_the_relative_pose_off_the_truth():
    """What the Huber kernel and the cut are up against: metre-sized outliers in a fifth of the matches leave LM, after its
    30 iterations, further than 10 cm from the true relative pose, where the 20 .. 40 cm outliers above stay within 5 cm."""
    s = S.scene(seed=1, n_points=50, outlier_share=0.2, outlier_size=(0.6, 1.2))
    r = pyfeat.run(1, s["Tcw0"], s["Tcw1"], s["xyz"], s["z0"], s["z1"], s["info0"], s["info1"], pyfeat.params(Tbc=s["Tbc"]))
    assert np.abs(r["measure"][:3, 3] - s["Tc0c1_true"][:3, 3]).max() > 0.1


@pytest.mark.parametrize("yaw", [0.3, np.pi - 1e-3, -2.0])
def test_the_prior_equals_a_scipy_rotation_construction(yaw):
    prm = pyfeat.params(Tbc=S.TBC, xrot=3e5, yrot=2e6, zinfo=7.0)
    Twb = S.se2_to_Twb(0.4, -1.1, yaw)
    Twb[:3, :3] = Twb[:3, :3] @ Rotation.from_euler("xy", [0.02, -0.015]).as_matrix()     # off the plane
    Twb[2, 3] = 0.07
    TBC = S.TBC.astype(np.float32).astype(np.float64)      # the parameter struct carries Tbc as float
    Twc = Twb @ TBC
    X = np.concatenate([Twc[:3, :3].ravel(), Twc[:3, 3]])
    meas, info, _, _ = pyfeat.prior(X, X, prm)
    rv = Rotation.from_matrix(Twb[:3, :3]).as_rotvec()
    Z = np.eye(4)
    Z[:3, :3] = Rotation.from_rotvec([0, 0, rv[2]]).as_matrix()
    Z[:2, 3] = Twb[:2, 3]
    Z = Z @ TBC
    np.testing.assert_allclose(meas[:9].reshape(3, 3), Z[:3, :3], atol=1e-12)
    np.testing.assert_allclose(meas[9:], Z[:3, 3], atol=1e-12)
    R, t = TBC[:3, :3], TBC[:3, 3]
    A = np.block([[R, fnp.skew(t) @ R], [np.zeros((3, 3)), R]])
    np.testing.assert_allclose(info, A.T @ np.diag([1e-4, 1e-4, 7.0, 3e5, 2e6, 1e-4]) @ A, rtol=1e-12, atol=1e-12)


NUMPY_SCENES = {
    "m0": (0, dict(seed=61, n_points=14, info_scale=1e-3)),
    "m1": (1, dict(seed=62, n_points=12, noise=0.3, info_scale=1e-3)),
    "m1_outliers": (1, dict(seed=32, n_points=60, noise=0.3, outlier_share=0.2, outlier_size=(0.2, 0.4))),
}


@pytest.mark.parametrize("name", sorted(NUMPY_SCENES))
def test_the_lm_trajectory_equals_the_numpy_restatement(name):
    """numeric Jacobians, the undivided damped system and scipy rotations against analytic Jacobians, the Schur complement
    and hand-written quaternions: same trials and acceptances, chi2 to 1e-6, lambda to 1e-3 (it amplifies chi2 differences
    through (2 rho - 1)^3 once steps get small), relative pose to 1e-6, same outliers."""
    mode, kw = NUMPY_SCENES[name]
    s = S.scene(**kw)
    args = (s["Tcw0"], s["Tcw1"], s["xyz"], s["z0"], s["z1"], s["info0"], s["info1"])
    a = pyfeat.run(mode, *args, pyfeat.params(Tbc=s["Tbc"]))
    b = fnp.run(mode, *args, s["Tbc"])
    st = a["stats"]
    assert len(b["stats"]) == len(st)
    assert [x["trials"] for x in b["stats"]] == list(st["trials"])
    assert [x["accepted"] for x in b["stats"]] == list(st["accepted"])
    assert [x["terminate"] for x in b["stats"]] == list(st["terminate"])
    np.testing.assert_allclose([x["chi2_before"] for x in b["stats"]], st["chi2_before"], rtol=1e-6)
    np.testing.assert_allclose([x["chi2_after"] for x in b["stats"]], st["chi2_after"], rtol=1e-6)
    np.testing.assert_allclose([x["lam"] for x in b["stats"]], st["lambda"], rtol=1e-3)
    np.testing.assert_allclose(a["measure"], b["measure"], atol=1e-6)
    assert np.array_equal(a["outlier"] != 0, b["outlier"])


@pytest.mark.parametrize("name", ["m0", "m1"])    # the pairs whose information stays below the 1e4 clamp
def test_the_marginalisation_equals_the_dense_numpy_one_on_the_same_state(name):
    """Block LDL^T, LU inverses and the Jacobi SVD clamp against the dense (12 + 3N)^2 matrix, numpy.linalg.solve / inv and
    numpy.linalg.svd, from the C++ oracle's final estimate: 1e-5 of |info| (measured 6e-7). The two full runs end 1e-8 apart
    in the poses, and that alone moves the information by percent: see DESIGN.md section 10."""
    mode, kw = NUMPY_SCENES[name]
    s = S.scene(**kw)
    a = pyfeat.run(mode, s["Tcw0"], s["Tcw1"], s["xyz"], s["z0"], s["z1"], s["info0"], s["info1"], pyfeat.params(Tbc=s["Tbc"]))
    KF = []
    for k in range(2):
        T = np.eye(4)
        T[:3, :3] = Rotation.from_quat(a["poses"][k, :4]).as_matrix()
        T[:3, 3] = a["poses"][k, 4:]
        KF.append(T)
    keep = a["outlier"] == 0
    om = [s["info0"].reshape(-1, 3, 3)[keep], s["info1"].reshape(-1, 3, 3)[keep]]
    m, I, _ = fnp.marginalize(KF, a["points"][keep], om)
    np.testing.assert_allclose(a["measure"], m, atol=1e-6)
    assert np.linalg.norm(a["info"] - I) <= 1e-5 * np.linalg.norm(I)
