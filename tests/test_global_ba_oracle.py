"""The global pose-graph oracle (oracle/global_ba_oracle.cpp) held to itself and to an independent restatement: EdgeSE3's
analytic Jacobians against central differences through the real oplus, the priors against the feature-graph oracle's
prior, the LM trajectory and estimates against oracle/global_ba_numpy.py, and the symbolic phase's host test."""
import os
import subprocess

import numpy as np
import pytest

from oracle import global_ba_numpy, pyfeat, pyglobal
from tools import posegraph_synth as S

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def iso12(T):
    T = np.asarray(T, float)
    return np.concatenate([T[:3, :3].ravel(), T[:3, 3]])


def pose(x, y, z, rv):
    T = np.eye(4)
    T[:3, :3] = S.rot(np.asarray(rv, float))
    T[:3, 3] = (x, y, z)
    return T


POSES = {
    "identity": (np.eye(4), np.eye(4)),
    "general": (pose(0.3, -1.2, 0.4, (0.2, -0.1, 0.7)), pose(1.1, 0.5, 0.2, (-0.3, 0.25, -0.4))),
    "yaw_plus_pi": (pose(1, 2, 0, (0, 0, np.pi - 1e-3)), pose(1.3, 2.1, 0, (0, 0, -np.pi + 2e-3))),
    "yaw_minus_pi": (pose(-1, 0.5, 0.1, (0.01, 0, -np.pi + 1e-3)), pose(-0.7, 0.6, 0.1, (0, 0.02, np.pi - 3e-3))),
}


def five_point(f, x, h=1e-5):
    cols = []
    for i in range(len(x)):
        d = np.zeros(len(x))
        d[i] = h
        cols.append((-f(x + 2 * d) + 8 * f(x + d) - 8 * f(x - d) + f(x - 2 * d)) / (12 * h))
    return np.stack(cols, 1)


@pytest.mark.parametrize("name", list(POSES))
def test_edge_se3_jacobians_match_central_differences(name):
    Xi, Xj = POSES[name]
    rng = np.random.default_rng(3)
    Z = (np.linalg.inv(Xi) @ Xj @ pose(0.02, -0.01, 0.03, (0.01, 0.02, -0.015))).astype(np.float32)
    info = S.info_matrix(rng).astype(float)
    _, e, Ji, Jj = pyglobal.edge(iso12(Xi), iso12(Xj), Z, info)
    fi = lambda d: pyglobal.edge(pyfeat.oplus(iso12(Xi), d), iso12(Xj), Z, info)[1]
    fj = lambda d: pyglobal.edge(iso12(Xi), pyfeat.oplus(iso12(Xj), d), Z, info)[1]
    np.testing.assert_allclose(Ji, five_point(fi, np.zeros(6)), atol=1e-8)
    np.testing.assert_allclose(Jj, five_point(fj, np.zeros(6)), atol=1e-8)
    chi, e2, _, _ = pyglobal.edge(iso12(Xi), iso12(Xj), Z, info)
    assert chi == pytest.approx(e2 @ info @ e2, rel=1e-12)


def test_prior_is_the_feature_graph_oracles_prior():
    """With no edges the start chi2 is the sum over every vertex, the fixed one included, of the feature-graph oracle's
    EdgeSE3Prior built and evaluated at the start pose."""
    g = S.graph(seed=4, N=6, start=(0.2, 0.1, 2.0))
    g["edges"] = []
    prm = pyglobal.params(g["Tbc"], iterations=1)
    o = pyglobal.run(g, prm)
    fprm = pyfeat.params(Tbc=g["Tbc"])
    chi = 0.0
    for T in g["Tcw"]:
        X = pyglobal.from_Tcw(T)
        _, info, e, _ = pyfeat.prior(X, X, fprm)
        chi += e @ info @ e
    assert o["stats"]["chi2_before"][0] == pytest.approx(chi, rel=1e-12)


SMALL = {
    "chain_10": dict(seed=1, N=10),
    "loop_30": dict(seed=2, N=30, kind="loop", hops=(2, 3)),
    "yaw_pi_16": dict(seed=3, N=16, kind="loop", start=(0.4, 0.2, np.pi - 0.01), hops=(2,)),
}


# The two restatements agree to 4e-8 in chi2 and 1e-7 in the estimates on these graphs, whatever the restatement's
# difference step (1e-3 and 1e-4 give the same figures), so what is left is not the numeric Jacobians: the restatement
# builds the prior and the rotations through scipy and 4 x 4 products, the C++ oracle through SE3Quat, and the float inputs'
# rotations are orthogonal only to 1e-7. The bounds sit just above that.
NUMPY_CHI2_RTOL = 1e-7
NUMPY_EST_ATOL = 2e-7


@pytest.mark.parametrize("name", list(SMALL))
def test_oracle_matches_numpy_restatement(name):
    g = S.graph(**SMALL[name])
    o = pyglobal.run(g, pyglobal.params(g["Tbc"]))
    ref = global_ba_numpy.Graph(g, g["Tbc"])
    st = ref.optimize(15)
    n = next((k for k in range(len(st)) if st[k]["chi2_before"] - st[k]["chi2_after"] < 1e-10 * st[k]["chi2_before"]), len(st))
    assert o["iterations"] >= n
    for k in range(n):
        for f in ("trials", "accepted", "terminate"):
            assert o["stats"][f][k] == st[k][f], (k, f)
        for f in ("chi2_before", "chi2_after"):
            assert o["stats"][f][k] == pytest.approx(st[k][f], rel=NUMPY_CHI2_RTOL), (k, f)
    for v, X in enumerate(ref.X):
        q = o["poses"][v]
        R = global_ba_numpy.quat_matrix(q[:4])
        np.testing.assert_allclose(R, X[:3, :3], atol=NUMPY_EST_ATOL)
        np.testing.assert_allclose(q[4:], X[:3, 3], atol=NUMPY_EST_ATOL)


def test_symbolic_phase_on_the_host(tmp_path):
    exe = str(tmp_path / "global_ba_plan_host")
    res = subprocess.run(["g++", "-O2", "-std=c++14", "-Wall", "-Werror", os.path.join(ROOT, "tests", "native", "global_ba_plan_host.cpp"),
                          "-o", exe], capture_output=True, text=True)
    assert res.returncode == 0, res.stderr
    res = subprocess.run([exe], capture_output=True, text=True)
    assert res.returncode == 0 and res.stdout.strip() == "ok", res.stdout + res.stderr


def test_oracle_spread_is_far_below_the_gpu_bounds():
    """The oracle's own spread over the GPU test scenes — its edges summed in descending order, and its factorisation in
    the reversed elimination order — stays 10x or more below the bounds tests/test_global_ba_gpu.py holds the kernel to,
    with identical trials / accepted / terminate."""
    from tests import test_global_ba_gpu as G
    worst_chi2, worst_est = 0.0, 0.0
    for name, make in G.SCENES.items():
        s = make()
        prm = pyglobal.params(s["Tbc"])
        base = pyglobal.run(s, prm)
        n = G.compared_iterations(base["stats"])
        for other in (pyglobal.run(s, prm, reverse=True), pyglobal.run(s, prm, reverse_order=True)):
            assert other["iterations"] >= n, name
            for f in ("trials", "accepted", "terminate"):
                assert np.array_equal(base["stats"][f][:n], other["stats"][f][:n]), (name, f)
            for f in ("chi2_before", "chi2_after"):
                a, b = base["stats"][f][:n], other["stats"][f][:n]
                worst_chi2 = max(worst_chi2, float(np.max(np.abs(a - b) / np.abs(a))) if n else 0.0)
            worst_est = max(worst_est, float(np.abs(base["poses"] - other["poses"]).max()))
    assert 10 * worst_chi2 <= G.CHI2_RTOL, worst_chi2
    assert 10 * worst_est <= G.EST_ATOL, worst_est


def test_failed_factorisation_after_an_infinite_chi2_keeps_the_estimate():
    """An infinite information entry on the first edge makes chi2 infinite and the system non-finite. The first trial fails
    its factorisation yet passes the rho test (rho = +inf): it counts as accepted with chi2 DBL_MAX and leaves the estimate
    as it was. The next iteration starts from that carried DBL_MAX, gets rho = 0 and terminates with NOT_PD."""
    g = S.graph(seed=1, N=10)
    i, j, m, info = g["edges"][0]
    info = np.array(info, np.float32)
    info[0, 0] = np.inf
    g["edges"][0] = (i, j, m, info)
    r = pyglobal.run(g, pyglobal.params(g["Tbc"]))
    start = pyglobal.run(g, pyglobal.params(g["Tbc"], iterations=0))
    big = np.finfo(np.float64).max
    assert r["status"] == 2 and r["iterations"] == 2 and start["iterations"] == 0
    assert [(int(s["trials"]), int(s["accepted"]), int(s["terminate"])) for s in r["stats"]] == [(1, 1, 0), (1, 0, 1)]
    assert r["stats"]["chi2_before"].tolist() == [np.inf, big] and r["stats"]["chi2_after"].tolist() == [big, big]
    assert np.array_equal(r["Tcw"], start["Tcw"]) and np.array_equal(r["poses"], start["poses"])
