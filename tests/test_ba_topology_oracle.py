"""The BA oracle on reference-shaped windows (tests/ba_cases.py) against the independent dense numpy restatement, and the
conditioning screen of every window that test_ba_paths_gpu.py holds to the strict per-step bar. CPU only.

Until these tests the oracle was pinned only on synth's forward chain with pose 0 as the only fixed pose; its transposed
odometry blocks (a < b), its free-pose indexing around fixed poses in the middle and at the tail, and its handling of
poses and landmarks without edges are what the GPU is compared against."""
import numpy as np
import pytest

from oracle import ba_numpy, pyoracle
from tests import ba_cases as bc

SMALL = {
    "reference_tail": lambda: bc.reference_tail(8, 2, 80, seed=3),
    "broken_chain": lambda: bc.broken_chain(10, 100, seed=3),
    "reversed_odometry": lambda: bc.reversed_odometry(10, 100, seed=3),
    "duplicated_odometry": lambda: bc.duplicated_odometry(10, 100, seed=3),
    "loop_closure": lambda: bc.loop_closure(5, 100, 60, seed=3),
    "sparse_extremes": lambda: bc.sparse_extremes(9, 100, seed=3),
    "dense_covisibility": lambda: bc.dense_covisibility(10, 100, seed=3),
}


def _hidx(prob):
    h = -np.ones(prob.P, int)
    free = np.flatnonzero(prob.fixed == 0)
    h[free] = np.arange(len(free))
    return h


def test_builders_have_the_advertised_topology():
    tail = SMALL["reference_tail"]()
    assert tail.fixed[-2:].all() and tail.fixed[4] == 1 and tail.fixed.sum() == 3
    assert not np.isin(tail.odo_i, [8, 9]).any() and not np.isin(tail.odo_j, [8, 9]).any()
    assert np.isin(tail.edge_pose, [8, 9]).any()                                   # the reference KFs observe landmarks
    br = SMALL["broken_chain"]()
    adj = np.eye(br.P, dtype=int)
    adj[br.odo_i, br.odo_j] = adj[br.odo_j, br.odo_i] = 1
    reach = np.linalg.matrix_power(adj, br.P) > 0
    assert len({tuple(r) for r in reach}) == 3                                     # three odometry components
    rv = SMALL["reversed_odometry"]()
    h = _hidx(rv)
    a, b = h[rv.odo_i], h[rv.odo_j]
    assert ((a > b) & (b >= 0)).any() and ((a < b) & (a >= 0)).any()               # both block orientations, free-free
    dup = SMALL["duplicated_odometry"]()
    f = dup.fixed
    assert (f[dup.odo_i] & f[dup.odo_j]).any()                                     # fixed -> fixed
    assert ((f[dup.odo_i] == 1) & (f[dup.odo_j] == 0)).any() and ((f[dup.odo_i] == 0) & (f[dup.odo_j] == 1)).any()
    pairs = [tuple(sorted(p)) for p in zip(dup.odo_i, dup.odo_j)]
    assert len(set(pairs)) < len(pairs)                                            # a parallel edge
    sp = SMALL["sparse_extremes"]()
    assert 2 not in sp.edge_pose and (sp.odo_i == 2).any()                         # odometry only
    assert sp.P - 1 not in sp.edge_pose and sp.P - 1 not in sp.odo_i and sp.P - 1 not in sp.odo_j and sp.fixed[-1] == 0
    free_obs = np.zeros(sp.L, bool); free_obs[sp.edge_point[sp.fixed[sp.edge_pose] == 0]] = True
    seen = np.zeros(sp.L, bool); seen[sp.edge_point] = True
    assert (seen & ~free_obs).any()                                                # landmarks seen by fixed poses only


@pytest.mark.parametrize("name", sorted(SMALL))
def test_oracle_schur_solve_equals_dense_full_system_solve(name):
    prob = SMALL[name]()
    o = pyoracle.BAOracle(prob)
    H, b, hidx, lidx, nf, nl = ba_numpy.build_full_system(prob, prob.poses, prob.points)
    assert nf == o.nf == (prob.fixed == 0).sum()
    lin = o.linearize()
    np.testing.assert_allclose(lin["Hpp"], H[:3 * nf, :3 * nf], rtol=1e-5, atol=1e-5 * np.abs(H).max())
    np.testing.assert_allclose(lin["bp"], b[:3 * nf], rtol=1e-5, atol=1e-5 * np.abs(b).max())
    lam = 1e-5 * np.abs(np.diag(H)).max()
    dx = np.linalg.solve(H + lam * np.eye(len(b)), b)
    ss = o.schur_solve(lam)
    assert ss["ok"] == 1
    scale = np.abs(dx).max()
    np.testing.assert_allclose(ss["dx_p"], dx[:3 * nf], rtol=0, atol=2e-5 * scale)
    act = lidx >= 0
    np.testing.assert_allclose(ss["dx_l"][act], dx[3 * nf:].reshape(-1, 3), rtol=0, atol=2e-5 * scale)
    np.testing.assert_array_equal(ss["dx_l"][~act], 0.0)


@pytest.mark.parametrize("name", sorted(SMALL))
def test_oracle_lm_trajectory_matches_numpy_restatement(name):
    prob = SMALL[name]()
    o = pyoracle.BAOracle(prob)
    n, st, tp, tl = o.optimize(5, trace=True)
    poses, points, stats = ba_numpy.lm_optimize(prob, 5)
    assert n == len(stats)
    for k in range(n):
        assert st["trials"][k] == stats[k]["trials"]
        assert st["accepted"][k] == stats[k]["accepted"]
        assert st["chi2_after"][k] == pytest.approx(stats[k]["chi2_after"], rel=1e-6)
        assert st["lambda"][k] == pytest.approx(stats[k]["lam"], rel=1e-4)
    np.testing.assert_allclose(tp[-1], poses, atol=1e-6)
    np.testing.assert_allclose(tl[-1], points, atol=1e-5)
    fixed = prob.fixed == 1
    np.testing.assert_array_equal(tp[-1][fixed], prob.poses[fixed])
    unobserved = np.ones(prob.L, bool); unobserved[prob.edge_point] = False
    np.testing.assert_array_equal(tl[-1][unobserved], prob.points[unobserved])
    if name == "sparse_extremes":                                                  # the pose without edges never moves
        np.testing.assert_array_equal(tp[:, -1], np.broadcast_to(prob.poses[-1], (n, 3)))


@pytest.mark.parametrize("name", list(bc.STRICT) + ["nonpd_twist_w10", "nonpd_band_w1"])
def test_strict_windows_are_insensitive_to_the_summation_order(name):
    """The conditioning screen: the oracle on the window and on a random edge permutation of it take the same decisions,
    and every per-step update agrees to 1e-8 relative. Only such windows can be held to the 1e-5 per-step bar on a GPU,
    whose summation order differs from the oracle's."""
    if name.startswith("nonpd_"):
        prob, iters = bc.strict(name[len("nonpd_"):])
        prob = bc.nonpd(prob)
    else:
        prob, iters = bc.strict(name)
    n1, st1, tp1, tl1 = pyoracle.BAOracle(prob).optimize(iters, trace=True)
    q = bc.edge_permuted(prob, seed=1)
    n2, st2, tp2, tl2 = pyoracle.BAOracle(q).optimize(iters, trace=True)
    assert n1 == n2
    for f in ("trials", "accepted", "terminate"):
        np.testing.assert_array_equal(st1[f], st2[f], err_msg=f)
    np.testing.assert_allclose(st1["lambda"], st2["lambda"], rtol=1e-7)
    prev_p, prev_l = prob.poses, prob.points
    for k in range(n1):                                  # each step from the first run's previous estimate
        dp1, dp2 = tp1[k] - prev_p, tp2[k] - prev_p
        dl1, dl2 = tl1[k] - prev_l, tl2[k] - prev_l
        assert np.abs(dp2 - dp1).max() <= 1e-8 * max(np.abs(dp1).max(), 1e-12), f"pose step {k}"
        assert np.abs(dl2 - dl1).max() <= 1e-8 * max(np.abs(dl1).max(), 1e-12), f"landmark step {k}"
        prev_p, prev_l = tp1[k], tl1[k]
    if name.startswith("nonpd_"):
        assert st1["trials"][0] > 1 and st1["accepted"][0] == 1
