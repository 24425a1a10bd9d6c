"""GPU parity of the local-BA path against the CPU oracle, through the C ABI (se2gpu_ba_*).

Bar (BASELINE.md section 4): pose / landmark updates within 1e-5 relative per LM step, identical
accept/reject decisions and lambda sequence.
"""
import copy

import numpy as np
import pytest

from oracle import pyoracle
from tools import synth
from se2lam_b200.ba import LocalBA

pytestmark = pytest.mark.gpu

REL = 1e-5
MODES = [pytest.param(1, id="multi-launch"), pytest.param(2, id="persistent")]


def rel_err(a, b):
    return np.abs(a - b).max() / max(np.abs(b).max(), 1e-30)


@pytest.mark.parametrize("cfg", ["C1", "C3", "C4"])
def test_linear_system_matches_oracle(cfg):
    prob = synth.ba_config(cfg)
    o = pyoracle.BAOracle(prob)
    lin = o.linearize()
    lam = 1e-5 * max(np.abs(np.diag(lin["Hpp"])).max(), np.abs(lin["Hll"][:, [0, 1, 2], [0, 1, 2]]).max())
    ss = o.schur_solve(lam)
    g = LocalBA.from_problem(prob)
    sysm = g.debug_system(lam)
    n = sysm["n"]
    assert n == 3 * o.nf
    assert sysm["chi2"] == pytest.approx(lin["chi2"], rel=1e-12)
    free = np.flatnonzero(prob.fixed == 0)
    for a in range(len(free)):  # diagonal blocks of Hpp (odometry off-diagonals are folded into S)
        blk = slice(3 * a, 3 * a + 3)
        np.testing.assert_allclose(sysm["Hpp"][blk, blk], lin["Hpp"][blk, blk], rtol=1e-11, atol=1e-9)
    np.testing.assert_allclose(sysm["bp"], lin["bp"], rtol=1e-10, atol=1e-8)
    np.testing.assert_allclose(sysm["Hll"], lin["Hll"], rtol=1e-11, atol=1e-9)
    np.testing.assert_allclose(sysm["bl"], lin["bl"], rtol=1e-10, atol=1e-8)
    np.testing.assert_allclose(sysm["Hpl"], lin["Hpl"], rtol=1e-11, atol=1e-9)
    tril = np.tril(np.ones((n, n), bool))
    assert rel_err(sysm["S"][tril], ss["S"][tril]) < 1e-10
    assert rel_err(sysm["bs"], ss["bs"]) < 1e-9
    assert rel_err(sysm["dx_p"], ss["dx_p"]) < REL
    assert rel_err(sysm["dx_l"], ss["dx_l"]) < REL


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("cfg,iters", [("C1", 10), ("C3", 10), ("C4", 10)])
def test_lm_trajectory_matches_oracle_per_step(cfg, iters, mode):
    prob = synth.ba_config(cfg)
    o = pyoracle.BAOracle(prob)
    n_o, st_o, tp_o, tl_o = o.optimize(iters, trace=True)
    g = LocalBA.from_problem(prob, mode=mode)
    n_g, st_g, tp_g, tl_g = g.optimize(iters, trace=True)
    assert n_g == n_o
    np.testing.assert_array_equal(st_g["trials"], st_o["trials"])
    np.testing.assert_array_equal(st_g["accepted"], st_o["accepted"])
    np.testing.assert_array_equal(st_g["terminate"], st_o["terminate"])
    np.testing.assert_allclose(st_g["lambda"], st_o["lambda"], rtol=1e-6)
    np.testing.assert_allclose(st_g["chi2_after"], st_o["chi2_after"], rtol=1e-8)
    prev_p, prev_l = prob.poses, prob.points
    for k in range(n_o):
        # per-step update parity: the step taken from the oracle's previous estimate, relative to its size
        dp_o, dp_g = tp_o[k] - prev_p, tp_g[k] - prev_p
        dl_o, dl_g = tl_o[k] - prev_l, tl_g[k] - prev_l
        assert np.abs(dp_g - dp_o).max() <= REL * max(np.abs(dp_o).max(), 1e-12), f"pose step {k}"
        assert np.abs(dl_g - dl_o).max() <= REL * max(np.abs(dl_o).max(), 1e-12), f"landmark step {k}"
        prev_p, prev_l = tp_o[k], tl_o[k]
    poses, pts = g.get()
    np.testing.assert_array_equal(poses, tp_g[-1])
    np.testing.assert_array_equal(poses[prob.fixed == 1], prob.poses[prob.fixed == 1])  # gauge


def _perturbed(n_kf, n_lm, seed, sp, sth, sl):
    prob = synth.ba_window(n_kf=n_kf, n_lm=n_lm, seed=42)
    rng = np.random.default_rng(seed)
    prob.poses = prob.poses.copy(); prob.points = prob.points.copy()
    if sp:
        prob.poses[1:, :2] += rng.normal(0, sp, (prob.P - 1, 2))
    if sth:
        prob.poses[1:, 2] += rng.normal(0, sth, prob.P - 1)
    if sl:
        prob.points += rng.normal(0, sl, prob.points.shape)
    return prob


def _assert_strict_trajectory(prob, iters, mode, need_reject=True):
    o = pyoracle.BAOracle(prob)
    n_o, st_o, tp_o, tl_o = o.optimize(iters, trace=True)
    g = LocalBA.from_problem(prob, mode=mode)
    n_g, st_g, tp_g, tl_g = g.optimize(iters, trace=True)
    if need_reject:
        assert st_o["trials"].max() > 1, "test input no longer triggers a rejected step"
    assert n_g == n_o
    np.testing.assert_array_equal(st_g["trials"], st_o["trials"])
    np.testing.assert_array_equal(st_g["accepted"], st_o["accepted"])
    np.testing.assert_array_equal(st_g["terminate"], st_o["terminate"])
    np.testing.assert_allclose(st_g["lambda"], st_o["lambda"], rtol=1e-6)
    np.testing.assert_allclose(st_g["chi2_after"], st_o["chi2_after"], rtol=1e-8)
    prev_p, prev_l = prob.poses, prob.points
    for k in range(n_o):
        dp_o, dp_g = tp_o[k] - prev_p, tp_g[k] - prev_p
        dl_o, dl_g = tl_o[k] - prev_l, tl_g[k] - prev_l
        assert np.abs(dp_g - dp_o).max() <= REL * max(np.abs(dp_o).max(), 1e-12), f"pose step {k}"
        assert np.abs(dl_g - dl_o).max(initial=0.0) <= REL * max(np.abs(dl_o).max(initial=0.0), 1e-12), f"landmark step {k}"
        prev_p, prev_l = tp_o[k], tl_o[k]
    return st_o


# Windows that REJECT steps and are still well conditioned: chosen with the oracle alone (the trajectory of each is
# insensitive to the summation order - a random edge permutation moves no per-step update by more than 3e-9 relative),
# so the strict bar applies: identical trials / accept / terminate sequence, lambda to 1e-6, every per-step update to 1e-5.
REJECTING = [
    # n_kf, n_lm, seed, sigma_xy, sigma_theta, sigma_landmark          oracle trial counts
    (10, 600, 9, 1.0, 0.3, 0.0),   # [1 1 1 1 1 1 1 1 7 2 2 2]
    (10, 600, 7, 1.0, 0.3, 0.0),   # [1 1 1 1 1 1 1 7 1 1 1 1]
    (10, 600, 2, 0.3, 0.1, 0.5),   # [1 1 1 1 1 1 1 6 1 1 1 1]
    (10, 600, 8, 1.0, 0.3, 0.0),   # [1 1 1 1 1 1 1 2 1 1 1 1]
    (20, 2000, 2, 0.0, 0.0, 1.0),  # [1 1 1 1 1 1 1 3 3 3 1 1]
    (20, 2000, 7, 0.0, 0.0, 1.0),  # [1 ... 1 2]
]


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("n_kf,n_lm,seed,sp,sth,sl", REJECTING)
def test_rejected_trials_hold_the_strict_bar(n_kf, n_lm, seed, sp, sth, sl, mode):
    """restore (pop) / nu-doubling / retry path of OptimizationAlgorithmLevenberg::solve at the full 1e-5-per-step bar."""
    _assert_strict_trajectory(_perturbed(n_kf, n_lm, seed, sp, sth, sl), 12, mode)


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("seed,sp,sl,sth", [(14, 0.5, 1.5, 0.0), (17, 1.0, 3.0, 0.2)])
def test_ill_conditioned_windows_keep_the_lm_decisions(seed, sp, sl, sth, mode):
    """Deliberately ill-conditioned windows (barely constrained landmarks amplify last-bit differences of the sums along
    the trajectory): only the LM decisions and the cost are held here; the strict bar lives in the tests above."""
    prob = synth.ba_window(n_kf=10, n_lm=400, seed=seed)
    rng = np.random.default_rng(1)
    prob.points = prob.points + rng.normal(0, sl, prob.points.shape)
    prob.poses[1:, :2] += rng.normal(0, sp, (prob.P - 1, 2))
    prob.poses[1:, 2] += rng.normal(0, sth, prob.P - 1)
    o = pyoracle.BAOracle(prob)
    n_o, st_o = o.optimize(12)
    g = LocalBA.from_problem(prob, mode=mode)
    n_g, st_g = g.optimize(12)
    assert st_o["trials"].max() > 1 and n_g == n_o
    np.testing.assert_array_equal(st_g["trials"], st_o["trials"])
    np.testing.assert_array_equal(st_g["accepted"], st_o["accepted"])
    np.testing.assert_allclose(st_g["chi2_after"], st_o["chi2_after"], rtol=5e-3)


def _indefinite_window(bfac):
    """A PreEdgeSE2 whose information matrix is indefinite ([[0,B],[B,0]] in x,y) next to a fixed pose with heading exactly
    0: it adds B to an OFF-diagonal entry of the free pose's Hessian block and nothing to any diagonal, so lambda_0 =
    1e-5 max|diag| ignores it and the reduced system is not positive definite until lambda outgrows B."""
    prob = synth.ba_window(n_kf=6, n_lm=200, seed=3)
    prob.poses = prob.poses.copy(); prob.odo_info = prob.odo_info.copy()
    prob.poses[0, 2] = 0.0
    lin = pyoracle.BAOracle(prob).linearize()
    md = max(np.abs(np.diag(lin["Hpp"])).max(), np.abs(lin["Hll"][:, [0, 1, 2], [0, 1, 2]]).max())
    prob.odo_info[0] = [0.0, bfac * md, 0.0, 0.0, 0.0, prob.odo_info[0][5]]
    return prob


@pytest.mark.parametrize("mode", MODES)
def test_non_positive_definite_trials_are_rejected_like_cholmod(mode):
    """LinearSolverCholmod::solve fails on a non-PD reduced system (`minor != n`) => the trial is rejected, lambda grows
    (x2, x4, ...) until the system is PD: B = 200 max|diag| keeps trials 1-7 non-PD, trial 8 succeeds; later iterations
    shrink lambda below B again and are rejected twice each."""
    st = _assert_strict_trajectory(_indefinite_window(200.0), 10, mode)
    assert st["trials"][0] == 8 and st["accepted"][0] == 1


@pytest.mark.parametrize("mode", MODES)
def test_ten_failed_trials_terminate(mode):
    """B = 1e14 max|diag|: no lambda of the schedule (<= 1e-5 * 2^45 max|diag|) makes the system PD => 10 failed trials =>
    OptimizationAlgorithmLevenberg::solve returns Terminate, optimize() stops after that iteration, estimates untouched."""
    prob = _indefinite_window(1e14)
    st = _assert_strict_trajectory(prob, 10, mode)
    assert len(st) == 1 and st["trials"][0] == 10 and st["accepted"][0] == 0 and st["terminate"][0] == 1
    g = LocalBA.from_problem(prob, mode=mode)
    n, st_g = g.optimize(10)
    assert n == 1 and st_g["chi2_after"][0] == st_g["chi2_before"][0]
    p, l = g.get()
    np.testing.assert_array_equal(p, prob.poses); np.testing.assert_array_equal(l, prob.points)


@pytest.mark.parametrize("mode", MODES)
def test_rho_zero_terminates(mode):
    """Nothing to optimise (all poses fixed, no EdgeSE2XYZ): the cost cannot change, rho == 0 => Terminate after one trial."""
    prob = synth.ba_window(n_kf=3, n_lm=20, seed=5)
    prob.fixed[:] = 1
    prob.edge_pose, prob.edge_point, prob.uv, prob.info = prob.edge_pose[:0], prob.edge_point[:0], prob.uv[:0], prob.info[:0]
    st = _assert_strict_trajectory(prob, 5, mode, need_reject=False)
    assert len(st) == 1 and st["trials"][0] == 1 and st["rho"][0] == 0 and st["terminate"][0] == 1


@pytest.mark.parametrize("mode", MODES)
def test_edge_cases_unobserved_landmarks_and_all_poses_fixed(mode):
    prob = synth.ba_window(n_kf=4, n_lm=50, seed=2)
    keep = prob.edge_point != 0  # landmark 0 loses all its edges: inactive vertex, must stay untouched
    prob.edge_pose, prob.edge_point, prob.uv, prob.info = prob.edge_pose[keep], prob.edge_point[keep], prob.uv[keep], prob.info[keep]
    o = pyoracle.BAOracle(prob)
    n_o, st_o = o.optimize(5)
    g = LocalBA.from_problem(prob, mode=mode)
    n_g, st_g = g.optimize(5)
    assert n_g == n_o
    po, lo = o.get(); pg, lg = g.get()
    np.testing.assert_array_equal(lg[0], prob.points[0])
    np.testing.assert_allclose(pg, po, atol=1e-7)
    np.testing.assert_allclose(lg, lo, atol=1e-6)
    prob2 = synth.ba_window(n_kf=3, n_lm=30, seed=4)
    prob2.fixed[:] = 1  # all poses fixed: only landmarks move
    o2 = pyoracle.BAOracle(prob2); g2 = LocalBA.from_problem(prob2, mode=mode)
    n_o2, _ = o2.optimize(4); n_g2, _ = g2.optimize(4)
    assert n_g2 == n_o2
    np.testing.assert_allclose(g2.get()[1], o2.get()[1], atol=1e-6)
    np.testing.assert_array_equal(g2.get()[0], prob2.poses)


def test_capacity_and_argument_errors_are_reported():
    from se2lam_b200 import _capi
    prob = synth.ba_config("C1")
    g = LocalBA(1, 10, 10, 1)
    with pytest.raises(_capi.Se2GpuError):
        g.set_problem(prob)
    bad = copy.copy(prob)
    bad.edge_pose = prob.edge_pose.copy(); bad.edge_pose[0] = 99
    g2 = LocalBA(prob.P, prob.L, prob.E, prob.O)
    with pytest.raises(_capi.Se2GpuError):
        g2.set_problem(bad)


def test_full_size_properties_c4():
    """Size-independent properties at BASELINE size: cost never increases, result independent of the
    order in which edges are handed over (the C ABI re-sorts edges by landmark)."""
    prob = synth.ba_config("C4")
    g = LocalBA.from_problem(prob)
    n, st = g.optimize(10)
    assert np.all(st["chi2_after"] <= st["chi2_before"] * (1 + 1e-12))
    p1, l1 = g.get()
    perm = np.random.default_rng(0).permutation(prob.E)
    q = copy.copy(prob)
    q.edge_pose, q.edge_point, q.uv, q.info = prob.edge_pose[perm], prob.edge_point[perm], prob.uv[perm], prob.info[perm]
    g2 = LocalBA.from_problem(q)
    g2.optimize(10)
    p2, l2 = g2.get()
    np.testing.assert_allclose(p2, p1, rtol=0, atol=1e-9)
    np.testing.assert_allclose(l2, l1, rtol=0, atol=1e-8)


def test_graph_facade_reads_like_the_reference_loader():
    """Drive the reference-style helper API exactly the way Map::loadLocalGraph does (Map.cpp:891-1053)."""
    from se2lam_b200 import ba as B
    prob = synth.ba_config("C1")
    Rbc, tbc = synth.default_Tbc()
    opt = B.SlamOptimizer()
    B.initOptimizer(opt)
    K = np.array([[prob.fx, 0, prob.cx], [0, prob.fx, prob.cy], [0, 0, 1]], np.float32)
    campr = B.addCamPara(opt, K, 0)
    for i in range(prob.P):
        B.addVertexSE2(opt, prob.poses[i], i, bool(prob.fixed[i]))
    for k in range(prob.O):
        w = prob.odo_info[k]
        info = np.array([[w[0], w[1], w[2]], [w[1], w[3], w[4]], [w[2], w[4], w[5]]])
        B.addEdgeSE2(opt, prob.odo_meas[k], int(prob.odo_i[k]), int(prob.odo_j[k]), info)
    maxKFid = prob.P + 1
    for j in range(prob.L):
        B.addVertexSBAXYZ(opt, prob.points[j], maxKFid + j)
    for e in range(prob.E):
        w = prob.info[e]
        B.addEdgeSE2XYZ(opt, prob.uv[e], int(prob.edge_pose[e]), maxKFid + int(prob.edge_point[e]), campr, (Rbc, tbc),
                        np.array([[w[0], w[1]], [w[1], w[2]]]), prob.huber_delta)
    opt.initializeOptimization(0)
    n = opt.optimize(10)
    o = pyoracle.BAOracle(prob)
    n_o, _ = o.optimize(10)
    assert n == n_o
    po, lo = o.get()
    for i in range(prob.P):
        np.testing.assert_allclose(B.estimateVertexSE2(opt, i), po[i], atol=1e-8)
    for j in range(0, prob.L, 17):
        np.testing.assert_allclose(B.estimateVertexSBAXYZ(opt, maxKFid + j), lo[j], atol=1e-7)


@pytest.mark.parametrize("mode", MODES)
def test_reset_and_stop_flag(mode):
    """se2gpu_ba_reset restores the loaded window bit for bit; a raised abort flag stops the optimiser
    (setForceStopFlag semantics: no iteration is started once the flag is set)."""
    prob = synth.ba_config("C3")
    g = LocalBA.from_problem(prob, mode=mode)
    n1, st1 = g.optimize(6)
    p1, l1 = g.get()
    g.reset()
    p0, l0 = g.get()
    np.testing.assert_array_equal(p0, prob.poses); np.testing.assert_array_equal(l0, prob.points)
    n2, st2 = g.optimize(6)
    p2, l2 = g.get()
    assert n1 == n2 and p1.tobytes() == p2.tobytes() and l1.tobytes() == l2.tobytes()      # bit-reproducible runs
    np.testing.assert_array_equal(st1["chi2_after"], st2["chi2_after"])
    g.reset()
    flag = np.ones(1, np.uint8)
    n3, _ = g.optimize(6, stop_flag=flag)
    assert n3 == 0
    np.testing.assert_array_equal(g.get()[0], prob.poses)
    # continuing after a finished optimize restarts the lambda schedule (g2o: iteration==0 of a new optimize call)
    flag[0] = 0
    n4, st4 = g.optimize(3, stop_flag=flag)
    assert n4 == 3 and st4["chi2_before"][0] == st1["chi2_before"][0]


@pytest.mark.parametrize("world", [2, 3])
@pytest.mark.parametrize("cfg", ["C3", "C4"])
def test_sharded_path_on_one_device(cfg, world):
    """The real N>1 path - se2gpu_ba_set_shard(rank, world, callback), landmark j on rank j % world, the per-trial
    all-reduce of [S | b_s] and of [chi2, scale, stop] - run with `world` contexts on ONE device (tests/local_shards.py):
    same kernels and host loop as a multi-GPU run. Must follow the single-device oracle trajectory at the strict bar and
    be identical on every rank."""
    from tests.local_shards import merge_landmarks, run_local_shards
    prob = synth.ba_config(cfg)
    o = pyoracle.BAOracle(prob)
    n_o, st_o, tp_o, tl_o = o.optimize(10, trace=True)
    res = run_local_shards(prob, world, 10)
    for r in range(world):
        n, st, tp, tl, p, l = res[r]
        assert n == n_o
        np.testing.assert_array_equal(st["trials"], st_o["trials"])
        np.testing.assert_array_equal(st["accepted"], st_o["accepted"])
        np.testing.assert_allclose(st["lambda"], st_o["lambda"], rtol=1e-6)
        np.testing.assert_allclose(st["chi2_after"], st_o["chi2_after"], rtol=1e-8)
        assert tp.tobytes() == res[0][2].tobytes(), "replicated pose solves must be bit-identical across ranks"
        prev_p = prob.poses
        for k in range(n_o):
            dp_o, dp_g = tp_o[k] - prev_p, tp[k] - prev_p
            assert np.abs(dp_g - dp_o).max() <= REL * max(np.abs(dp_o).max(), 1e-12), f"rank {r} pose step {k}"
            prev_p = tp_o[k]
    pts = merge_landmarks(prob, res, world)
    po, lo = o.get()
    active = np.zeros(prob.L, bool); active[prob.edge_point] = True
    assert np.abs(pts[active] - lo[active]).max() <= 1e-7
    np.testing.assert_array_equal(pts[~active], prob.points[~active])


@pytest.mark.parametrize("cfg,world", [("C3", 2), ("C4", 2), ("C4", 3)])
def test_sharded_persistent_kernel_on_one_device(cfg, world, monkeypatch):
    """The multi-GPU production path for local windows: every rank runs ONE persistent cooperative kernel and the kernels
    exchange [S | b] and [chi2, scale, abort] through peer memory (no collective library, no host round trip). Here the
    ranks are contexts of one process on one GPU (se2gpu_ba_peer_attach_local), each limited to a share of the SMs so that
    the cooperative grids are co-resident. Strict per-step bar against the single-device oracle; all ranks bit-identical."""
    from tests.local_shards import merge_landmarks, pk_grid_share, run_local_shards
    monkeypatch.setenv("SE2GPU_BA_PK_GRID", pk_grid_share(world))
    monkeypatch.setenv("SE2GPU_BA_PEER_TIMEOUT_S", "20")
    prob = synth.ba_config(cfg)
    o = pyoracle.BAOracle(prob)
    n_o, st_o, tp_o, tl_o = o.optimize(10, trace=True)
    res = run_local_shards(prob, world, 10, setup=LocalBA.attach_local, mode=2)
    for r in range(world):
        n, st, tp, tl, p, l = res[r]
        assert n == n_o
        np.testing.assert_array_equal(st["trials"], st_o["trials"])
        np.testing.assert_array_equal(st["accepted"], st_o["accepted"])
        np.testing.assert_allclose(st["lambda"], st_o["lambda"], rtol=1e-6)
        np.testing.assert_allclose(st["chi2_after"], st_o["chi2_after"], rtol=1e-8)
        assert tp.tobytes() == res[0][2].tobytes(), "replicated pose solves must be bit-identical across ranks"
        prev_p = prob.poses
        for k in range(n_o):
            dp_o, dp_g = tp_o[k] - prev_p, tp[k] - prev_p
            assert np.abs(dp_g - dp_o).max() <= REL * max(np.abs(dp_o).max(), 1e-12), f"rank {r} pose step {k}"
            prev_p = tp_o[k]
    pts = merge_landmarks(prob, res, world)
    active = np.zeros(prob.L, bool); active[prob.edge_point] = True
    assert np.abs(pts[active] - o.get()[1][active]).max() <= 1e-7


def test_sharded_persistent_rejections_and_abort(monkeypatch):
    """Step rejections (restore / nu doubling) and the collective abort flag inside the sharded persistent kernel."""
    from tests.local_shards import pk_grid_share, run_local_shards
    monkeypatch.setenv("SE2GPU_BA_PK_GRID", pk_grid_share(2))
    monkeypatch.setenv("SE2GPU_BA_PEER_TIMEOUT_S", "20")
    prob = _perturbed(10, 600, 9, 1.0, 0.3, 0.0)
    n_o, st_o, tp_o, tl_o = pyoracle.BAOracle(prob).optimize(12, trace=True)
    res = run_local_shards(prob, 2, 12, setup=LocalBA.attach_local, mode=2)
    for r in range(2):
        assert res[r][0] == n_o
        np.testing.assert_array_equal(res[r][1]["trials"], st_o["trials"])
        np.testing.assert_allclose(res[r][1]["lambda"], st_o["lambda"], rtol=1e-6)
        assert np.abs(res[r][2][-1] - tp_o[-1]).max() < 1e-8
    flags = [np.zeros(1, np.uint8), np.ones(1, np.uint8)]
    res = run_local_shards(synth.ba_config("C3"), 2, 6, setup=LocalBA.attach_local, mode=2, stop_flags=flags)
    assert res[0][0] == res[1][0] == 0


@pytest.mark.parametrize("mode", MODES)
def test_sliced_optimize_continues_the_lambda_schedule(mode):
    """se2gpu_ba_optimize_from: ten one-iteration slices (what g2o's solve(iteration) hands to an OptimizationAlgorithm)
    are bit-identical to optimize(10); lambda is initialised at iteration 0 only."""
    prob = _perturbed(10, 600, 9, 1.0, 0.3, 0.0)        # rejects steps late in the run
    g = LocalBA.from_problem(prob, mode=mode)
    n, st, tp, tl = g.optimize(12, trace=True)
    g2 = LocalBA.from_problem(prob, mode=mode)
    sts = []
    for k in range(12):
        nk, sk = g2.optimize(1, first_iteration=k)
        assert nk == 1
        sts.append(sk[0])
    sts = np.array(sts, dtype=st.dtype)
    for f in ("trials", "accepted", "terminate", "lambda", "chi2_after", "rho"):
        np.testing.assert_array_equal(sts[f], st[f], err_msg=f)
    p1, l1 = g.get(); p2, l2 = g2.get()
    assert p1.tobytes() == p2.tobytes() and l1.tobytes() == l2.tobytes()


def test_sharded_abort_flag_is_collective():
    """Only ONE rank sees the abort flag raised: the decision is OR-ed over the ranks (third word of the per-trial
    all-reduce), so every rank stops after the same iteration instead of one rank leaving the collective sequence."""
    from tests.local_shards import run_local_shards
    prob = synth.ba_config("C3")
    flags = [np.zeros(1, np.uint8), np.ones(1, np.uint8)]     # rank 1 asks to stop from the start
    res = run_local_shards(prob, 2, 6, stop_flags=flags)
    assert res[0][0] == res[1][0] == 0
    np.testing.assert_array_equal(res[0][4], prob.poses)


def _medium_window():
    return synth.ba_window(n_kf=120, n_lm=3000, seed=11)         # n = 357 unknowns: beyond one CTA's shared memory


@pytest.mark.parametrize("solver", ["band", "envelope"])
def test_large_window_solvers_match_oracle(solver, monkeypatch):
    """Reduced systems that do not fit one CTA's shared memory: the partitioned block-band LDL^T (ba_band.cu) and the
    single-CTA global-memory envelope factorisation it replaces (SE2GPU_BA_NO_BAND=1) both hold the strict per-step bar."""
    if solver == "envelope":
        monkeypatch.setenv("SE2GPU_BA_NO_BAND", "1")
    prob = _medium_window()
    _assert_strict_trajectory(prob, 6, 0, need_reject=False)
    o = pyoracle.BAOracle(prob)
    lin = o.linearize()
    lam = 1e-5 * max(np.abs(np.diag(lin["Hpp"])).max(), np.abs(lin["Hll"][:, [0, 1, 2], [0, 1, 2]]).max())
    ss = o.schur_solve(lam)
    sysm = LocalBA.from_problem(prob).debug_system(lam)
    n = sysm["n"]
    tril = np.tril(np.ones((n, n), bool))
    assert rel_err(sysm["S"][tril], ss["S"][tril]) < 1e-10
    assert rel_err(sysm["dx_p"], ss["dx_p"]) < REL and rel_err(sysm["dx_l"], ss["dx_l"]) < REL


def test_band_solver_rejects_non_pd_and_recovers():
    """The partitioned factorisation is a symmetric permutation of S: a non-PD pivot block in any partition == S not PD."""
    prob = _medium_window()
    prob.poses = prob.poses.copy(); prob.odo_info = prob.odo_info.copy()
    prob.poses[0, 2] = 0.0
    lin = pyoracle.BAOracle(prob).linearize()
    md = max(np.abs(np.diag(lin["Hpp"])).max(), np.abs(lin["Hll"][:, [0, 1, 2], [0, 1, 2]]).max())
    prob.odo_info[0] = [0.0, 200.0 * md, 0.0, 0.0, 0.0, prob.odo_info[0][5]]
    st = _assert_strict_trajectory(prob, 4, 0)
    assert st["trials"][0] == 8


def test_sharded_large_window_on_one_device():
    """Sharded run of a band-mode window: the per-trial all-reduce carries the band-stored reduced system."""
    from tests.local_shards import merge_landmarks, run_local_shards
    prob = _medium_window()
    o = pyoracle.BAOracle(prob)
    n_o, st_o, tp_o, tl_o = o.optimize(5, trace=True)
    res = run_local_shards(prob, 2, 5)
    for r in range(2):
        n, st, tp, tl, p, l = res[r]
        assert n == n_o
        np.testing.assert_array_equal(st["trials"], st_o["trials"])
        np.testing.assert_allclose(st["lambda"], st_o["lambda"], rtol=1e-6)
        assert np.abs(tp[-1] - tp_o[-1]).max() < 1e-8
    pts = merge_landmarks(prob, res, 2)
    active = np.zeros(prob.L, bool); active[prob.edge_point] = True
    assert np.abs(pts[active] - o.get()[1][active]).max() < 1e-7


@pytest.mark.parametrize("mode", MODES)
def test_same_topology_reload_refreshes_values_only(mode):
    """set_problem with the graph structure of the loaded window (same vertices / fixed flags / edge endpoints) keeps the
    device-side structure and refreshes the values: the result must equal a fresh context's, bit for bit; a changed edge
    list falls back to the full rebuild."""
    a = synth.ba_config("C3")
    b = copy.copy(a)
    rng = np.random.default_rng(3)
    b.poses = a.poses + rng.normal(0, 0.01, a.poses.shape); b.poses[0] = a.poses[0]
    b.points = a.points + rng.normal(0, 0.02, a.points.shape)
    b.uv = a.uv + rng.normal(0, 0.3, a.uv.shape); b.info = a.info * 1.1; b.odo_meas = a.odo_meas + 1e-3; b.odo_info = a.odo_info * 0.9
    g = LocalBA.from_problem(a, mode=mode)
    g.optimize(4)
    g.set_problem(b)                       # same topology: fast path
    n1, st1 = g.optimize(6)
    p1, l1 = g.get()
    f = LocalBA.from_problem(b, mode=mode)
    n2, st2 = f.optimize(6)
    p2, l2 = f.get()
    assert n1 == n2 and p1.tobytes() == p2.tobytes() and l1.tobytes() == l2.tobytes()
    np.testing.assert_array_equal(st1["chi2_after"], st2["chi2_after"])
    c = copy.copy(b)
    keep = np.ones(b.E, bool); keep[::7] = False
    c.edge_pose, c.edge_point, c.uv, c.info = b.edge_pose[keep], b.edge_point[keep], b.uv[keep], b.info[keep]
    g.set_problem(c)                       # different edge list: full rebuild
    g.optimize(5)
    o = pyoracle.BAOracle(c); o.optimize(5)
    np.testing.assert_allclose(g.get()[0], o.get()[0], atol=1e-8)


def test_scale_config_c5_matches_oracle():
    """BASELINE config 5 (2000 KF / 50k landmarks / ~300k edges): the reduced system (n = 5997) does not fit one CTA's
    shared memory, so this exercises the global-memory envelope LDL^T and the multi-launch path at scale."""
    prob = synth.ba_config("C5")
    iters = 3
    o = pyoracle.BAOracle(prob)
    n_o, st_o, tp_o, tl_o = o.optimize(iters, trace=True)
    g = LocalBA.from_problem(prob)
    n_g, st_g, tp_g, tl_g = g.optimize(iters, trace=True)
    assert n_g == n_o
    np.testing.assert_array_equal(st_g["trials"], st_o["trials"])
    np.testing.assert_array_equal(st_g["accepted"], st_o["accepted"])
    np.testing.assert_allclose(st_g["lambda"], st_o["lambda"], rtol=1e-6)
    np.testing.assert_allclose(st_g["chi2_after"], st_o["chi2_after"], rtol=1e-8)
    prev_p, prev_l = prob.poses, prob.points
    for k in range(n_o):
        dp_o, dp_g = tp_o[k] - prev_p, tp_g[k] - prev_p
        dl_o, dl_g = tl_o[k] - prev_l, tl_g[k] - prev_l
        assert np.abs(dp_g - dp_o).max() <= REL * max(np.abs(dp_o).max(), 1e-12), f"pose step {k}"
        assert np.abs(dl_g - dl_o).max() <= REL * max(np.abs(dl_o).max(), 1e-12), f"landmark step {k}"
        prev_p, prev_l = tp_o[k], tl_o[k]
