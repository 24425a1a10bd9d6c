"""GPU parity of the local BA on the code paths that set_problem and the persistent kernel choose per window: the reduced
solvers (single CTA, twisted, partitioned band, global-memory envelope), the structure build (dense table or sorted), the
persistent kernel's Schur work split (cached concurrent plan or uncached sequential sweep) and reference-shaped window
topologies (tests/ba_cases.py). Every test first proves its path with se2gpu_ba_debug_plan, then holds the run to the
strict bar of test_ba_gpu against the CPU oracle: identical trials / accept / terminate sequences, lambda to 1e-6, chi2 to
1e-8 and every per-step update to 1e-5. Each window passes the conditioning screen of test_ba_topology_oracle."""
import numpy as np
import pytest

from oracle import pyoracle
from se2lam_b200.ba import LocalBA
from tests import ba_cases as bc
from tests.test_ba_gpu import REL, _assert_strict_trajectory, rel_err
from tools import synth

pytestmark = pytest.mark.gpu


def _plan(case, prob, mode=0):
    """debug_plan of a fresh context (same environment as the run under test); printed for the record"""
    p = LocalBA.from_problem(prob, mode=mode).debug_plan()
    print(f"\nPLAN {case}: " + " ".join(f"{k}={v}" for k, v in p.items()))
    return p


def _assert_system(prob):
    """debug_system's reduced system and step at one lambda against BAOracle.schur_solve"""
    o = pyoracle.BAOracle(prob)
    lin = o.linearize()
    lam = 1e-5 * max(np.abs(np.diag(lin["Hpp"])).max(), np.abs(lin["Hll"][:, [0, 1, 2], [0, 1, 2]]).max())
    ss = o.schur_solve(lam)
    assert ss["ok"] == 1
    sysm = LocalBA.from_problem(prob).debug_system(lam)
    n = sysm["n"]
    assert n == 3 * o.nf
    tril = np.tril(np.ones((n, n), bool))
    assert rel_err(sysm["S"][tril], ss["S"][tril]) < 1e-10
    assert rel_err(sysm["bs"], ss["bs"]) < 1e-9
    assert rel_err(sysm["dx_p"], ss["dx_p"]) < REL
    assert rel_err(sysm["dx_l"], ss["dx_l"]) < REL


# ---- reduced solve: twisted separator width, and where the twist is not taken -------------------------------------------
@pytest.mark.parametrize("no_twist", [False, True], ids=["twist", "no-twist"])
@pytest.mark.parametrize("name,sep", [("twist_w6", 6), ("twist_w10", 10), ("twist_w16", 16), ("smem_w17", None),
                                      ("chain_nf16", None)])
def test_twisted_separator_widths(name, sep, no_twist, monkeypatch):
    if no_twist:
        monkeypatch.setenv("SE2GPU_BA_NO_TWIST", "1")
    prob, iters = bc.strict(name)
    p = _plan(name + ("/no-twist" if no_twist else ""), prob, mode=2)
    assert p["n"] <= 156 and p["structure"] == "dense"
    if sep is not None and not no_twist:
        assert p["solver"] == "twisted" and p["tw_w"] == sep and p["env_w"] == sep and p["n"] == 156
        assert p["workers"] == p["pk_grid"] - 2
    else:
        assert p["solver"] == "smem" and p["tw_m0"] == 0 and p["workers"] == p["pk_grid"] - 1
        if name == "smem_w17":
            assert p["env_w"] == 17                      # one block beyond TW_MAX_W
        if name == "chain_nf16":
            assert p["nf"] == 16 and p["env_w"] == 5     # the chain rule, not the width, rejects the twist
    _assert_strict_trajectory(prob, iters, 2, need_reject=False)
    if not no_twist:
        _assert_system(prob)


# ---- n = 156 (one CTA's shared memory) against n = 159 ------------------------------------------------------------------
def test_shared_memory_boundary(monkeypatch):
    monkeypatch.setenv("SE2GPU_BA_NO_TWIST", "1")
    small, it_s = bc.strict("smem_nf52")
    large, it_l = bc.strict("large_nf53")
    ps, pl = _plan("smem_nf52", small, mode=1), _plan("large_nf53", large)
    assert ps["n"] == 156 and ps["solver"] == "smem"
    assert pl["n"] == 159 and pl["solver"] in ("band", "envelope")
    _assert_strict_trajectory(small, it_s, 1, need_reject=False)
    _assert_strict_trajectory(large, it_l, 0, need_reject=False)
    _assert_system(small)
    _assert_system(large)


# ---- partitioned band solver: half-width 1 .. 10, uneven partitions, w = 11 -> envelope ------------------------------------
@pytest.mark.parametrize("w", [1, 2, 3, 4, 6, 8, 10])
def test_band_half_width(w):
    prob, iters = bc.strict(f"band_w{w}")
    p = _plan(f"band_w{w}", prob)
    assert p["nf"] == 59 and p["solver"] == "band" and p["band_w"] == w == p["env_w"] and p["band_p"] >= 2
    _assert_strict_trajectory(prob, iters, 0, need_reject=False)
    _assert_system(prob)


def test_band_partitions_of_unequal_length():
    """nf - w (p - 1) interior blocks that do not divide by p: the first partitions are one block longer."""
    prob, iters = bc.strict("band_w2")
    p = _plan("band_w2/uneven", prob)
    assert p["solver"] == "band" and (p["nf"] - p["band_w"] * (p["band_p"] - 1)) % p["band_p"] != 0
    _assert_strict_trajectory(prob, iters, 0, need_reject=False)


def test_band_rejects_w11_for_the_envelope():
    prob, iters = bc.strict("env_w11")
    p = _plan("env_w11", prob)
    assert p["solver"] == "envelope" and p["env_w"] == 11 and p["band_p"] == 0
    _assert_strict_trajectory(prob, iters, 0, need_reject=False)
    _assert_system(prob)


# ---- nf >= 2049: the comparison-sorted structure build, with a fixed tail and w = 10 ---------------------------------------
def test_sorted_structure_build_with_fixed_tail():
    """2 060 zigzag KFs, 6 fixed reference KFs at the tail and one fixed in the middle (nf = 2 053, ~117 k edges). At this
    size and w = 10 the band solver's shared-memory budget, not its cost model, bounds the partition count."""
    prob, iters = bc.strict("sorted_w10")
    p = _plan("sorted_w10", prob, mode=1)
    assert p["nf"] >= 2049 and p["structure"] == "sorted" and p["env_w"] == 10
    assert p["solver"] in ("band", "envelope")
    if p["solver"] == "band":
        assert p["band_w"] == 10 and p["band_p"] >= 2
    _assert_strict_trajectory(prob, iters, 1, need_reject=False)


# ---- persistent kernel: Schur work split over a limited grid -------------------------------------------------------------
def _split_window(name):
    if name in ("C3", "C4"):
        return synth.ba_config(name), 10
    return bc.strict(name)


@pytest.mark.parametrize("grid", [2, 3, 4, 5, 9])
@pytest.mark.parametrize("name", ["C3", "C4", "dense_nf29"])
def test_persistent_work_split(name, grid, monkeypatch):
    """SE2GPU_BA_PK_GRID limits the cooperative grid. Grid 2: one worker owns every block (more than 16), so the uncached
    sequential Schur sweep runs; grid 4 gives the twisted solve only 2 workers. Each grid is held to the oracle."""
    monkeypatch.setenv("SE2GPU_BA_PK_GRID", str(grid))
    prob, iters = _split_window(name)
    p = _plan(f"{name}/grid{grid}", prob, mode=2)
    assert p["pk_grid"] == grid
    assert p["workers"] == grid - (2 if p["solver"] == "twisted" else 1)
    if grid < 4:
        assert p["solver"] == "smem"
    if grid == 2:
        assert p["workers"] == 1 and p["max_own"] == p["nblk"] > 16 and p["uncached"] == 1
    if grid == 4 and name in ("C3", "C4"):
        assert p["solver"] == "twisted" and p["workers"] == 2
    _assert_strict_trajectory(prob, iters, 2, need_reject=False)


def test_full_grid_arena_limits_the_cache():
    """Full grid, one block per worker, but diagonal blocks whose pair and edge lists exceed a worker's shared-memory arena:
    those workers fall back to the uncached sweep although they own far fewer than 16 blocks."""
    prob, iters = bc.strict("dense_arena")
    p = _plan("dense_arena", prob, mode=2)
    assert p["max_own"] <= 16 and p["uncached"] > 0
    _assert_strict_trajectory(prob, iters, 2, need_reject=False)


# ---- reference-shaped topologies ----------------------------------------------------------------------------------------
TOPOLOGY = ["tail_nf23", "broken_nf29", "reversed_nf28", "duplicated_nf28", "loop_nf39", "sparse_nf29", "dense_nf29"]


@pytest.mark.parametrize("mode", [1, 2], ids=["multi-launch", "persistent"])
@pytest.mark.parametrize("name", TOPOLOGY)
def test_topology_small_windows(name, mode):
    prob, iters = bc.strict(name)
    p = _plan(f"{name}/mode{mode}", prob, mode=mode)
    assert p["n"] <= 156 and p["nf"] == (prob.fixed == 0).sum()
    if name == "loop_nf39":
        assert p["env_w"] > 16 and p["solver"] == "smem"                 # the loop closure widens the envelope past the twist
    _assert_strict_trajectory(prob, iters, mode, need_reject=False)
    if mode == 1:
        _assert_system(prob)
    if name == "sparse_nf29":                                         # the free pose without edges never moves
        g = LocalBA.from_problem(prob, mode=mode)
        g.optimize(iters)
        np.testing.assert_array_equal(g.get()[0][-1], prob.poses[-1])


@pytest.mark.parametrize("name,solver", [("tail_nf59", "band"), ("loop_nf79", "envelope")])
def test_topology_large_windows(name, solver):
    prob, iters = bc.strict(name)
    p = _plan(name, prob)
    assert p["solver"] == solver
    if name == "loop_nf79":
        assert p["env_w"] > 10
    _assert_strict_trajectory(prob, iters, 0, need_reject=False)
    _assert_system(prob)


def _assert_sharded(prob, iters, **kw):
    from tests.local_shards import merge_landmarks, run_local_shards
    o = pyoracle.BAOracle(prob)
    n_o, st_o, tp_o, tl_o = o.optimize(iters, trace=True)
    res = run_local_shards(prob, 2, iters, **kw)
    for r in range(2):
        n, st, tp, tl, _, _ = res[r]
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
    pts = merge_landmarks(prob, res, 2)
    active = np.zeros(prob.L, bool); active[prob.edge_point] = True
    assert np.abs(pts[active] - o.get()[1][active]).max() <= 1e-7
    np.testing.assert_array_equal(pts[~active], prob.points[~active])


@pytest.mark.parametrize("path", ["callback", "persistent"])
@pytest.mark.parametrize("name", ["tail_nf23", "reversed_nf28"])
def test_topology_sharded_on_one_device(name, path, monkeypatch):
    """world 2 on one device: the per-trial all-reduce through the callback, and the persistent kernels exchanging through
    peer memory. Every rank rebuilds the envelope from the unsharded edge list, so the plan is the unsharded one."""
    from tests.local_shards import pk_grid_share
    prob, iters = bc.strict(name)
    if path == "persistent":
        monkeypatch.setenv("SE2GPU_BA_PK_GRID", pk_grid_share(2))
        monkeypatch.setenv("SE2GPU_BA_PEER_TIMEOUT_S", "20")
        p = _plan(f"{name}/sharded-{path}", prob, mode=2)
        assert p["solver"] == "twisted"
        _assert_sharded(prob, iters, setup=LocalBA.attach_local, mode=2)
    else:
        p = _plan(f"{name}/sharded-{path}", prob, mode=1)
        assert p["n"] <= 156
        _assert_sharded(prob, iters)


# ---- non-positive-definite trials on the twisted and band solvers ----------------------------------------------------------
@pytest.mark.parametrize("name,mode,solver", [("twist_w10", 2, "twisted"), ("band_w1", 0, "band")])
def test_non_positive_definite_trials_on_new_paths(name, mode, solver):
    prob, iters = bc.strict(name)
    prob = bc.nonpd(prob)
    p = _plan(f"nonpd_{name}", prob, mode=mode)
    assert p["solver"] == solver
    st = _assert_strict_trajectory(prob, iters, mode)
    assert st["trials"][0] > 1 and st["accepted"][0] == 1
