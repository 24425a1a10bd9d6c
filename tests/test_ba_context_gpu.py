"""One local-BA context across a sequence of windows, the way the drop-in SparseOptimizer keeps its device context while the
capacity suffices (include/se2lam/g2o_compat.h) and LocalMapper reloads the graph after removeOutlierChi2.

The bar: after every set_problem on the reused context, optimize(trace=True) (iteration count, stats and trace bytes), the
bytes of get() / get_f32() and debug_plan() equal those of a FRESH context loaded with that window alone - one with the
same capacities and mode, and one with tight capacities (LocalBA.from_problem). State left over from an earlier window
shows up as a difference here. Each step also proves which path set_problem took: SE2GPU_BA_DEBUG=1 makes it report a
values-only refresh on stderr, and a full rebuild reports its plan (solver, structure, uncached Schur workers).
Windows that no other test holds against the oracle also get the strict per-step bar of test_ba_gpu."""
import ctypes as C
import os
import struct
import subprocess
import threading

import numpy as np
import pytest
import torch

from oracle import pyoracle
from se2lam_b200 import _capi, build
from se2lam_b200.ba import LocalBA
from tests import ba_cases as bc
from tests.local_shards import _as_tensor, pk_grid_share, run_local_shards
from tests.test_ba_gpu import _assert_strict_trajectory
from tools import synth

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FAST = "same topology: values refreshed"
MODES = [pytest.param(1, id="multi-launch"), pytest.param(2, id="persistent")]
ERR_INVALID, ERR_CAPACITY = -3, -4          # SE2GPU_ERR_INVALID, SE2GPU_ERR_CAPACITY
gpu = pytest.mark.gpu                        # every test but the demo's compile-and-link check


@pytest.fixture
def debug(monkeypatch):
    """The BA reads its switches when a context is created: set before any context of the test exists."""
    monkeypatch.setenv("SE2GPU_BA_DEBUG", "1")
    return monkeypatch


# ------------------------------------------------------------------------------------------------------------ windows
def slide(prob, start, length):
    """Keyframes [start, start + length) of one long trajectory with the landmarks they observe, re-indexed, the first
    keyframe fixed: LocalMapper's window moving along the trajectory."""
    q = bc._copy(prob)
    stop = start + length
    keep = (prob.edge_pose >= start) & (prob.edge_pose < stop)
    lms = np.unique(prob.edge_point[keep])
    new_lm = np.full(prob.L, -1, np.int32); new_lm[lms] = np.arange(len(lms), dtype=np.int32)
    bc._keep_edges(q, keep)
    q.edge_pose = (q.edge_pose - start).astype(np.int32); q.edge_point = new_lm[q.edge_point]
    bc._keep_odo(q, (prob.odo_i >= start) & (prob.odo_i < stop) & (prob.odo_j >= start) & (prob.odo_j < stop))
    q.odo_i = (q.odo_i - start).astype(np.int32); q.odo_j = (q.odo_j - start).astype(np.int32)
    q.poses = prob.poses[start:stop].copy(); q.gt_poses = prob.gt_poses[start:stop].copy()
    q.points = prob.points[lms].copy(); q.gt_points = prob.gt_points[lms].copy()
    q.fixed = np.zeros(length, np.uint8); q.fixed[0] = 1
    return q


def new_values(prob, seed, camera=False):
    """Same graph structure, every value changed; with camera=True also fx / cx / cy, Tcb and the Huber delta."""
    q = bc._copy(prob)
    rng = np.random.default_rng(seed)
    free = prob.fixed == 0
    q.poses[free] += rng.normal(0, [0.01, 0.01, 0.003], (int(free.sum()), 3))
    q.points += rng.normal(0, 0.02, q.points.shape)
    q.uv += rng.normal(0, 0.3, q.uv.shape); q.info *= 1.1
    q.odo_meas += 1e-3; q.odo_info *= 0.9
    if camera:
        q.fx, q.cx, q.cy = prob.fx * 1.01, prob.cx + 1.5, prob.cy - 1.0
        c, s = np.cos(0.01), np.sin(0.01)
        Rcb = np.asarray(prob.Tcb[:9]).reshape(3, 3) @ np.array([[c, -s, 0], [s, c, 0], [0, 0, 1.0]])
        q.Tcb = np.concatenate([Rcb.reshape(-1), np.asarray(prob.Tcb[9:]) + [0.01, -0.005, 0.0]])
        q.huber_delta = prob.huber_delta * 1.5
    return q


def fixed_flipped(prob, k):
    q = bc._copy(prob)
    q.fixed[k] ^= 1
    return q


def odometry_reversed(prob, o):
    q = bc._copy(prob)
    q.odo_meas[o], q.odo_info[o] = bc.reversed_measurement(prob.odo_meas[o], prob.odo_info[o])
    q.odo_i[o], q.odo_j[o] = prob.odo_j[o], prob.odo_i[o]
    return q


def edge_chi2(prob, poses, points):
    """non-robust chi2 of every EdgeSE2XYZ at the given estimates (EdgeSE2XYZ::computeError + chi2)"""
    Rcb = np.asarray(prob.Tcb[:9]).reshape(3, 3); tcb = np.asarray(prob.Tcb[9:])
    x, y, th = poses[prob.edge_pose].T
    c, s = np.cos(th), np.sin(th)
    d = points[prob.edge_point] - np.stack([x, y, np.zeros_like(x)], 1)
    lb = np.stack([c * d[:, 0] + s * d[:, 1], -s * d[:, 0] + c * d[:, 1], d[:, 2]], 1)
    lc = lb @ Rcb.T + tcb
    e = prob.fx * lc[:, :2] / lc[:, 2:] + [prob.cx, prob.cy] - prob.uv
    w = prob.info
    return e[:, 0] * (w[:, 0] * e[:, 0] + w[:, 1] * e[:, 1]) + e[:, 1] * (w[:, 1] * e[:, 0] + w[:, 2] * e[:, 1])


def caps_of(probs):
    return (max(p.P for p in probs), max(max(p.L for p in probs), 1), max(max(p.E for p in probs), 1), max(max(p.O for p in probs), 1))


# ------------------------------------------------------------------------------------------------------------ the bar
def context(caps, mode):
    ba = LocalBA(*caps)
    ba.set_mode(mode)
    return ba


def outcome(ba, iters):
    n, st, tp, tl = ba.optimize(iters, trace=True)
    p, l = ba.get()
    pf, lf = ba.get_f32()
    return dict(n=n, stats=st.tobytes(), trace_poses=tp.tobytes(), trace_points=tl.tobytes(), poses=p.tobytes(),
                points=l.tobytes(), poses_f32=pf.tobytes(), points_f32=lf.tobytes(), plan=ba.debug_plan())


def assert_same(got, want, what):
    for k in want:
        assert got[k] == want[k], f"{what}: {k} differs from a fresh context's"


def load(ba, prob, capfd, fast):
    """set_problem, and the path it took: the values-only refresh (fast) or a full rebuild"""
    capfd.readouterr()
    ba.set_problem(prob)
    err = capfd.readouterr().err
    assert (FAST in err) == fast, f"expected {'the values-only refresh' if fast else 'a full rebuild'}; set_problem said: {err!r}"


def step(ba, prob, iters, capfd, fast, caps, mode, plan=None):
    """one window on the reused context against fresh contexts; plan: expected debug_plan entries"""
    load(ba, prob, capfd, fast)
    got = outcome(ba, iters)
    for fresh, what in ((context(caps, mode), "same capacities"), (LocalBA(*caps_of([prob])), "tight capacities")):
        fresh.set_mode(mode)
        fresh.set_problem(prob)
        assert_same(got, outcome(fresh, iters), what)
        fresh.close()
    for k, v in (plan or {}).items():
        assert got["plan"][k] == v, f"plan {k}: {got['plan'][k]} != {v}"
    return got


# ------------------------------------------------------------------------------------------------------------ transitions
def _c3():
    return synth.ba_config("C3")


@gpu
@pytest.mark.parametrize("mode", MODES)
def test_values_only_reload_takes_the_new_camera_and_huber_delta(mode, debug, capfd):
    """Transition 1: same topology, new values, and new fx / cx / cy, Tcb and Huber delta: the values-only path."""
    a = _c3()
    b = new_values(a, 1, camera=True)
    caps = caps_of([a, b])
    ba = context(caps, mode)
    step(ba, a, 8, capfd, False, caps, mode, dict(solver="twisted", structure="dense"))
    step(ba, b, 8, capfd, True, caps, mode, dict(solver="twisted", structure="dense"))
    _assert_strict_trajectory(b, 8, mode, need_reject=False)


@gpu
@pytest.mark.parametrize("mode", MODES)
def test_same_counts_other_topology_rebuilds(mode, debug, capfd):
    """Transitions 2-4: P / L / E / O unchanged, the structure not: the edge list permuted, one fixed flag flipped (nf
    changes), one odometry edge stated from its other end. Each is a full rebuild equal to a fresh load."""
    a = _c3()
    perm = bc.edge_permuted(a, seed=4)
    flip = fixed_flipped(perm, 10)
    rev = odometry_reversed(flip, 5)
    caps = caps_of([a])
    ba = context(caps, mode)
    step(ba, a, 8, capfd, False, caps, mode, dict(nf=19))
    step(ba, perm, 8, capfd, False, caps, mode, dict(nf=19))
    step(ba, flip, 8, capfd, False, caps, mode, dict(nf=18))
    step(ba, rev, 8, capfd, False, caps, mode, dict(nf=18))
    step(ba, a, 8, capfd, False, caps, mode, dict(nf=19))
    for w in (perm, flip, rev):
        _assert_strict_trajectory(w, 8, mode, need_reject=False)


@gpu
@pytest.mark.parametrize("mode", MODES)
def test_outlier_edges_removed_then_reloaded(mode, debug, capfd):
    """Transition 5, LocalMapper::removeOutlierChi2: optimise, drop the EdgeSE2XYZ whose chi2 exceeds 5.991 at the result,
    and load the remaining graph from the optimised estimates."""
    a = _c3()
    caps = caps_of([a])
    ba = context(caps, mode)
    step(ba, a, 8, capfd, False, caps, mode)
    poses, points = ba.get()
    inl = bc._copy(a)
    inl.poses, inl.points = poses, points
    keep = edge_chi2(a, poses, points) <= 5.991
    assert 0 < (~keep).sum() < a.E // 4
    bc._keep_edges(inl, keep)
    step(ba, inl, 8, capfd, False, caps, mode)
    _assert_strict_trajectory(inl, 8, mode, need_reject=False)


@gpu
@pytest.mark.parametrize("mode", MODES)
def test_sliding_window(mode, debug, capfd):
    """Transition 6: the window slides along one trajectory, one keyframe per step; two steps keep every count and change
    the structure (the edges handed over in another order; the second keyframe fixed as well)."""
    base = synth.ba_window(22, 1400, seed=5)
    seq = [slide(base, k, 12) for k in range(8)]
    seq.insert(3, bc.edge_permuted(seq[2], seed=1))
    seq.insert(6, fixed_flipped(seq[5], 1))
    caps = caps_of(seq)
    ba = context(caps, mode)
    for k, w in enumerate(seq):
        step(ba, w, 8, capfd, False, caps, mode, dict(nf=int((w.fixed == 0).sum())))
    for k, w in enumerate(seq):
        if k not in (3, 6):
            _assert_strict_trajectory(w, 8, mode, need_reject=False)


REGIMES = [   # STRICT window, debug_plan entries its full load must report
    ("chain_nf16", dict(solver="smem", structure="dense", uncached=0)),
    ("tail_nf23", dict(solver="twisted", structure="dense", uncached=0)),
    ("twist_w10", dict(solver="twisted", structure="dense", uncached=0)),
    ("band_w4", dict(solver="band", structure="dense")),
    ("env_w11", dict(solver="envelope", structure="dense")),
    ("dense_arena", dict(solver="smem", structure="dense")),
]


@gpu
@pytest.mark.parametrize("mode", [pytest.param(0, id="auto"), pytest.param(1, id="multi-launch")])
def test_grow_and_shrink_across_the_solver_regimes(mode, debug, capfd):
    """Transition 7: one context sized for the largest window runs smem -> twisted (reference-shaped tail, then separator
    w = 10) -> band -> envelope -> the uncached Schur sweep (the longest pair list) -> twisted -> smem, then the first
    window with new values (values-only). Pair, block and envelope lists regrow, and the band is planned and released."""
    wins = {name: bc.strict(name) for name, _ in REGIMES}
    caps = caps_of([w for w, _ in wins.values()])
    ba = context(caps, mode)
    for name, plan in REGIMES:
        prob, iters = wins[name]
        got = step(ba, prob, iters, capfd, False, caps, mode, plan)
        if name == "dense_arena":
            assert got["plan"]["uncached"] > 0
    for name, plan in (REGIMES[1], REGIMES[0]):
        prob, iters = wins[name]
        step(ba, prob, iters, capfd, False, caps, mode, plan)
    step(ba, new_values(prob, 5), iters, capfd, True, caps, mode, REGIMES[0][1])


@gpu
@pytest.mark.parametrize("mode", MODES)
def test_degenerate_windows_between_normal_ones(mode, debug, capfd):
    """Transition 8: an odometry-only window (E = 0, no landmarks), an all-fixed window (nf = 0) and a window with
    unobserved landmarks, each between two normal windows."""
    normal = [synth.ba_window(8, 400, seed=s) for s in (2, 3, 4, 5)]
    odo = bc._copy(normal[0])
    bc._keep_edges(odo, np.zeros(odo.E, bool)); odo.points = odo.points[:0]; odo.gt_points = odo.gt_points[:0]
    # a second path 0 -> 3 keeps the optimum's cost away from round-off (a lone chain converges to chi2 ~ 1e-17)
    bc._add_odo(odo, 0, 3, bc._rel(odo.gt_poses[0], odo.gt_poses[3]) + [0.02, -0.01, 0.005], odo.odo_info[0])
    allfixed = bc._copy(synth.ba_window(6, 300, seed=6)); allfixed.fixed[:] = 1
    unobs = bc._copy(synth.ba_window(8, 400, seed=7)); bc._keep_edges(unobs, ~np.isin(unobs.edge_point, [0, 5, 77]))
    seq = [normal[0], odo, normal[1], allfixed, normal[2], unobs, normal[3]]
    iters = {id(odo): 3}                # odometry alone converges fast: later steps are below the per-step bar's resolution
    caps = caps_of(seq)
    ba = context(caps, mode)
    for w in seq:
        step(ba, w, iters.get(id(w), 6), capfd, False, caps, mode, dict(nf=int((w.fixed == 0).sum())))
        if w is unobs:
            np.testing.assert_array_equal(ba.get()[1][[0, 5, 77]], unobs.points[[0, 5, 77]])
    for w in (odo, allfixed, unobs):
        _assert_strict_trajectory(w, iters.get(id(w), 6), mode, need_reject=False)


@gpu
@pytest.mark.parametrize("mode", MODES)
def test_structural_zeros_inside_the_envelope_after_a_dense_window(mode, debug, capfd):
    """A window whose reduced system has every block non-zero, then one of the same nf whose envelope is nearly full but
    whose blocks form a band and one long-range co-observation: the entries inside the new envelope that no block covers
    must read as zeros, not as the previous window's S."""
    dense = bc.dense_covisibility(12, 600, seed=3)
    band = bc._copy(synth.ba_window(12, 600, seed=4, obs_per_lm=3))
    e0 = int(np.flatnonzero(band.edge_pose == 1)[0])
    band.edge_pose = np.r_[band.edge_pose, np.int32(11)].astype(np.int32)
    band.edge_point = np.r_[band.edge_point, band.edge_point[e0]].astype(np.int32)
    band.uv = np.vstack([band.uv, band.uv[e0]]); band.info = np.vstack([band.info, band.info[e0]])
    caps = caps_of([dense, band])
    ba = context(caps, mode)
    full = step(ba, dense, 6, capfd, False, caps, mode)
    got = step(ba, band, 6, capfd, False, caps, mode)
    assert got["plan"]["nf"] == full["plan"]["nf"] and got["plan"]["nblk"] < full["plan"]["nblk"]
    assert got["plan"]["env_w"] == 10


@gpu
@pytest.mark.parametrize("modes",[pytest.param((2, 2, 2), id="persistent-growing"), pytest.param((1, 2, 0), id="switch-1-2-0")])
def test_trace_buffers_regrow_and_mode_switches(modes, debug, capfd):
    """Transition 9: windows grow in P and L with trace=True and more iterations each time, so the persistent kernel's
    trace buffers regrow; set_mode between windows."""
    seq = [(synth.ba_window(6, 300, seed=8), 4), (synth.ba_window(12, 900, seed=9), 6), (synth.ba_window(20, 2000, seed=10), 8)]
    caps = caps_of([w for w, _ in seq])
    ba = context(caps, modes[0])
    for (w, iters), m in zip(seq, modes):
        ba.set_mode(m)
        step(ba, w, iters, capfd, False, caps, m)
    w, _ = seq[0]
    ba.set_mode(modes[0])
    step(ba, w, 10, capfd, False, caps, modes[0])


@gpu
@pytest.mark.parametrize("mode", MODES)
def test_reset_and_slices_after_a_reload(mode, debug, capfd):
    """Transition 10: reset() restores the estimates of the window loaded last, after a rebuild and after a values-only
    reload; optimize_from slices after a reload equal one optimize(n) of a fresh context."""
    a = _c3()
    b = slide(synth.ba_window(24, 2000, seed=11), 2, 16)
    b2 = new_values(b, 2)
    caps = caps_of([a, b])
    ba = context(caps, mode)
    load(ba, a, capfd, False)
    ba.optimize(6)
    for w, fast in ((b, False), (b2, True)):
        load(ba, w, capfd, fast)
        ba.optimize(6)
        ba.reset()
        p, l = ba.get()
        assert p.tobytes() == w.poses.tobytes() and l.tobytes() == w.points.tobytes()
        sts = []
        for k in range(8):
            nk, sk = ba.optimize(1, first_iteration=k)
            assert nk == 1
            sts.append(sk[0])
        fresh = context(caps, mode)
        fresh.set_problem(w)
        n, st = fresh.optimize(8)
        assert n == 8 and np.array(sts, st.dtype).tobytes() == st.tobytes()
        assert ba.get()[0].tobytes() == fresh.get()[0].tobytes() and ba.get()[1].tobytes() == fresh.get()[1].tobytes()
        fresh.close()


# ------------------------------------------------------------------------------------------------------------ failed loads
def assert_nothing_loaded(ba, P, L):
    """Every call that reads the window refuses (SE2GPU_ERR_INVALID); the buffers are sized for the rejected window."""
    lib = _capi.lib()
    st = np.zeros(8, _capi.BA_STATS_DTYPE)
    p, l = np.zeros((P, 3)), np.zeros((L, 3))
    pf, lf = np.zeros((P, 3), np.float32), np.zeros((L, 3), np.float32)
    chi = C.c_double()
    plan = np.zeros(len(LocalBA.PLAN_FIELDS), np.int32)
    inv = ERR_INVALID
    assert lib.se2gpu_ba_optimize_from(ba.h, 0, 8, None, _capi.ptr(st), None, None) == inv, "optimize ran a window"
    assert lib.se2gpu_ba_get(ba.h, _capi.ptr(p), _capi.ptr(l)) == inv, "get read a window"
    assert lib.se2gpu_ba_get_f32(ba.h, _capi.ptr(pf), _capi.ptr(lf)) == inv, "get_f32 read a window"
    assert lib.se2gpu_ba_reset(ba.h) == inv, "reset restored a window"
    assert lib.se2gpu_ba_debug_system(ba.h, 1.0, C.byref(chi), *([None] * 9)) == inv, "debug_system ran a window"
    assert lib.se2gpu_ba_debug_plan(ba.h, _capi.ptr(plan), len(plan)) == inv, "debug_plan reported a window"
    with pytest.raises(_capi.Se2GpuError):
        ba.get()


@gpu
@pytest.mark.parametrize("mode", MODES)
def test_failed_set_problem_leaves_no_window(mode, debug, capfd):
    """Transition 11: a rejected window (an edge to a missing pose, an odometry edge to a missing pose, more poses than the
    capacity) after a successful load leaves NO window loaded; the next valid load equals a fresh context's, also when it
    has the topology loaded before the failure. Every rejected window has at least the loaded window's P and L."""
    a = synth.ba_window(10, 600, seed=12)
    big = synth.ba_window(16, 1200, seed=13)
    caps = caps_of([a, big])
    bad_edge = bc._copy(big); bad_edge.edge_pose[3] = big.P
    bad_odo = bc._copy(big); bad_odo.odo_j[2] = big.P + 5
    too_big = synth.ba_window(caps[0] + 2, 1200, seed=14)
    ba = context(caps, mode)
    step(ba, a, 6, capfd, False, caps, mode)
    for bad, rc in ((bad_edge, ERR_INVALID), (bad_odo, ERR_INVALID), (too_big, ERR_CAPACITY)):
        assert bad.P >= a.P and bad.L >= a.L
        with pytest.raises(_capi.Se2GpuError, match=rf"\({rc}\)"):
            ba.set_problem(bad)
        assert_nothing_loaded(ba, bad.P, bad.L)
        step(ba, a, 6, capfd, False, caps, mode)           # the pre-failure topology: rebuilt, not refreshed
    with pytest.raises(_capi.Se2GpuError):
        ba.set_problem(bad_edge)
    step(ba, big, 6, capfd, False, caps, mode)


# ------------------------------------------------------------------------------------------------------------ shards
def run_shard_sequence(probs, world, iters, capfd, device=0, setup=None, mode=0):
    """tests/local_shards.run_local_shards over a SEQUENCE of windows: the ranks' contexts (sized for the largest window)
    stay alive and are loaded with one window after the other. Returns per window the per-rank (n, stats, trace_poses,
    trace_points, poses, points) and how many ranks took the values-only refresh."""
    dev = torch.device("cuda", device)
    world_barrier = threading.Barrier(world)
    step_barrier = threading.Barrier(world + 1)         # the ranks and this thread: one window at a time
    slots = [None] * world
    results = [[None] * world for _ in probs]
    fast = []
    errors = []
    streams = [torch.cuda.Stream(device=dev) for _ in range(world)]
    caps = caps_of(probs)
    bas = [None] * world

    def make_cb(rank):
        def allreduce(ptr, count, op, stream):
            torch.cuda.synchronize(dev)
            slots[rank] = _as_tensor(ptr, count, dev)
            world_barrier.wait()
            acc = slots[0].clone()
            for t in slots[1:]:
                acc = acc + t if op == 0 else torch.maximum(acc, t)
            torch.cuda.synchronize(dev)
            world_barrier.wait()
            slots[rank].copy_(acc)
            torch.cuda.synchronize(dev)
        return allreduce

    def worker(rank):
        try:
            torch.cuda.set_device(dev)
            with torch.cuda.stream(streams[rank]):
                ba = LocalBA(*caps, device=device)
                ba.set_mode(mode)
                ba.set_stream(streams[rank].cuda_stream)
                ba.set_shard(rank, world, make_cb(rank))
                bas[rank] = ba
                world_barrier.wait()
                if setup is not None and rank == 0:
                    setup(bas)
                world_barrier.wait()
                for k, prob in enumerate(probs):
                    step_barrier.wait()
                    ba.set_problem(prob)
                    world_barrier.wait()
                    n, st, tp, tl = ba.optimize(iters, trace=True)
                    p, l = ba.get()
                    results[k][rank] = (n, st, tp, tl, p, l)
                    step_barrier.wait()
        except Exception as e:      # noqa: BLE001
            errors.append((rank, e))
            world_barrier.abort()
            step_barrier.abort()

    threads = [threading.Thread(target=worker, args=(r,)) for r in range(world)]
    for t in threads:
        t.start()
    try:
        for _ in probs:
            capfd.readouterr()
            step_barrier.wait()
            step_barrier.wait()
            fast.append(capfd.readouterr().err.count(FAST))
    except threading.BrokenBarrierError:
        pass
    for t in threads:
        t.join(timeout=300)
    for ba in bas:
        if ba is not None:
            ba.close()
    if errors:
        raise errors[0][1]
    return results, fast


@gpu
@pytest.mark.parametrize("path", ["allreduce", "peer"])
def test_sharded_contexts_reused(path, debug, capfd):
    """Transition 12, world = 2 on one device: C3 -> C3 with new values (values-only on every rank) -> C3 with every 7th
    edge dropped (rebuild). Every rank equals, byte for byte, a fresh sharded run on that window."""
    kw = {}
    if path == "peer":
        debug.setenv("SE2GPU_BA_PK_GRID", pk_grid_share(2))
        debug.setenv("SE2GPU_BA_PEER_TIMEOUT_S", "20")
        kw = dict(setup=LocalBA.attach_local, mode=2)
    else:
        kw = dict(mode=1)
    a = _c3()
    b = new_values(a, 3)
    c = bc._copy(b)
    keep = np.ones(c.E, bool); keep[::7] = False
    bc._keep_edges(c, keep)
    seq = [a, b, c]
    res, fast = run_shard_sequence(seq, 2, 8, capfd, **kw)
    assert fast == [0, 2, 0]
    for k, w in enumerate(seq):
        ref = run_local_shards(w, 2, 8, **kw)
        for r in range(2):
            for got, want, what in zip(res[k][r], ref[r], ("n", "stats", "trace_poses", "trace_points", "poses", "points")):
                got_b = got if isinstance(got, int) else got.tobytes()
                want_b = want if isinstance(want, int) else want.tobytes()
                assert got_b == want_b, f"window {k} rank {r}: {what} differs from a fresh sharded run"


# ------------------------------------------------------------------------------------------------------------ drop-in header
def compile_reuse_demo(tmp_path):
    build.build_lib()
    exe = str(tmp_path / "shim_reuse_demo")
    libdir = os.path.dirname(build.LIB_PATH)
    cmd = ["g++", "-O1", "-std=c++14", "-Wall", "-I", os.path.join(ROOT, "include"), os.path.join(ROOT, "tests", "native", "shim_reuse_demo.cpp"),
           "-o", exe, "-L", libdir, "-lse2gpu", f"-Wl,-rpath,{libdir}"]
    res = subprocess.run(cmd, capture_output=True, text=True)
    assert res.returncode == 0, res.stderr
    return exe


def _write_window(f, prob, iters, delta_last=None):
    Rbc, tbc = synth.default_Tbc()
    f.write(struct.pack("iiiii", prob.P, prob.L, prob.E, prob.O, iters))
    for a, dt in ((prob.poses, "f8"), (prob.fixed, "u1"), (prob.points, "f8"), (prob.edge_pose, "i4"), (prob.edge_point, "i4"),
                  (prob.uv, "f8"), (prob.info, "f8"), (prob.odo_i, "i4"), (prob.odo_j, "i4"), (prob.odo_meas, "f8"), (prob.odo_info, "f8")):
        f.write(np.ascontiguousarray(a, dt).tobytes())
    f.write(np.array([prob.fx, prob.cx, prob.cy], "f8").tobytes())
    f.write(np.concatenate([Rbc.reshape(-1), tbc]).astype("f8").tobytes())
    f.write(struct.pack("dd", prob.huber_delta, prob.huber_delta if delta_last is None else delta_last))


def _read_window(buf, off, prob):
    ok, done = struct.unpack_from("ii", buf, off); off += 8
    poses = np.frombuffer(buf, "f8", 3 * prob.P, off).reshape(-1, 3); off += 24 * prob.P
    pts = np.frombuffer(buf, "f8", 3 * prob.L, off).reshape(-1, 3); off += 24 * prob.L
    return (ok, done, poses, pts), off


def test_reuse_demo_compiles_and_links(tmp_path):
    compile_reuse_demo(tmp_path)


@gpu
def test_reused_slam_optimizer_matches_fresh_ones_and_rejects_cleanly(tmp_path):
    """One SlamOptimizer through: window A; clear() and a smaller B; clear() and a C beyond the context's capacity (the
    destroy / recreate branch); clear() and a graph D with two Huber deltas and at least C's P and L, which
    initializeOptimization rejects; then C again, with one more edge of another Huber delta added to the loaded graph.
    A, B and C equal the same windows on new SlamOptimizers byte for byte, and the oracle; after each rejection optimize()
    returns -1 and leaves every vertex estimate as it was."""
    exe = compile_reuse_demo(tmp_path)
    A, B, Cw = synth.ba_window(10, 600, seed=21), synth.ba_window(6, 300, seed=22), synth.ba_window(24, 1500, seed=23)
    D = synth.ba_window(24, 1600, seed=24)
    wins = [(A, None), (B, None), (Cw, None), (D, 2 * D.huber_delta)]
    assert Cw.P > A.P + A.P // 2 + 8                       # beyond the capacity the optimizer sized for A
    assert D.P >= Cw.P and D.L >= Cw.L
    fin = str(tmp_path / "reuse_in.bin")
    with open(fin, "wb") as f:
        f.write(struct.pack("i", len(wins)))
        for w, dl in wins:
            _write_window(f, w, 10, dl)
    out = {}
    for how in ("reuse", "fresh"):
        fout = str(tmp_path / f"reuse_out_{how}.bin")
        res = subprocess.run([exe, fin, fout, how], capture_output=True, text=True)
        assert res.returncode == 0, res.stderr
        buf = open(fout, "rb").read()
        off, got = 0, []
        for w, _ in wins + [(Cw, None)]:
            r, off = _read_window(buf, off, w)
            got.append(r)
        assert off == len(buf)
        out[how] = got
    for k, (w, _) in enumerate(wins[:3]):
        ok, done, poses, pts = out["reuse"][k]
        ok_f, done_f, poses_f, pts_f = out["fresh"][k]
        assert ok == ok_f == 1 and done == done_f
        assert poses.tobytes() == poses_f.tobytes() and pts.tobytes() == pts_f.tobytes(), f"window {'ABC'[k]}"
        o = pyoracle.BAOracle(w)
        n_o, _ = o.optimize(10)
        po, lo = o.get()
        assert done == n_o
        np.testing.assert_allclose(poses, po, atol=1e-8)
        np.testing.assert_allclose(pts, lo, atol=1e-7)
    for how in ("reuse", "fresh"):
        ok, done, poses, pts = out[how][3]
        assert ok == 0 and done == -1, f"{how}: graph D was optimised"
        assert poses.tobytes() == D.poses.tobytes() and pts.tobytes() == D.points.tobytes()
        ok, done, poses, pts = out[how][4]
        assert ok == 0 and done == -1, f"{how}: the rejected reload of C ran the window loaded before"
        assert poses.tobytes() == out[how][2][2].tobytes() and pts.tobytes() == out[how][2][3].tobytes()
