"""Batched local BA (se2gpu_ba_optimize_batch): many windows in one launch, one thread-block cluster per window.

The central claim: the cluster kernel runs the persistent kernel's arithmetic on C CTAs. Every window of a batch therefore
gives the bytes - iteration count, stats, per-iteration traces, get() and get_f32() - of a fresh single context optimising it
in persistent mode under SE2GPU_BA_PK_GRID = C, where C is the cluster size the library picked for it (batch_cluster()). The
windows between them reach every cluster size; each also holds test_ba_gpu's strict bar against the CPU oracle.
"""
import numpy as np
import pytest

from oracle import pyoracle
from se2lam_b200 import _capi
from se2lam_b200.ba import LocalBA
from tests import ba_cases as bc
from tests.test_ba_gpu import REJECTING, REL, _perturbed
from tools import synth

pytestmark = pytest.mark.gpu

ITERS = 8
STRICT_NAMES = ["twist_w6", "twist_w16", "smem_w17", "chain_nf16", "smem_nf52", "dense_nf29", "dense_arena", "tail_nf23",
                "broken_nf29", "reversed_nf28", "duplicated_nf28", "loop_nf39", "sparse_nf29"]


def _windows():
    """name -> (problem, iterations): C3, C4, the STRICT cases with n <= 156 and one window that rejects trials."""
    w = {"C3": (synth.ba_config("C3"), 10), "C4": (synth.ba_config("C4"), 10)}
    for name in STRICT_NAMES:
        w[name] = bc.strict(name)
    w["rejecting"] = (_perturbed(*REJECTING[0]), 12)
    return w


@pytest.fixture(scope="module")
def windows():
    return _windows()


def _result(ba, out):
    """Everything a caller can read after an optimize: (n, stats, traces) bytes and the estimates as double and float."""
    n, st, tp, tl = out
    poses, pts = ba.get()
    fp, fl = ba.get_f32()
    return (n, st.tobytes(), tp.tobytes(), tl.tobytes(), poses.tobytes(), pts.tobytes(), fp.tobytes(), fl.tobytes())


def _context(prob, monkeypatch, grid=None, mode=0, cluster=None):
    """A context created with SE2GPU_BA_PK_GRID = grid (None: the default grid) and SE2GPU_BA_BATCH_CLUSTER = cluster (None:
    the library's size, 8); the BA reads both at creation."""
    for k, v in (("SE2GPU_BA_PK_GRID", grid), ("SE2GPU_BA_BATCH_CLUSTER", cluster)):
        if v is None:
            monkeypatch.delenv(k, raising=False)
        else:
            monkeypatch.setenv(k, str(v))
    ba = LocalBA.from_problem(prob, mode=mode)
    monkeypatch.delenv("SE2GPU_BA_PK_GRID", raising=False)
    monkeypatch.delenv("SE2GPU_BA_BATCH_CLUSTER", raising=False)
    return ba


def _single(prob, iters, C, monkeypatch):
    ba = _context(prob, monkeypatch, grid=C, mode=2)
    return _result(ba, ba.optimize(iters, trace=True))


def _batch(probs, iters, monkeypatch, stop_flags=None):
    bas = [_context(p, monkeypatch) for p in probs]
    outs = LocalBA.optimize_batch(bas, iters, trace=True, stop_flags=stop_flags)
    return bas, [_result(ba, o) for ba, o in zip(bas, outs)]


def _assert_oracle(prob, iters, n_g, st_g, tp_g, tl_g):
    """test_ba_gpu's strict bar: trials / accepted / terminate, lambda to 1e-6, chi2 to 1e-8, every per-step update to 1e-5."""
    n_o, st_o, tp_o, tl_o = pyoracle.BAOracle(prob).optimize(iters, trace=True)
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


FORCED = {"C3": 2, "chain_nf16": 4, "rejecting": 2, "tail_nf23": 4}   # extra copies at the sizes only the switch selects


def test_mixed_batch_equals_single_contexts_and_the_oracle(windows, monkeypatch):
    names = list(windows) + [f"{k}@{c}" for k, c in FORCED.items()]
    probs = [windows[k.split("@")[0]][0] for k in names]
    bas = [_context(p, monkeypatch, cluster=int(k.split("@")[1]) if "@" in k else None) for k, p in zip(names, probs)]
    sizes = {name: ba.batch_cluster() for name, ba in zip(names, bas)}
    assert {sizes[k] for k in windows} == {8} and set(sizes.values()) == {2, 4, 8}, sizes
    iters = max(it for _, it in windows.values())
    n0 = _capi.lib().se2gpu_launch_count()
    outs = LocalBA.optimize_batch(bas, iters, trace=True)
    assert _capi.lib().se2gpu_launch_count() - n0 == 3
    for name, ba, prob, out in zip(names, bas, probs, outs):
        assert _result(ba, out) == _single(prob, iters, sizes[name], monkeypatch), name
        n, st, tp, tl = out
        it = windows[name.split("@")[0]][1]   # the iteration count the window was screened at: LM iteration k does not see later ones
        _assert_oracle(prob, it, min(n, it), st[:it], tp[:it], tl[:it])


def test_batched_context_runs_the_plan_for_its_cluster_size(windows, monkeypatch):
    """After a batch a context holds decide()'s plan for its cluster size - the serving order and the mirrored envelope equal
    those of a fresh context created at that grid - and a single optimize afterwards holds the plan for its own grid again."""
    names = ("C3", "C4", "chain_nf16", "rejecting", "twist_w6")
    bas = [_context(windows[k][0], monkeypatch) for k in names]
    own = [{a: ba.debug_structure(a).tobytes() for a in ("blk_order", "tw_cmax1")} for ba in bas]
    LocalBA.optimize_batch(bas, 2)
    for name, ba in zip(names, bas):
        ref = _context(windows[name][0], monkeypatch, grid=ba.batch_cluster())
        for a in ("blk_order", "tw_cmax1"):
            assert ba.debug_structure(a).tobytes() == ref.debug_structure(a).tobytes(), (name, a)
    assert any(own[k]["blk_order"] != bas[k].debug_structure("blk_order").tobytes() for k in range(len(bas)))
    for ba, o in zip(bas, own):
        ba.reset()
        ba.optimize(1)
        assert {a: ba.debug_structure(a).tobytes() for a in ("blk_order", "tw_cmax1")} == o


def _tilted(prob, a=0.03, b=0.02):
    """The window seen through a camera pitched and rolled on the body: no extrinsic product is exact any more."""
    q = bc._copy(prob)
    ca, sa, cb, sb = np.cos(a), np.sin(a), np.cos(b), np.sin(b)
    Ry = np.array([[ca, 0, sa], [0, 1, 0], [-sa, 0, ca]])
    Rx = np.array([[1, 0, 0], [0, cb, -sb], [0, sb, cb]])
    Rcb = Rx @ Ry @ np.asarray(prob.Tcb[:9]).reshape(3, 3)
    q.Tcb = np.concatenate([Rcb.reshape(-1), np.asarray(prob.Tcb[9:]) + [0.013, -0.007, 0.021]])
    return q


def test_general_extrinsic_equals_single_contexts(windows, monkeypatch):
    """A camera whose Rcb products round: the cluster kernel contracts edge_xyz as ba_persistent does."""
    probs = [_tilted(windows[k][0]) for k in ("C3", "C4", "chain_nf16", "rejecting", "twist_w16", "loop_nf39")]
    probs.append(_tilted(synth.ba_window(10, 400, seed=21)))
    assert not np.all(np.isin(np.asarray(probs[0].Tcb[:9]), (-1.0, 0.0, 1.0)))
    bas = [_context(p, monkeypatch, cluster=c) for p, c in zip(probs, (None, None, 4, 2, None, 4, 2))]
    res = [_result(b, o) for b, o in zip(bas, LocalBA.optimize_batch(bas, ITERS, trace=True))]
    assert {ba.batch_cluster() for ba in bas} == {2, 4, 8}
    for ba, prob, r in zip(bas, probs, res):
        assert r == _single(prob, ITERS, ba.batch_cluster(), monkeypatch)


def test_result_is_independent_of_the_batch(windows, monkeypatch):
    prob = windows["tail_nf23"][0]
    alone = _batch([prob], ITERS, monkeypatch)[1][0]
    others8 = [synth.ba_window(10, 400, seed=100 + k) for k in range(6)] + [windows["C4"][0]]

    def batch_with_forced(probs, forced):   # the windows of `forced` positions on clusters of 2 CTAs: another launch next to it
        bas = [_context(p, monkeypatch, cluster=2 if k in forced else None) for k, p in enumerate(probs)]
        return [_result(b, o) for b, o in zip(bas, LocalBA.optimize_batch(bas, ITERS, trace=True))]
    first = batch_with_forced([prob] + others8, {1, 2, 3})
    last = batch_with_forced(others8 + [prob], {0, 1, 2})
    assert first[0] == alone and last[7] == alone
    big = _batch([synth.ba_window(8, 200, seed=200 + k) for k in range(40)] + [prob] +
                 [synth.ba_window(20, 600, seed=300 + k) for k in range(23)], ITERS, monkeypatch)[1]
    assert big[40] == alone
    assert first[1] == last[0]         # a filler moves position and neighbours, its bytes stay


def _expect_error(code, bas, iters=ITERS):
    with pytest.raises(_capi.Se2GpuError) as e:
        LocalBA.optimize_batch(bas, iters)
    assert f"({code})" in str(e.value), str(e.value)
    return str(e.value)


def test_refusals_change_nothing(windows, monkeypatch):
    small = [synth.ba_window(10, 400, seed=400 + k) for k in range(4)]
    large, _ = bc.strict("large_nf53")
    probs = small[:3] + [large] + [small[3]]
    bas = [_context(p, monkeypatch) for p in probs]
    before = [ba.get() for ba in bas]
    st = np.zeros((len(bas), ITERS), _capi.BA_STATS_DTYPE)
    its = np.full(len(bas), -7, np.int32)
    arr = (_capi.C.c_void_p * len(bas))(*[b.h for b in bas])
    rc = _capi.lib().se2gpu_ba_optimize_batch(arr, len(bas), ITERS, None, _capi.ptr(its), _capi.ptr(st), None, None)
    assert rc == -4 and "window 3" in _capi.last_error()         # n = 159 at position 3
    assert np.all(its == -7) and not st.tobytes().strip(b"\0")   # nothing written to the caller's buffers either
    unloaded = LocalBA(10, 400, 4000, 20)
    sharded = _context(small[0], monkeypatch)
    sharded.set_shard(1, 2, lambda *a: None)
    sharded.set_problem(small[0])
    multi = _context(small[1], monkeypatch, mode=1)
    assert "window 1" in _expect_error(-3, [bas[0], None])
    assert "window 2" in _expect_error(-3, [bas[0], bas[1], bas[0]])
    assert "window 1" in _expect_error(-3, [bas[0], unloaded])
    assert "window 1" in _expect_error(-3, [bas[0], sharded])
    assert "window 1" in _expect_error(-3, [bas[0], multi])
    _expect_error(-4, [bas[0]], iters=65)                         # above the stats capacity
    for ba, (p, l) in zip(bas, before):
        p2, l2 = ba.get()
        assert p2.tobytes() == p.tobytes() and l2.tobytes() == l.tobytes()
    for ba, p in zip(bas, probs):                                 # the next single optimize (stats, traces, estimates) is a fresh context's
        fresh = _context(p, monkeypatch)
        assert _result(ba, ba.optimize(ITERS, trace=True)) == _result(fresh, fresh.optimize(ITERS, trace=True))


def test_degenerate_windows_next_to_normal_ones(windows, monkeypatch):
    fixed = synth.ba_window(10, 400, seed=7)
    fixed.fixed = np.ones_like(fixed.fixed)
    nonpd_small = bc.nonpd(synth.ba_window(30, 1500, seed=3))
    nonpd_twist = bc.nonpd(bc.strict("twist_w10")[0])
    probs = [windows["C3"][0], fixed, nonpd_small, windows["rejecting"][0], nonpd_twist]
    bas, res = _batch(probs, ITERS, monkeypatch)
    for ba, prob, r in zip(bas, probs, res):
        assert r == _single(prob, ITERS, ba.batch_cluster(), monkeypatch)


def test_stop_flag_set_before_the_call(windows, monkeypatch):
    probs = [windows["C3"][0], synth.ba_window(10, 400, seed=9), windows["chain_nf16"][0]]
    flags = [None, np.ones(1, np.uint8), np.zeros(1, np.uint8)]
    bas, res = _batch(probs, ITERS, monkeypatch, stop_flags=flags)
    assert res[1][0] == 0
    poses, pts = bas[1].get()
    assert poses.tobytes() == probs[1].poses.tobytes() and pts.tobytes() == probs[1].points.tobytes()
    for k in (0, 2):
        assert res[k] == _single(probs[k], ITERS, bas[k].batch_cluster(), monkeypatch)


def test_reuse_across_batches_reloads_and_a_single_optimize(windows, monkeypatch):
    a, b, c = windows["C3"][0], windows["chain_nf16"][0], synth.ba_window(10, 400, seed=11)
    b2 = windows["C4"][0]
    monkeypatch.delenv("SE2GPU_BA_PK_GRID", raising=False)
    bas = [_context(a, monkeypatch), LocalBA(b2.P, b2.L, b2.E, b2.O), _context(c, monkeypatch)]   # room for b2's rebuild
    bas[1].set_problem(b)
    outs = LocalBA.optimize_batch(bas, ITERS, trace=True)
    for ba, p, o in zip(bas, (a, b, c), outs):
        assert _result(ba, o) == _single(p, ITERS, ba.batch_cluster(), monkeypatch)
    # values-only refresh (same graph, moved estimates) and a rebuild with another window
    a2 = bc._copy(a)
    a2.poses = a.poses + 1e-3 * np.arange(a.P * 3).reshape(a.P, 3) * (1 - a.fixed[:, None])
    bas[0].set_problem(a2)
    bas[1].set_problem(b2)
    extra = _context(synth.ba_window(12, 500, seed=12), monkeypatch)
    step2 = [bas[0], bas[1], extra]
    outs = LocalBA.optimize_batch(step2, ITERS, trace=True)
    for ba, p, o in zip(step2, (a2, b2, synth.ba_window(12, 500, seed=12)), outs):
        assert _result(ba, o) == _single(p, ITERS, ba.batch_cluster(), monkeypatch)
    # a single optimize afterwards plans for the context's own grid again
    bas[1].reset()
    fresh = _context(b2, monkeypatch)
    assert _result(bas[1], bas[1].optimize(ITERS, trace=True)) == _result(fresh, fresh.optimize(ITERS, trace=True))


def test_one_launch_per_cluster_size(windows, monkeypatch):
    lib = _capi.lib()
    for names, forced in ((["C3"], ()), (["C3", "chain_nf16", "C4"], ()), (["C3", "chain_nf16", "rejecting", "tail_nf23"], (1, 3)),
                          (["C3", "C4", "rejecting", "tail_nf23"], (0, 2))):
        bas = [_context(windows[k][0], monkeypatch, cluster=(2 if i == forced[0] else 4) if i in forced else None)
               for i, k in enumerate(names)]
        sizes = {ba.batch_cluster() for ba in bas}
        n0 = lib.se2gpu_launch_count()
        LocalBA.optimize_batch(bas, 3)
        assert lib.se2gpu_launch_count() - n0 == len(sizes)
