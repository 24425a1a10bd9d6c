"""The SE(3)-XYZ window BA on the GPU (se2gpu_se3_ba) over the directly built windows of
tools/se3_window_synth.DIRECT_SCENES — reference-shaped layouts, long tracks and a full envelope, a loop closure, rotations
in every branch of quat_from_R, empty and one-keyframe windows, chunk boundaries and a window larger than the grid —
against the C++ oracle with tests/test_se3_ba_gpu.py's bounds; and the paths those scenes reach: a permuted window, the
cooperative grid capped by SE2GPU_SE3_BA_GRID (the bytes must not depend on the grid size), one context's device entry
on two streams, and one context across windows that grow and shrink."""
from __future__ import annotations

import ctypes as C

import numpy as np
import pytest

from oracle import pyse3ba
from se2lam_b200 import _capi, se3ba
from tests.test_se3_ba_gpu import compare
from tools import se3_window_synth as S

pytestmark = pytest.mark.gpu

NAMES = sorted(S.DIRECT_SCENES)


def scene(name):
    f, iterations = S.DIRECT_SCENES[name]
    return f(False), S.direct_params(iterations)


def outside_graph(w):
    """keyframes g2o does not optimise: fixed, or touched by no edge, odometry link or prior"""
    active = w.prior.astype(bool).copy()
    active[w.odo_from] = True; active[w.odo_to] = True; active[w.edge_kf] = True
    return np.nonzero((w.fixed != 0) | ~active)[0]


def same_bytes(a, b):
    for k in ("status", "iterations"):
        assert a[k] == b[k], k
    for k in ("chi2", "outlier", "poses", "points", "stats", "Tcw", "xyz", "trace"):
        if k in a or k in b:
            assert a[k].tobytes() == b[k].tobytes(), k


@pytest.mark.parametrize("name", NAMES)
def test_against_oracle(name):
    w, prm = scene(name)
    g, o = se3ba.local_se3_ba(w, prm), pyse3ba.run(w, prm)
    assert g["iterations"] == o["iterations"]
    compare(g, o)
    kept = outside_graph(w)
    assert np.array_equal(g["Tcw"][kept].view(np.uint32), w.Tcw.reshape(-1, 4, 4)[kept].view(np.uint32))
    edgeless = np.setdiff1d(np.arange(len(w.xyz)), w.edge_point)
    assert np.array_equal(g["xyz"][edgeless].view(np.uint32), w.xyz[edgeless].view(np.uint32))


@pytest.mark.parametrize("name", ["local_graph", "loop_closure", "only_ba_x", "dense"])
def test_permuted_window_gives_the_unpermuted_result(name):
    w, prm = scene(name)
    w2, (pk, pp, po, pe) = S.permute(w, np.random.default_rng(5))
    g2 = se3ba.local_se3_ba(w2, prm)
    g = dict(g2)
    g["poses"] = np.empty_like(g2["poses"]); g["poses"][pk] = g2["poses"]
    g["points"] = np.empty_like(g2["points"]); g["points"][pp] = g2["points"]
    g["chi2"] = np.empty_like(g2["chi2"]); g["chi2"][pe] = g2["chi2"]
    g["outlier"] = np.empty_like(g2["outlier"]); g["outlier"][pe] = g2["outlier"]
    o = pyse3ba.run(w, prm)
    assert g["iterations"] == o["iterations"]
    compare(g, o)


def _c4():
    f, iterations = S.SCENES["c4"]
    prob, w = f()
    return w, S.window_params(prob, iterations=iterations)


GRID_SCENES = ["c4", "dense"] + [f"{k}_{n}" for k in ("items", "points") for n in (255, 256, 257)]


@pytest.mark.parametrize("name", GRID_SCENES)
def test_grid_cap_changes_no_byte(name, monkeypatch):
    """every sum is taken over fixed chunks of 256 items, added in chunk order: a grid of 1, 2, 3 or 7 CTAs (every CTA
    walking several chunks, and every strided loop several rounds) gives the bytes of the natural grid"""
    w, prm = _c4() if name == "c4" else scene(name)
    runs = []
    for grid in (None, 1, 2, 3, 7):
        if grid is None:
            monkeypatch.delenv("SE2GPU_SE3_BA_GRID", raising=False)
        else:
            monkeypatch.setenv("SE2GPU_SE3_BA_GRID", str(grid))
        ctx = se3ba.Context()  # the variable is read when the context is created
        try:
            runs.append((ctx.run(w, prm), ctx.run(w, prm, trace=True)))
        finally:
            ctx.close()
    assert runs[0][0]["iterations"] > 0
    for r in runs[1:]:
        same_bytes(r[0], runs[0][0])
        same_bytes(r[1], runs[0][1])


def _launch(ctx, w, prm, stream):
    """se2gpu_se3_ba_device on `stream`, inputs and outputs allocated on it; returns the output tensors without waiting"""
    import torch
    N, O, L, E = w.sizes
    with torch.cuda.stream(stream):
        t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to("cuda", non_blocking=False)  # noqa: E731
        ins = [t(w.Tcw), t(w.odo_measure), t(w.odo_info), t(w.xyz), t(w.uv), t(w.inv_sigma2)]
        z = lambda n, dt: torch.zeros(n, dtype=dt, device="cuda")  # noqa: E731
        out = dict(chi2=z(max(E, 1), torch.float64), outlier=z(max(E, 1), torch.uint8), status=z(1, torch.int32), iters=z(1, torch.int32),
                   stats=z(max(prm.iterations, 1) * _capi.BA_STATS_DTYPE.itemsize, torch.uint8), poses=z(N * 7, torch.float64),
                   points=z(max(L, 1) * 3, torch.float64), Tcw=z(N * 16, torch.float32), xyz=z(max(L, 1) * 3, torch.float32))
    p = _capi.ptr
    dT, dm, di, dx, du, dw = ins
    _capi.check(_capi.lib().se2gpu_se3_ba_device(
        ctx.h, N, p(dT), p(w.fixed), p(w.prior), O, p(w.odo_from), p(w.odo_to), p(dm), p(di), L, p(dx), E, p(w.edge_point),
        p(w.edge_kf), p(du), p(dw), C.addressof(prm), p(out["chi2"]), p(out["outlier"]), p(out["status"]), p(out["iters"]),
        p(out["stats"]), p(out["poses"]), p(out["points"]), p(out["Tcw"]), p(out["xyz"]), C.c_void_p(stream.cuda_stream)),
        "se2gpu_se3_ba_device")
    return out, ins


def test_device_entry_on_two_streams():
    """a large window on stream A, then a small one on stream B, through one context with no wait in between: the second
    call's plan upload and buffers must not disturb what the first kernel reads"""
    import torch
    big, small = scene("large"), scene("local_graph")
    ctx = se3ba.Context()
    a, b = torch.cuda.Stream(), torch.cuda.Stream()
    first, keep_a = _launch(ctx, *big, a)
    second, keep_b = _launch(ctx, *small, b)
    a.synchronize(); b.synchronize()
    ctx.close()
    for (w, prm), got in ((big, first), (small, second)):
        ref = se3ba.local_se3_ba(w, prm)
        N, O, L, E = w.sizes
        n = int(got["iters"].cpu()[0])
        assert n == ref["iterations"] and int(got["status"].cpu()[0]) == ref["status"]
        assert got["chi2"].cpu().numpy()[:E].tobytes() == ref["chi2"].tobytes()
        assert got["outlier"].cpu().numpy()[:E].astype(bool).tobytes() == ref["outlier"].tobytes()
        assert got["poses"].cpu().numpy().tobytes() == ref["poses"].tobytes()
        assert got["points"].cpu().numpy()[:3 * L].tobytes() == ref["points"].tobytes()
        assert got["Tcw"].cpu().numpy().tobytes() == ref["Tcw"].tobytes()
        assert got["xyz"].cpu().numpy()[:3 * L].tobytes() == ref["xyz"].tobytes()
        st = np.frombuffer(got["stats"].cpu().numpy().tobytes(), _capi.BA_STATS_DTYPE)[:n]
        assert st.tobytes() == ref["stats"].tobytes()


def test_one_context_across_growing_and_shrinking_windows():
    ctx = se3ba.Context()
    for name in ("items_255", "large", "one_kf", "dense", "no_points", "loop_closure", "only_ba_no_edges", "points_257",
                 "edgeless", "only_ba_y", "one_kf_fixed", "large", "shuffled"):
        w, prm = scene(name)
        same_bytes(ctx.run(w, prm), se3ba.local_se3_ba(w, prm))
    ctx.close()
