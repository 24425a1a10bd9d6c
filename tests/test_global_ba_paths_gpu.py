"""se2gpu_global_ba on the graphs of tests/test_global_ba_paths_oracle.py against the CPU oracle: fixed sets other than
vertex 0 alone, dense envelopes and the 256-thread strides; the device entry's d_edge_status with non-finite values in
the skipped slots; the NOT_PD ending; the chained feat_edge -> global_ba device path at scale; one context across dense and
sparse envelopes; and the map-point write-back at its block boundaries."""
import ctypes as C

import numpy as np
import pytest

from oracle import pyglobal
from se2lam_b200 import _capi, featgraph, globalba
from tests import test_global_ba_gpu as G
from tests import test_global_ba_paths_oracle as P
from tools import posegraph_synth as S

pytestmark = pytest.mark.gpu

SEVERAL_FIXED = ("loop_fixed_middle", "loop_fixed_last", "chain_split_in_four", "covisibility_fixed_pairs", "loop_all_but_one_fixed")


def check_parity(g, o, name):
    """tests/test_global_ba_gpu.py::check_parity with this scene's bound on the absolute estimates (P.est_atol), and the
    poses relative to vertex 0 at the usual estimate bar."""
    assert g["status"] == o["status"]
    n = G.compared_iterations(o["stats"])
    assert g["iterations"] >= n
    gs, os_ = g["stats"][:n], o["stats"][:n]
    for f in ("trials", "accepted", "terminate"):
        assert np.array_equal(gs[f], os_[f]), f
    for f in ("chi2_before", "chi2_after"):
        np.testing.assert_allclose(gs[f], os_[f], rtol=G.CHI2_RTOL, atol=G.CHI2_ATOL, err_msg=f)
    np.testing.assert_allclose(gs["lambda"], os_["lambda"], rtol=G.LAMBDA_RTOL)
    np.testing.assert_allclose(g["poses"], o["poses"], rtol=0, atol=P.est_atol(name))
    np.testing.assert_allclose(P.relative_poses(g["poses"]), P.relative_poses(o["poses"]), rtol=0, atol=G.EST_ATOL)
    assert G.float_close(g["Tcw"], o["Tcw"], ulps=64)


@pytest.fixture(scope="module")
def scenes():
    return {k: f() for k, f in P.SCENES.items()}


def all_fixed(s):
    return dict(s, fixed=np.ones(len(s["Tcw"]), np.uint8))


@pytest.mark.parametrize("name", list(P.SCENES))
def test_global_ba_matches_oracle(scenes, name):
    s = scenes[name]
    prm = globalba.params(s["Tbc"])
    g = globalba.GlobalBA(s["Tcw"], s["fixed"], s["edges"], prm)
    o = pyglobal.run(s, pyglobal.params(s["Tbc"]))
    check_parity(g, o, name)
    fixed = np.asarray(s["fixed"], bool)
    if fixed.all():
        assert g["iterations"] == o["iterations"] == 0
        z = globalba.GlobalBA(s["Tcw"], s["fixed"], s["edges"], globalba.params(s["Tbc"], iterations=0))
        assert g["Tcw"].tobytes() == z["Tcw"].tobytes() and g["poses"].tobytes() == z["poses"].tobytes()
    else:
        assert g["iterations"] > 0
    if name in SEVERAL_FIXED:
        a = all_fixed(s)
        f = globalba.GlobalBA(a["Tcw"], a["fixed"], a["edges"], prm)
        assert f["iterations"] == 0
        assert g["Tcw"][fixed].tobytes() == f["Tcw"][fixed].tobytes()
        assert g["poses"][fixed].tobytes() == f["poses"][fixed].tobytes()


def _device(ctx, s, prm, status=None, measure=None, info=None):
    """se2gpu_global_ba_device on s's edges, with measure / info [E,16] / [E,36] in place of s's when given and status
    [E] as d_edge_status."""
    import torch
    fr, to, me, inf = globalba.edge_arrays(s["edges"])
    me = me if measure is None else measure
    inf = inf if info is None else info
    N = len(s["Tcw"])
    dev = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()
    d_status = None if status is None else dev(np.asarray(status, np.int32))
    return G._device_call(ctx, s, prm, N, fr, to, dev(np.asarray(s["Tcw"], np.float32).reshape(N, 16)), dev(me), dev(inf), d_status)


def test_device_edge_status_skips_too_few_and_counts_every_other_status():
    """d_edge_status mixing OK, NOT_PD and TOO_FEW on 300 keyframes. The TOO_FEW slots hold NaN and +-inf, as a caller's
    uninitialised arrays may; one of them is the only link between two components and one the only edge of vertex 299,
    which keeps nothing but its prior. The result is the graph without the TOO_FEW edges (host entry and oracle), the same
    bytes as with finite values in those slots, and an edge of status NOT_PD counts."""
    g, status = P.status_graph()
    prm = globalba.params(g["Tbc"])
    _, _, me, inf = globalba.edge_arrays(g["edges"])
    skip = np.flatnonzero(status == 1)
    junk_me, junk_inf = me.copy(), inf.copy()
    fills = (np.nan, np.inf, -np.inf)
    for k, e in enumerate(skip):
        junk_me[e] = fills[k % 3]
        junk_inf[e] = fills[(k + 1) % 3]
        junk_inf[e, ::7] = np.nan
    ctx = globalba.Context(0)
    # a first call that counts every slot, junk included, leaves non-finite linearisation records of the skipped edges in
    # the context's work buffer: the skipped edges' records must never be read, whatever they hold
    _device(ctx, g, prm, np.zeros_like(status), junk_me, junk_inf)
    d = _device(ctx, g, prm, status, junk_me, junk_inf)
    finite = _device(ctx, g, prm, status)
    fresh = globalba.Context(0)
    first = _device(fresh, g, prm, status)
    fresh.close()
    for k in ("Tcw", "poses", "stats"):
        assert d[k].tobytes() == finite[k].tobytes() == first[k].tobytes(), k
    assert (d["status"], d["iterations"]) == (finite["status"], finite["iterations"])
    assert np.isfinite(d["poses"]).all() and np.isfinite(d["stats"]["chi2_after"]).all()
    reduced = P.without(g, skip)
    h = ctx.run(reduced["Tcw"], reduced["fixed"], reduced["edges"], prm)
    o = pyglobal.run(reduced, pyglobal.params(g["Tbc"]))
    check_parity(h, o, "status_300_skipped_removed")
    check_parity(d, o, "status_300_skipped_removed")
    check_parity(d, h, "status_300_skipped_removed")
    # the NOT_PD-status edges are counted: leaving one of them out as well moves the result far past the bars
    one = int(np.flatnonzero(status == 2)[0])
    less = P.without(g, list(skip) + [one])
    h2 = ctx.run(less["Tcw"], less["fixed"], less["edges"], prm)
    assert np.abs(h2["poses"] - d["poses"]).max() > 100 * G.EST_ATOL
    assert abs(h2["stats"]["chi2_after"][-1] - d["stats"]["chi2_after"][-1]) > 1e-6 * d["stats"]["chi2_after"][-1]
    ctx.close()


@pytest.mark.parametrize("name", ["chain_10", "loop_none_fixed"])
def test_not_pd_ending_through_the_device_entry(name):
    """An infinite information entry, which only the device entry accepts: the oracle's trajectory word for word (a failed
    factorisation accepted at chi2 inf -> DBL_MAX, then rho = 0 and NOT_PD), and the estimate left at the start."""
    s = (G.SCENES.get(name) or P.SCENES[name])()
    s["edges"] = P.infinite_first_info(s["edges"])
    prm = globalba.params(s["Tbc"])
    ctx = globalba.Context(0)
    d = _device(ctx, s, prm)
    z = _device(ctx, s, globalba.params(s["Tbc"], iterations=0))
    ctx.close()
    o = pyglobal.run(s, pyglobal.params(s["Tbc"]))
    assert d["status"] == o["status"] == globalba.NOT_PD
    assert d["iterations"] == o["iterations"] == 2 and z["iterations"] == 0
    for f in ("trials", "accepted", "terminate"):
        assert np.array_equal(d["stats"][f], o["stats"][f]), f
    for f in ("chi2_before", "chi2_after"):
        assert d["stats"][f].tobytes() == o["stats"][f].tobytes(), f
    assert d["stats"]["chi2_before"][0] == np.inf and d["stats"]["chi2_after"][0] == np.finfo(np.float64).max
    assert d["Tcw"].tobytes() == z["Tcw"].tobytes() and d["poses"].tobytes() == z["poses"].tobytes()


def test_feat_edge_device_chained_into_global_ba_device_at_scale():
    """48 keyframe pairs through se2gpu_feat_edge_device, 24 in each mode, with point counts on both sides of min_points
    and of the 192-point staging, written into slices of a 200-keyframe graph's edge arrays pre-filled with NaN; then
    se2gpu_global_ba_device on the same stream. The TOO_FEW slots keep their NaN and are left out."""
    import torch
    g, pairs = P.feat_graph()
    fprm = featgraph.params(pairs[0][0][2]["Tbc"])
    Eo = len(g["edges"])
    links = [(a, b) for m in (0, 1) for a, b, _ in pairs[m]]
    fr = np.array([e[0] for e in g["edges"]] + [a for a, _ in links], np.int32)
    to = np.array([e[1] for e in g["edges"]] + [b for _, b in links], np.int32)
    _, _, me, inf = globalba.edge_arrays(g["edges"])
    E = Eo + len(links)
    dm = torch.full((E, 16), float("nan"), dtype=torch.float32, device="cuda"); dm[:Eo] = torch.from_numpy(me).cuda()
    di = torch.full((E, 36), float("nan"), dtype=torch.float32, device="cuda"); di[:Eo] = torch.from_numpy(inf).cuda()
    dstat = torch.zeros(E, dtype=torch.int32, device="cuda")
    stream = torch.cuda.current_stream().cuda_stream
    p_ = _capi.ptr
    keep = []
    for mode in (0, 1):
        ps = [p for _, _, p in pairs[mode]]
        cat = lambda k, w, dt: torch.from_numpy(np.concatenate([np.asarray(p[k], dt).reshape(-1, w) for p in ps])).cuda()
        counts = [len(p["xyz"]) for p in ps]
        pp = torch.tensor(np.r_[0, np.cumsum(counts)], dtype=torch.int32, device="cuda")
        Pn = int(sum(counts))
        T0, T1 = cat("Tcw0", 16, np.float32), cat("Tcw1", 16, np.float32)
        xyz, z0, z1 = cat("xyz", 3, np.float32), cat("z0", 3, np.float32), cat("z1", 3, np.float32)
        o0, o1 = cat("info0", 9, np.float64), cat("info1", 9, np.float64)
        pts = torch.zeros((Pn, 3), dtype=torch.float64, device="cuda"); work = torch.zeros_like(pts)
        keep += [T0, T1, xyz, z0, z1, o0, o1, pts, work, pp]
        lo = Eo + 24 * mode
        _capi.check(_capi.lib().se2gpu_feat_edge_device(len(ps), mode, p_(T0), p_(T1), p_(pp), p_(xyz), p_(z0), p_(z1), p_(o0), p_(o1),
                                                        C.addressof(fprm), p_(dm[lo:]), p_(di[lo:]), p_(dstat[lo:]), None, None, None,
                                                        None, p_(pts), p_(work), stream), "se2gpu_feat_edge_device")
    ctx = globalba.Context(0)
    prm = globalba.params(g["Tbc"])
    N = len(g["Tcw"])
    dT = torch.from_numpy(np.ascontiguousarray(g["Tcw"].reshape(N, 16))).cuda()
    d = G._device_call(ctx, g, prm, N, fr, to, dT, dm, di, dstat)
    st, dme, dinf = dstat.cpu().numpy(), dm.cpu().numpy(), di.cpu().numpy()
    edges = list(g["edges"])
    seen = set()
    for mode in (0, 1):
        host = featgraph.UpdateFeatGraph([p for _, _, p in pairs[mode]], fprm, mode=mode)
        for k, ((a, b, _), r) in enumerate(zip(pairs[mode], host)):
            e = Eo + 24 * mode + k
            assert st[e] == r["status"], (mode, k)
            seen.add(r["status"])
            if r["status"] == featgraph.TOO_FEW:
                assert np.isnan(dme[e]).all() and np.isnan(dinf[e]).all()
                continue
            assert r["measure"].tobytes() == dme[e].tobytes() and r["info"].tobytes() == dinf[e].tobytes()
            edges.append((a, b, r["measure"], r["info"]))
    assert featgraph.TOO_FEW in seen and featgraph.OK in seen
    h = ctx.run(g["Tcw"], g["fixed"], edges, prm)
    o = pyglobal.run(dict(g, edges=edges), pyglobal.params(g["Tbc"]))
    check_parity(h, o, "feature_edges_200")
    check_parity(d, o, "feature_edges_200")
    ctx.close()


def test_one_context_across_dense_and_sparse_envelopes(scenes):
    """The grow-only buffers and the gathered H after a dense envelope leave nothing behind: every call on one context
    equals a fresh context's bytes."""
    seq = ["complete_64_free", "loop_fixed_middle", "chain_split_in_four", "stride_nf61", "hub_300", "loop_none_fixed",
           "loop_all_fixed", "complete_64_free"]
    ctx = globalba.Context(0)
    for name in seq:
        s = scenes[name]
        prm = globalba.params(s["Tbc"])
        a = ctx.run(s["Tcw"], s["fixed"], s["edges"], prm)
        b = globalba.GlobalBA(s["Tcw"], s["fixed"], s["edges"], prm)
        for k in ("Tcw", "poses", "stats"):
            assert a[k].tobytes() == b[k].tobytes(), (name, k)
        assert (a["status"], a["iterations"]) == (b["status"], b["iterations"])
    ctx.close()


@pytest.mark.parametrize("M", [1, 255, 256, 257, 100_000])
def test_map_points_over_fixed_and_free_keyframes(scenes, M):
    s = scenes["chain_split_in_four"]
    g = globalba.GlobalBA(s["Tcw"], s["fixed"], s["edges"], globalba.params(s["Tbc"]))
    kf, view = S.map_points(40 + M, s, M)
    kf[0] = 20                                   # a fixed keyframe
    if M > 1:
        kf[-1] = 79                              # the last, free one
    assert M < 255 or (s["fixed"][kf] == 1).any() and (s["fixed"][kf] == 0).any()
    pos = globalba.update_map_points(kf, view, g["Tcw"])
    assert pos.tobytes() == pyglobal.update_points(kf, view, g["Tcw"]).tobytes()
