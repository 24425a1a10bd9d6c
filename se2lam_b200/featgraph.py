"""Feature-graph constraints on the GPU: GlobalMapper::CreateFeatEdge (both overloads) and Map::UpdateFeatGraph's loop over
keyframe pairs, through se2gpu_feat_edge. numpy in, numpy out; there is no CPU fallback."""
from __future__ import annotations

import ctypes as C

import numpy as np

from ._capi import BA_STATS_DTYPE, FeatEdgeParams, check, lib, ptr

OK, TOO_FEW, NOT_PD = 0, 1, 2


def params(Tbc, xrot_info=1e6, yrot_info=1e6, z_info=1.0, huber_delta=5.99, iterations=(15, 30), chi2_cut=5.0, min_points=(10, 3)):
    """se2gpu_feat_edge_params with the reference's values; Tbc = Config::bTc [4,4]."""
    p = FeatEdgeParams()
    p.Tbc[:] = [float(v) for v in np.asarray(Tbc, np.float32).reshape(16)]
    p.xrot_info, p.yrot_info, p.z_info, p.huber_delta, p.chi2_cut = xrot_info, yrot_info, z_info, huber_delta, chi2_cut
    p.iterations[:] = list(iterations)
    p.min_points[:] = list(min_points)
    return p


def _cat(pairs, key, dtype, width):
    parts = [np.ascontiguousarray(p[key], dtype).reshape(-1, width) for p in pairs]
    return np.ascontiguousarray(np.concatenate(parts)) if parts else np.zeros((0, width), dtype)


def UpdateFeatGraph(pairs, prm, mode=0, device=0, trace=False):
    """Every pair of one call of Map::UpdateFeatGraph (mode 0) or a batch of verified loop matches (mode 1) in one launch.
    pairs: a list of dicts with Tcw0, Tcw1 [4,4], xyz, z0, z1 [P,3] and info0, info1 [P,3,3] (mViewMPsInfo, as
    se2lam_b200.geometry.xyz_info returns them). Returns a list of dicts, one per pair: status, iterations, measure [4,4]
    and info [6,6] float32 (None when the status is TOO_FEW), outlier [P] uint8, poses [2,7], points [P,3], stats
    (and trace [iterations,2,12] when asked for)."""
    B = len(pairs)
    T0 = _cat(pairs, "Tcw0", np.float32, 16); T1 = _cat(pairs, "Tcw1", np.float32, 16)
    xyz = _cat(pairs, "xyz", np.float32, 3); z0 = _cat(pairs, "z0", np.float32, 3); z1 = _cat(pairs, "z1", np.float32, 3)
    o0 = _cat(pairs, "info0", np.float64, 9); o1 = _cat(pairs, "info1", np.float64, 9)
    counts = [len(np.asarray(p["xyz"]).reshape(-1, 3)) for p in pairs]
    pp = np.zeros(B + 1, np.int32); pp[1:] = np.cumsum(counts)
    P = int(pp[-1])
    assert len(z0) == P and len(z1) == P and len(o0) == P and len(o1) == P
    nit = max(int(prm.iterations[mode]), 1)
    measure = np.zeros((B, 16), np.float32); info = np.zeros((B, 36), np.float32)
    status = np.zeros(B, np.int32); iters = np.zeros(B, np.int32)
    stats = np.zeros((B, nit), BA_STATS_DTYPE); outlier = np.zeros(max(P, 1), np.uint8)
    poses = np.zeros((B, 14)); points = np.zeros((max(P, 1), 3))
    args = [B, int(mode), ptr(T0), ptr(T1), ptr(pp), ptr(xyz), ptr(z0), ptr(z1), ptr(o0), ptr(o1), C.addressof(prm), ptr(measure),
            ptr(info), ptr(status), ptr(iters), ptr(stats) if prm.iterations[mode] else None, ptr(outlier), ptr(poses), ptr(points)]
    if trace:
        tr = np.zeros((B, nit, 2, 12))
        check(lib().se2gpu_feat_edge_debug_trace(*args, ptr(tr) if prm.iterations[mode] else None, device), "se2gpu_feat_edge_debug_trace")
    else:
        check(lib().se2gpu_feat_edge(*args, device), "se2gpu_feat_edge")
    out = []
    for b in range(B):
        few = status[b] == TOO_FEW
        n = int(iters[b])
        r = dict(status=int(status[b]), iterations=n, measure=None if few else measure[b].reshape(4, 4).copy(),
                 info=None if few else info[b].reshape(6, 6).copy(), outlier=outlier[pp[b]:pp[b + 1]].copy(),
                 poses=poses[b].reshape(2, 7).copy(), points=points[pp[b]:pp[b + 1]].copy(), stats=stats[b, :n].copy())
        if trace:
            r["trace"] = tr[b, :n].copy()
        out.append(r)
    return out


def CreateFeatEdge(Tcw0, Tcw1, xyz, z0, z1, info0, info1, prm, matched=False, device=0, trace=False):
    """One keyframe pair: CreateFeatEdge(from, to, cnstr) or, with matched=True, CreateFeatEdge(from, to, mapMatch, cnstr)
    over the matches whose two map points exist. See UpdateFeatGraph for the arrays and the result."""
    pair = dict(Tcw0=Tcw0, Tcw1=Tcw1, xyz=xyz, z0=z0, z1=z1, info0=info0, info1=info1)
    return UpdateFeatGraph([pair], prm, mode=1 if matched else 0, device=device, trace=trace)[0]
