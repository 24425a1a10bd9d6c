"""ctypes bindings of the feature-graph constraint oracle (oracle/libfeat_edge_oracle.so) — TEST INFRASTRUCTURE ONLY.

A library of its own next to liboracle.so, built with the same flags (no -march, -ffp-contract=off). It restates
GlobalMapper::CreateFeatEdge's two-keyframe BA and the Sparsifier marginalisation (oracle/feat_edge_oracle.cpp). The
product package (se2lam_b200) never imports this module.
"""
from __future__ import annotations

import ctypes as C

import numpy as np

from oracle.pyoracle import BA_STATS_DTYPE, make


class Params(C.Structure):
    """se2gpu_feat_edge_params with the reference's values."""
    _fields_ = [("Tbc", C.c_float * 16), ("xrot_info", C.c_float), ("yrot_info", C.c_float), ("z_info", C.c_float),
                ("huber_delta", C.c_float), ("iterations", C.c_int * 2), ("chi2_cut", C.c_float), ("min_points", C.c_int * 2)]


def params(Tbc=None, xrot=1e6, yrot=1e6, zinfo=1.0, huber_delta=5.99, iterations=(15, 30), chi2_cut=5.0, min_points=(10, 3)):
    p = Params()
    T = np.eye(4, dtype=np.float32) if Tbc is None else np.ascontiguousarray(Tbc, np.float32).reshape(4, 4)
    p.Tbc[:] = [float(v) for v in T.ravel()]
    p.xrot_info, p.yrot_info, p.z_info, p.huber_delta, p.chi2_cut = xrot, yrot, zinfo, huber_delta, chi2_cut
    p.iterations[:] = list(iterations)
    p.min_points[:] = list(min_points)
    return p


_lib = None


def lib():
    global _lib
    if _lib is None:
        L = C.CDLL(make("libfeat_edge_oracle.so"))
        vp, i = C.c_void_p, C.c_int
        L.feat_edge_oracle_run.argtypes = [i, vp, vp, i] + [vp] * 14 + [i, vp]
        L.feat_edge_oracle_from_Tcw.argtypes = [vp, vp]
        L.feat_edge_oracle_oplus.argtypes = [vp, vp, vp]
        L.feat_edge_oracle_xyz_edge.argtypes = [vp] * 6
        L.feat_edge_oracle_prior.argtypes = [vp] * 7
        L.feat_edge_oracle_clamp.argtypes = [vp]
        _lib = L
    return _lib


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def _d(a):
    return np.ascontiguousarray(a, np.float64)


def run(mode, Tcw0, Tcw1, xyz, z0, z1, info0, info1, prm=None, reverse=False, cofactor=False):
    """One keyframe pair. Returns dict(status, iterations, measure [4,4] f32, info [6,6] f32, outlier [P] u8, poses [2,7],
    points [P,3], stats, trace [iterations,2,12], Hm [12,12]); measure / info are None when the status is 1 (too few)."""
    prm = prm or params()
    f32 = lambda a, s: np.ascontiguousarray(a, np.float32).reshape(s)
    T0, T1 = f32(Tcw0, 16), f32(Tcw1, 16)
    xyz = f32(xyz, (-1, 3)); P = len(xyz)
    z0, z1 = f32(z0, (-1, 3)), f32(z1, (-1, 3))
    o0, o1 = _d(info0).reshape(-1, 9), _d(info1).reshape(-1, 9)
    assert len(z0) == P and len(z1) == P and len(o0) == P and len(o1) == P
    nit = max(prm.iterations[mode], 1)
    measure = np.zeros(16, np.float32); info = np.zeros(36, np.float32)
    outlier = np.zeros(max(P, 1), np.uint8); poses = np.zeros(14); points = np.zeros(max(3 * P, 1))
    stats = np.zeros(nit, BA_STATS_DTYPE); trace = np.zeros(nit * 24); Hm = np.zeros(144)
    status = C.c_int(0)
    pad = lambda a, w: a if P else np.zeros((1, w), a.dtype)
    n = lib().feat_edge_oracle_run(int(mode), _p(T0), _p(T1), P, _p(pad(xyz, 3)), _p(pad(z0, 3)), _p(pad(z1, 3)), _p(pad(o0, 9)),
                                   _p(pad(o1, 9)), C.addressof(prm), _p(measure), _p(info), _p(outlier), _p(poses), _p(points),
                                   _p(stats), _p(trace), _p(Hm), int(bool(reverse)) | 2 * int(bool(cofactor)), C.addressof(status))
    too_few = status.value == 1
    return dict(status=status.value, iterations=n, measure=None if too_few else measure.reshape(4, 4),
                info=None if too_few else info.reshape(6, 6), outlier=outlier[:P].copy(), poses=poses.reshape(2, 7),
                points=points[:3 * P].reshape(P, 3).copy(), stats=stats[:n].copy(), trace=trace.reshape(nit, 2, 12)[:n].copy(),
                Hm=Hm.reshape(12, 12))


def from_Tcw(Tcw):
    out = np.zeros(12)
    lib().feat_edge_oracle_from_Tcw(_p(np.ascontiguousarray(Tcw, np.float32).reshape(16)), _p(out))
    return out


def oplus(X12, d6):
    out = np.zeros(12)
    lib().feat_edge_oracle_oplus(_p(_d(X12)), _p(_d(d6)), _p(out))
    return out


def xyz_edge(X12, p, z):
    """EdgeSE3PointXYZ: error [3], pose Jacobian [3,6], point Jacobian [3,3]."""
    e = np.zeros(3); Jp = np.zeros(18); Jl = np.zeros(9)
    lib().feat_edge_oracle_xyz_edge(_p(_d(X12)), _p(_d(p)), _p(_d(z)), _p(e), _p(Jp), _p(Jl))
    return e, Jp.reshape(3, 6), Jl.reshape(3, 3)


def prior(X0_12, X12, prm=None):
    """addVertexSE3PlaneMotion built at X0, EdgeSE3Prior evaluated at X: (measurement [12], info [6,6], error [6], J [6,6])."""
    prm = prm or params()
    meas = np.zeros(12); info = np.zeros(36); e = np.zeros(6); J = np.zeros(36)
    lib().feat_edge_oracle_prior(_p(_d(X0_12)), C.addressof(prm), _p(_d(X12)), _p(meas), _p(info), _p(e), _p(J))
    return meas, info.reshape(6, 6), e, J.reshape(6, 6)


def clamp(I):
    out = _d(I).reshape(36).copy()
    lib().feat_edge_oracle_clamp(_p(out))
    return out.reshape(6, 6)
