"""ctypes bindings of the global pose-graph oracle (oracle/libglobal_ba_oracle.so) — TEST INFRASTRUCTURE ONLY.

A library of its own, built by oracle/Makefile with the flags of the other oracles (no -march, -ffp-contract=off). It
restates GlobalMapper::GlobalBA (oracle/global_ba_oracle.cpp) on the SE(3) pieces the feature-graph oracle also runs
(oracle/se3_oracle.h). The product package (se2lam_b200) never imports this module.
"""
from __future__ import annotations

import ctypes as C

import numpy as np

from oracle.pyoracle import BA_STATS_DTYPE, make


class Params(C.Structure):
    """se2gpu_global_ba_params."""
    _fields_ = [("Tbc", C.c_float * 16), ("xrot_info", C.c_float), ("yrot_info", C.c_float), ("z_info", C.c_float),
                ("iterations", C.c_int)]


def params(Tbc=None, xrot=1e6, yrot=1e6, zinfo=1.0, iterations=15):
    p = Params()
    T = np.eye(4, dtype=np.float32) if Tbc is None else np.ascontiguousarray(Tbc, np.float32).reshape(4, 4)
    p.Tbc[:] = [float(v) for v in T.ravel()]
    p.xrot_info, p.yrot_info, p.z_info, p.iterations = xrot, yrot, zinfo, iterations
    return p


_lib = None


def lib():
    global _lib
    if _lib is None:
        L = C.CDLL(make("libglobal_ba_oracle.so"))
        vp, i = C.c_void_p, C.c_int
        L.global_ba_oracle_run.argtypes = [i, vp, vp, i] + [vp] * 9 + [i, vp]
        L.global_ba_oracle_edge.argtypes = [vp] * 7
        L.global_ba_oracle_edge.restype = C.c_double
        L.global_ba_oracle_from_Tcw.argtypes = [vp, vp]
        L.global_ba_oracle_update_points.argtypes = [i, vp, vp, vp, vp]
        _lib = L
    return _lib


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def _arrays(g):
    N = len(g["Tcw"])
    E = len(g["edges"])
    T = np.ascontiguousarray(g["Tcw"], np.float32).reshape(N, 16)
    fixed = np.ascontiguousarray(g["fixed"], np.uint8).reshape(N)
    fr = np.array([e[0] for e in g["edges"]] or [0], np.int32)
    to = np.array([e[1] for e in g["edges"]] or [0], np.int32)
    me = np.ascontiguousarray([np.asarray(e[2], np.float32).reshape(16) for e in g["edges"]] or [np.zeros(16)], np.float32)
    inf = np.ascontiguousarray([np.asarray(e[3], np.float32).reshape(36) for e in g["edges"]] or [np.zeros(36)], np.float32)
    return N, E, T, fixed, fr, to, me, inf


def elimination_order(N, fixed, fr, to, reverse_order=False):
    """scipy's reverse Cuthill-McKee order of the free vertices' block graph (position -> vertex); reversed with
    reverse_order (the Cuthill-McKee order: the same bandwidth, another factorisation sequence)."""
    from scipy.sparse import coo_matrix
    from scipy.sparse.csgraph import reverse_cuthill_mckee
    free = np.flatnonzero(np.asarray(fixed) == 0)
    idx = -np.ones(N, np.int64)
    idx[free] = np.arange(len(free))
    a, b = idx[fr], idx[to]
    keep = (a >= 0) & (b >= 0)
    n = len(free)
    A = coo_matrix((np.ones(2 * int(keep.sum())), (np.r_[a[keep], b[keep]], np.r_[b[keep], a[keep]])), shape=(n, n)).tocsr()
    perm = reverse_cuthill_mckee(A, symmetric_mode=True) if n else np.zeros(0, np.int64)
    if reverse_order:
        perm = perm[::-1]
    return np.ascontiguousarray(free[perm], np.int32)


def run(g, prm, reverse=False, reverse_order=False):
    """g: dict(Tcw [N,4,4], fixed [N], edges [(from, to, measure [4,4], info [6,6])]). reverse sums the edges in
    descending order, reverse_order factorises in the reversed elimination order (the oracle's two spreads). Returns
    dict(status, iterations, Tcw [N,4,4] float32, poses [N,7], stats)."""
    N, E, T, fixed, fr, to, me, inf = _arrays(g)
    order = elimination_order(N, fixed, fr[:E], to[:E], reverse_order)
    order_buf = order if len(order) else np.zeros(1, np.int32)
    out = np.zeros((N, 16), np.float32)
    poses = np.zeros((N, 7))
    stats = np.zeros(max(prm.iterations, 1), BA_STATS_DTYPE)
    status = C.c_int(0)
    n = lib().global_ba_oracle_run(N, _p(T), _p(fixed), E, _p(fr), _p(to), _p(me), _p(inf), C.addressof(prm), _p(order_buf), _p(out), _p(poses),
                                   _p(stats), int(bool(reverse)), C.addressof(status))
    return dict(status=status.value, iterations=n, Tcw=out.reshape(N, 4, 4), poses=poses, stats=stats[:n].copy())


def edge(Xi12, Xj12, measure, info):
    """EdgeSE3: (chi2, e [6], Ji [6,6], Jj [6,6])."""
    d = lambda a: np.ascontiguousarray(a, np.float64)
    e = np.zeros(6); Ji = np.zeros(36); Jj = np.zeros(36)
    chi = lib().global_ba_oracle_edge(_p(d(Xi12)), _p(d(Xj12)), _p(np.ascontiguousarray(measure, np.float32).reshape(16)),
                                      _p(d(info).reshape(36)), _p(e), _p(Ji), _p(Jj))
    return chi, e, Ji.reshape(6, 6), Jj.reshape(6, 6)


def from_Tcw(Tcw):
    out = np.zeros(12)
    lib().global_ba_oracle_from_Tcw(_p(np.ascontiguousarray(Tcw, np.float32).reshape(16)), _p(out))
    return out


def update_points(kf, view, Tcw):
    kf = np.ascontiguousarray(kf, np.int32)
    view = np.ascontiguousarray(view, np.float32).reshape(-1, 3)
    T = np.ascontiguousarray(Tcw, np.float32).reshape(-1, 16)
    pos = np.zeros((max(len(kf), 1), 3), np.float32)
    if len(kf):
        lib().global_ba_oracle_update_points(len(kf), _p(kf), _p(view), _p(T), _p(pos))
    return pos[:len(kf)]
