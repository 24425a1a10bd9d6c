"""ctypes binding of the SE(3)-XYZ window BA oracle (oracle/libse3_ba_oracle.so) — TEST INFRASTRUCTURE ONLY.

A library of its own, built by oracle/Makefile with the flags of the other oracles (no -march, -ffp-contract=off). It
restates the window of Map::loadLocalGraph / loadLocalGraphOnlyBa and removeOutlierChi2's cut (oracle/se3_ba_oracle.cpp) on
the SE3Quat pieces the pose-only BA oracle also runs (oracle/se3_oracle.h). The product package (se2lam_b200) never imports
this module.
"""
from __future__ import annotations

import ctypes as C

import numpy as np

from oracle.pyoracle import BA_STATS_DTYPE, make


_lib = None


def lib():
    global _lib
    if _lib is None:
        L = C.CDLL(make("libse3_ba_oracle.so"))
        vp, i = C.c_void_p, C.c_int
        L.se3_ba_oracle_run.restype = i
        L.se3_ba_oracle_run.argtypes = [i, vp, vp, vp, i, vp, vp, vp, vp, i, vp, i, vp, vp, vp, vp, vp, i, i] + [vp] * 7
        _lib = L
    return _lib


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def run(w, prm, rev_sums=False, rev_order=False, trace=False):
    """w: se2lam_b200.se3ba.Window, prm: its se2gpu_se3_ba_params. rev_sums takes every sum over edges in descending order,
    rev_order eliminates the free keyframes in reversed order. Returns the dict se3ba.Context.run returns (poses, points,
    chi2, outlier, status, iterations, stats, and trace when asked)."""
    N, O, L, E = w.sizes
    it = max(prm.iterations, 1)
    stats = np.zeros(it, BA_STATS_DTYPE)
    poses = np.zeros((N, 7)); points = np.zeros((max(L, 1), 3))
    chi2 = np.zeros(max(E, 1)); outl = np.zeros(max(E, 1), np.uint8); status = np.zeros(1, np.int32)
    tr = np.zeros((it, 7 * N + 3 * L)) if trace else None
    n = lib().se3_ba_oracle_run(N, _p(w.Tcw), _p(w.fixed), _p(w.prior), O, _p(w.odo_from), _p(w.odo_to), _p(w.odo_measure),
                                _p(w.odo_info), L, _p(w.xyz), E, _p(w.edge_point), _p(w.edge_kf), _p(w.uv), _p(w.inv_sigma2),
                                C.addressof(prm), int(rev_sums), int(rev_order), _p(stats), _p(poses), _p(points), _p(chi2),
                                _p(outl), _p(status), _p(tr) if trace else None)
    out = dict(status=int(status[0]), iterations=n, chi2=chi2[:E], outlier=outl[:E].astype(bool), poses=poses,
               points=points[:L], stats=stats[:n].copy())
    if trace:
        out["trace"] = tr[:n]
    return out
