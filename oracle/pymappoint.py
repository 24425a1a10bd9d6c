"""ctypes bindings of the map-point update oracle (oracle/libmappoint_oracle.so) — TEST INFRASTRUCTURE ONLY.

Same tables as se2lam_b200.mappoint (dicts of numpy arrays, updated in place), the same structs, and the oracle's restatement
of MapPoint::addObservation / eraseObservation / updateMeasureInKFs in the reference's float types.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

from se2lam_b200 import mappoint

HERE = os.path.dirname(os.path.abspath(__file__))
_lib = None


def make() -> str:
    """Bring oracle/libmappoint_oracle.so up to date with oracle/mappoint.mk (oracle/Makefile's compiler and flags, whatever
    CXX / CXXFLAGS the environment holds) and return its path."""
    env = {k: v for k, v in os.environ.items() if k not in ("CXX", "CXXFLAGS")}
    subprocess.run(["make", "-C", HERE, "-s", "-f", "mappoint.mk", "CXX=g++"], check=True, env=env)
    return os.path.join(HERE, "libmappoint_oracle.so")


def lib():
    global _lib
    if _lib is None:
        L = C.CDLL(make())
        vp, i, d = C.c_void_p, C.c_int, C.c_double
        L.mp_oracle_updates.argtypes = [i] + [vp] * 6
        L.mp_oracle_updates.restype = None
        L.mp_oracle_update_measure.argtypes = [vp, vp, i, vp]
        L.mp_oracle_update_measure.restype = None
        for name in ("mp_oracle_gemm3_a_bt", "mp_oracle_rt_m_r", "mp_oracle_r_m_rt"):
            getattr(L, name).argtypes = [vp, vp, vp]
            getattr(L, name).restype = None
        L.mp_oracle_norm3.argtypes = [vp]
        L.mp_oracle_norm3.restype = d
        L.mp_oracle_mul_pd.argtypes = [vp, d, vp]
        L.mp_oracle_mul_pd.restype = None
        _lib = L
    return _lib


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def _updates(add, kf, mp, upd_ptr, upd_pos, params):
    mappoint._host(kf, mappoint.KF_FIELDS)
    mappoint._host(mp, mappoint.MP_FIELDS)
    upd_ptr = np.ascontiguousarray(upd_ptr, np.int32)
    upd_pos = np.ascontiguousarray(upd_pos, np.int32)
    k, p, prm = mappoint.keyframes(kf), mappoint.points(mp), mappoint.params(**params)
    ab = np.zeros(p.n_mp, np.uint8)
    lib().mp_oracle_updates(int(add), C.byref(k), C.byref(p), _p(upd_ptr), _p(upd_pos), C.byref(prm), _p(ab))
    return ab.astype(bool)


def add_observations(kf, mp, upd_ptr, upd_pos, params):
    """MapPoint::addObservation for every point's updates; returns the abandoned flags"""
    return _updates(True, kf, mp, upd_ptr, upd_pos, params)


def erase_observations(kf, mp, upd_ptr, upd_pos, params):
    """MapPoint::eraseObservation for every point's updates; returns the points set null"""
    return _updates(False, kf, mp, upd_ptr, upd_pos, params)


def update_measure(kf, mp, points):
    """MapPoint::updateMeasureInKFs of the listed points"""
    points = np.ascontiguousarray(points, np.int32)
    lib().mp_oracle_update_measure(C.byref(mappoint.keyframes(kf)), C.byref(mappoint.points(mp)), len(points), _p(points))


def _f3(a):
    return np.ascontiguousarray(a, np.float32)


def rt_m_r(R, M):
    out = np.zeros((3, 3), np.float32); lib().mp_oracle_rt_m_r(_p(_f3(R)), _p(_f3(M)), _p(out)); return out


def r_m_rt(R, M):
    out = np.zeros((3, 3), np.float32); lib().mp_oracle_r_m_rt(_p(_f3(R)), _p(_f3(M)), _p(out)); return out


def gemm3_a_bt(A, B):
    out = np.zeros((3, 3), np.float32); lib().mp_oracle_gemm3_a_bt(_p(_f3(A)), _p(_f3(B)), _p(out)); return out


def norm3(p):
    return lib().mp_oracle_norm3(_p(_f3(p)))


def mul_pd(p, s):
    out = np.zeros(3, np.float32); lib().mp_oracle_mul_pd(_p(_f3(p)), float(s), _p(out)); return out
