"""ctypes bindings of the pose-only BA oracle (oracle/libpose_ba_oracle.so) — TEST INFRASTRUCTURE ONLY.

A library of its own next to liboracle.so, built with the same flags (no -march, -ffp-contract=off). It restates
Localizer::DoLocalBA's g2o graph (oracle/pose_ba_oracle.cpp). The product package (se2lam_b200) never imports this module.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

from oracle.pyoracle import BA_STATS_DTYPE

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, "pose_ba_oracle.cpp")
LIB_PATH = os.path.join(HERE, "libpose_ba_oracle.so")
CXXFLAGS = ["-O2", "-std=c++17", "-fPIC", "-ffp-contract=off", "-fno-fast-math", "-fvisibility=default", "-Wall",
            "-Wno-unused-function", "-Wno-maybe-uninitialized"]


def build(force: bool = False) -> str:
    if force or not os.path.exists(LIB_PATH) or os.path.getmtime(SRC) > os.path.getmtime(LIB_PATH):
        tmp = LIB_PATH + f".{os.getpid()}.tmp"
        subprocess.run(["g++", *CXXFLAGS, "-shared", "-o", tmp, SRC], check=True)
        os.replace(tmp, LIB_PATH)
    return LIB_PATH


_lib = None


def lib():
    global _lib
    if _lib is None:
        build()
        L = C.CDLL(LIB_PATH)
        vp, i, f, d = C.c_void_p, C.c_int, C.c_float, C.c_double
        L.pose_ba_oracle_run.argtypes = [vp, i, vp, vp, vp, f, f, f, vp, f, f, f, f, i, vp, vp, vp, vp]
        L.pose_ba_oracle_from_f32.argtypes = [vp, vp]
        L.pose_ba_oracle_exp.argtypes = [vp, vp]
        L.pose_ba_oracle_log.argtypes = [vp, vp]
        L.pose_ba_oracle_mul.argtypes = [vp, vp, vp]
        L.pose_ba_oracle_prior.argtypes = [vp, vp, f, f, f, vp, vp]
        L.pose_ba_oracle_edge.argtypes = [vp, vp, vp, d, d, d, vp, vp]
        _lib = L
    return _lib


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def _f(a, shape):
    return np.ascontiguousarray(a, np.float32).reshape(shape)


def run(Tcw, xyz, uv, info, fx, cx, cy, Tbc, huber_delta, xrot=1e6, yrot=1e6, zinfo=1.0, iterations=30):
    """One DoLocalBA problem. Returns dict(Tcw [4,4] float32, pose [7] (qx,qy,qz,qw,tx,ty,tz), iterations, status,
    stats [iterations done] BA_STATS_DTYPE, trace [iterations done, 7])."""
    T = _f(Tcw, 16).copy()
    xyz = _f(xyz, (-1, 3)); E = len(xyz)
    uv = _f(uv, (-1, 2)); w = _f(info, -1)
    assert len(uv) == E and len(w) == E
    xyz_ = xyz if E else np.zeros((1, 3), np.float32)
    uv_ = uv if E else np.zeros((1, 2), np.float32)
    w_ = w if E else np.zeros(1, np.float32)
    stats = np.zeros(max(iterations, 1), BA_STATS_DTYPE)
    trace = np.zeros((max(iterations, 1), 7))
    pose = np.zeros(7); status = C.c_int(0)
    n = lib().pose_ba_oracle_run(_p(T), E, _p(xyz_), _p(uv_), _p(w_), float(fx), float(cx), float(cy), _p(_f(Tbc, 16)),
                                 float(huber_delta), float(xrot), float(yrot), float(zinfo), int(iterations), _p(stats),
                                 _p(trace), _p(pose), C.byref(status))
    return dict(Tcw=T.reshape(4, 4), pose=pose, iterations=n, status=status.value, stats=stats[:n].copy(), trace=trace[:n].copy())


def from_f32(T):
    out = np.zeros(7)
    lib().pose_ba_oracle_from_f32(_p(_f(T, 16)), _p(out))
    return out


def se3_exp(u):
    out = np.zeros(7)
    lib().pose_ba_oracle_exp(_p(np.ascontiguousarray(u, np.float64)), _p(out))
    return out


def se3_log(pose7):
    out = np.zeros(6)
    lib().pose_ba_oracle_log(_p(np.ascontiguousarray(pose7, np.float64)), _p(out))
    return out


def se3_mul(a, b):
    out = np.zeros(7)
    lib().pose_ba_oracle_mul(_p(np.ascontiguousarray(a, np.float64)), _p(np.ascontiguousarray(b, np.float64)), _p(out))
    return out


def prior(pose7, Tbc, xrot=1e6, yrot=1e6, zinfo=1.0):
    """addPlaneMotionSE3Expmap: (measurement pose7, information [6,6])."""
    meas = np.zeros(7); info = np.zeros(36)
    lib().pose_ba_oracle_prior(_p(np.ascontiguousarray(pose7, np.float64)), _p(_f(Tbc, 16)), float(xrot), float(yrot), float(zinfo),
                               _p(meas), _p(info))
    return meas, info.reshape(6, 6)


def edge(pose7, xyz, uv, fx, cx, cy):
    """EdgeProjectXYZ2UV error [2] and pose Jacobian [2,6] (omega columns first)."""
    err = np.zeros(2); J = np.zeros(12)
    lib().pose_ba_oracle_edge(_p(np.ascontiguousarray(pose7, np.float64)), _p(np.ascontiguousarray(xyz, np.float64)),
                              _p(np.ascontiguousarray(uv, np.float64)), float(fx), float(cx), float(cy), _p(err), _p(J))
    return err, J.reshape(2, 6)
