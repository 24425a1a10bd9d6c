"""ctypes bindings of the outlier-rejection oracle (oracle/libfundam_oracle.so) — TEST INFRASTRUCTURE ONLY.

A library of its own next to liboracle.so, built with the same flags (oracle/Makefile: no -march, -ffp-contract=off).
It restates Track::removeOutliers and cv::findFundamentalMat's FM_RANSAC / LMedS path (oracle/fundam_oracle.cpp).
The product package (se2lam_b200) never imports this module.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, "fundam_oracle.cpp")
LIB_PATH = os.path.join(HERE, "libfundam_oracle.so")
CXXFLAGS = ["-O2", "-std=c++17", "-fPIC", "-ffp-contract=off", "-fno-fast-math", "-fvisibility=hidden", "-Wall",
            "-Wno-unused-function"]


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
        vp, i = C.c_void_p, C.c_int
        L.fundam_oracle_find.argtypes = [vp, vp, i, vp, vp, vp, vp]
        L.fundam_oracle_remove_outliers.argtypes = [vp, i, vp, i, vp, vp, vp]
        L.fundam_oracle_niters_range.argtypes = [i, i, i, vp]
        L.fundam_oracle_niters.argtypes = [C.c_double, i]
        _lib = L
    return _lib


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def find_fundamental_mat(pt1, pt2):
    """cv::findFundamentalMat(pt1, pt2, mask) with the defaults. Returns (mask [n] uint8 or None when OpenCV never creates
    it, F [3k,3] float64 with k = 0..3 matrices, hypotheses run)."""
    p1 = np.ascontiguousarray(pt1, np.float32).reshape(-1, 2)
    p2 = np.ascontiguousarray(pt2, np.float32).reshape(-1, 2)
    n = len(p1)
    mask = np.zeros(max(n, 1), np.uint8)
    F = np.zeros(27)
    created = C.c_int(0); iters = C.c_int(0)
    k = lib().fundam_oracle_find(_p(p1), _p(p2), n, _p(mask), _p(F), C.byref(created), C.byref(iters))
    return (mask[:n].copy() if created.value else None), F[:9 * k].reshape(-1, 3).copy(), iters.value


def remove_outliers(kp1, kp2, matches12):
    """Track::removeOutliers(kp1, kp2, matches12) on KP_DTYPE keypoints. Returns (nInlier, matches12 after the call,
    F [3,3] of the returned model or zeros, hypotheses run); the inputs are not modified."""
    kp1 = np.ascontiguousarray(kp1); kp2 = np.ascontiguousarray(kp2)
    assert kp1.dtype.itemsize == 28 and kp2.dtype.itemsize == 28
    m = np.ascontiguousarray(matches12, np.int32).copy()
    assert len(m) == len(kp1) and (m < len(kp2)).all()
    F = np.zeros(9); iters = C.c_int(0)
    k2 = kp2 if len(kp2) else np.zeros(1, kp1.dtype)
    n = lib().fundam_oracle_remove_outliers(_p(kp1), len(kp1), _p(k2), 7, _p(m), _p(F), C.byref(iters))
    return n, m, F.reshape(3, 3), iters.value


def niters_range(n_lo, n_hi, max_iters=1000):
    """RANSACUpdateNumIters(0.99, (n - good) / n, 7, max_iters) through libm, for n in [n_lo, n_hi], good in [0, n]:
    one flat int32 array, row n after row n - 1."""
    out = np.zeros(sum(n + 1 for n in range(n_lo, n_hi + 1)), np.int32)
    lib().fundam_oracle_niters_range(n_lo, n_hi, max_iters, _p(out))
    return out


def niters(ep, max_iters=1000):
    return lib().fundam_oracle_niters(float(ep), int(max_iters))
