"""ctypes bindings of the two-view geometry oracle (oracle/libgeom_oracle.so) — TEST INFRASTRUCTURE ONLY.

A library of its own next to liboracle.so, built with the same flags (oracle/Makefile: no -march, -ffp-contract=off).
The product package (se2lam_b200) never imports this module.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, "geom_oracle.cpp")
LIB_PATH = os.path.join(HERE, "libgeom_oracle.so")
CXXFLAGS = ["-O2", "-std=c++17", "-fPIC", "-ffp-contract=off", "-fno-fast-math", "-Wall", "-Wno-unused-function"]


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
        L.geom_oracle_svd4.argtypes = [vp, vp, vp]
        L.geom_oracle_svd4_libm_hypot.argtypes = [vp, vp, vp]
        L.geom_oracle_build_a.argtypes = [vp] * 5
        L.geom_oracle_triangulate.argtypes = [i] + [vp] * 6
        L.geom_oracle_inv.argtypes = [vp, vp]
        L.geom_oracle_gemm3_fast.argtypes = [vp, vp, i, d, vp]
        L.geom_oracle_gemm3_at_b.argtypes = [vp, vp, vp]
        L.geom_oracle_check_parallax.argtypes = [vp, vp, vp, i]
        L.geom_oracle_rodrigues.argtypes = [vp, vp]
        L.geom_oracle_xyz_info.argtypes = [i, vp, vp, vp, vp, f, vp, vp]
        L.geom_oracle_track_triangulate.argtypes = [vp, i, vp, vp, vp, vp, vp, vp, f, f, i, vp, vp, vp]
        L.geom_oracle_accept_new_observe.argtypes = [vp, vp, i, i, f, f]
        L.geom_oracle_projection_observations.argtypes = [i, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, f, f, f, vp, vp, vp]
        _lib = L
    return _lib


def _c(a, dt):
    return np.ascontiguousarray(a, dt)


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def svd4(A, libm_hypot=False):
    """cv::SVD::compute(A, w, u, vt, MODIFY_A|FULL_UV) on 4x4 float32 matrices [..., 4, 4]: returns (w [..., 4], vt [..., 4, 4]).
    libm_hypot=True swaps lapack.cpp's hypot for libm's (only for checking that a sample tells the two apart)."""
    A = _c(A, np.float32)
    flat = A.reshape(-1, 16)
    w = np.zeros((len(flat), 4), np.float32); vt = np.zeros((len(flat), 16), np.float32)
    fn = lib().geom_oracle_svd4_libm_hypot if libm_hypot else lib().geom_oracle_svd4
    for k in range(len(flat)):
        fn(_p(flat[k]), _p(w[k]), _p(vt[k]))
    return w.reshape(A.shape[:-2] + (4,)), vt.reshape(A.shape)


def build_a(pt1, pt2, P1, P2):
    out = np.zeros(16, np.float32)
    a = [_c(pt1, np.float32), _c(pt2, np.float32), _c(P1, np.float32), _c(P2, np.float32)]
    lib().geom_oracle_build_a(*[_p(x) for x in a], _p(out))
    return out.reshape(4, 4)


def triangulate(pt1, pt2, P, idx1, idx2):
    """cvu::triangulate for n pairs: pt1/pt2 [n,2] float32, P [n_proj,3,4] float32, idx1/idx2 [n] int32 -> xyz [n,3]."""
    pt1 = _c(pt1, np.float32); pt2 = _c(pt2, np.float32); P = _c(P, np.float32)
    idx1 = _c(idx1, np.int32); idx2 = _c(idx2, np.int32)
    xyz = np.zeros((len(idx1), 3), np.float32)
    lib().geom_oracle_triangulate(len(idx1), _p(pt1), _p(pt2), _p(P), _p(idx1), _p(idx2), _p(xyz))
    return xyz


def inv(T):
    T = _c(T, np.float32); out = np.zeros((4, 4), np.float32)
    lib().geom_oracle_inv(_p(T), _p(out))
    return out


def gemm3(A, B, alpha=1.0):
    A = _c(A, np.float32); B = _c(B, np.float32)
    out = np.zeros((3, B.shape[1]), np.float32)
    lib().geom_oracle_gemm3_fast(_p(A), _p(B), B.shape[1], alpha, _p(out))
    return out


def gemm3_at_b(A, B):
    A = _c(A, np.float32); B = _c(B, np.float32); out = np.zeros((3, 3), np.float32)
    lib().geom_oracle_gemm3_at_b(_p(A), _p(B), _p(out))
    return out


def check_parallax(o1, o2, pt3, min_degree=2):
    return bool(lib().geom_oracle_check_parallax(_p(_c(o1, np.float32)), _p(_c(o2, np.float32)), _p(_c(pt3, np.float32)), min_degree))


def rodrigues(rv):
    rv = _c(rv, np.float32); out = np.zeros((3, 3), np.float32)
    lib().geom_oracle_rodrigues(_p(rv), _p(out))
    return out


def xyz_info(xyz1, pose1, pose2, Tcw, fx):
    """Track::calcSE3toXYZInfo for n points: Tcw [n_pose,4,4]; returns (info1, info2) [n,3,3] float64."""
    xyz1 = _c(xyz1, np.float32); pose1 = _c(pose1, np.int32); pose2 = _c(pose2, np.int32); Tcw = _c(Tcw, np.float32)
    n = len(pose1)
    i1 = np.zeros((n, 3, 3)); i2 = np.zeros((n, 3, 3))
    lib().geom_oracle_xyz_info(n, _p(xyz1), _p(pose1), _p(pose2), _p(Tcw), float(fx), _p(i1), _p(i2))
    return i1, i2


def track_triangulate(kp_kf, kp_frame, matches12, kf_observed, kf_view_mp, Tcr, K, lower, upper, min_prl_deg, local_mps):
    """Track::doTriangulate. Returns (matches12, local_mps, good_prl, (nTrackedOld, nGoodPrl)); inputs are not modified."""
    kp_kf = np.ascontiguousarray(kp_kf); kp_frame = np.ascontiguousarray(kp_frame)
    m = _c(matches12, np.int32).copy(); obs = _c(kf_observed, np.uint8); vm = _c(kf_view_mp, np.float32)
    Tcr = _c(Tcr, np.float32); K = _c(K, np.float32); lm = _c(local_mps, np.float32).copy()
    n = len(kp_kf)
    good = np.zeros(n, np.uint8); counts = np.zeros(2, np.int32)
    lib().geom_oracle_track_triangulate(_p(kp_kf), n, _p(kp_frame), _p(m), _p(obs), _p(vm), _p(Tcr), _p(K), float(lower),
                                        float(upper), int(min_prl_deg), _p(lm), _p(good), _p(counts))
    return m, lm, good, (int(counts[0]), int(counts[1]))


def accept_new_observe(pos, normal, main_octave, octave, min_dist, max_dist):
    return bool(lib().geom_oracle_accept_new_observe(_p(_c(pos, np.float32)), _p(_c(normal, np.float32)), int(main_octave),
                                                     int(octave), float(min_dist), float(max_dist)))


def projection_observations(kf_kp, matches_idx_mp, Tcw_new, mp, Tcw_table, K, lower, upper, fx, pos_init=None, info_init=None):
    """findCorrespd's MatchByProjection branch. mp = dict(main_measure [M,2], main_pose [M], main_octave [M], normal [M,3],
    min_dist [M], max_dist [M]). Returns (accept [n] u8, pos_new_kf [n,3] f4, info_new [n,3,3] f8)."""
    kf_kp = np.ascontiguousarray(kf_kp); n = len(kf_kp)
    a = [_c(matches_idx_mp, np.int32), _c(Tcw_new, np.float32), _c(mp["main_measure"], np.float32), _c(mp["main_pose"], np.int32),
         _c(mp["main_octave"], np.int32), _c(mp["normal"], np.float32), _c(mp["min_dist"], np.float32),
         _c(mp["max_dist"], np.float32), _c(Tcw_table, np.float32), _c(K, np.float32)]
    acc = np.zeros(n, np.uint8)
    pos = np.zeros((n, 3), np.float32) if pos_init is None else _c(pos_init, np.float32).copy()
    info = np.zeros((n, 3, 3)) if info_init is None else _c(info_init, np.float64).copy()
    lib().geom_oracle_projection_observations(n, _p(kf_kp), *[_p(x) for x in a], float(lower), float(upper), float(fx),
                                              _p(acc), _p(pos), _p(info))
    return acc, pos, info
