"""CPU restatement of loop closure (reference GlobalMapper / Localizer DetectLoopClose and VerifyLoopClose) — TEST
INFRASTRUCTURE ONLY.

`detect` and `score` run oracle/loop_oracle.cpp (built by oracle/loop.mk). `verify` composes the SearchByBoW oracle
(pyoracle.search_by_bow), RemoveMatchOutlierRansac over cv::findFundamentalMat's oracle (pyfundam.find_fundamental_mat)
and loop_oracle.cpp's RemoveKPMatch and verdict. `dbow2_score` is DBoW2's own L1Scoring::score, compiled from the reference
tree by oracle/dbow2_ref.mk into oracle/_ref/ (None when that library was never built).
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

from oracle import pyfundam, pyoracle

HERE = os.path.dirname(os.path.abspath(__file__))
REF_LIB = os.path.join(HERE, "_ref", "libdbow2_l1.so")
_lib = None
_ref = None

DETECT_GLOBAL_MAPPER, DETECT_LOCALIZER = (20, 0.005), (0, 0.05)
VERIFY_GLOBAL_MAPPER, VERIFY_LOCALIZER = (0, 15, 30, 0.05), (1, 0, 45, 0.0)


def make() -> str:
    """Bring oracle/libloop_oracle.so up to date with oracle/loop.mk and return its path."""
    env = {k: v for k, v in os.environ.items() if k not in ("CXX", "CXXFLAGS")}
    subprocess.run(["make", "-C", HERE, "-s", "-f", "loop.mk", "CXX=g++"], check=True, env=env)
    return os.path.join(HERE, "libloop_oracle.so")


def reference_tree():
    """The reference source tree: $SE2LAM_REFERENCE, else a checkout named `reference` beside this repository; None when
    neither holds DBoW2."""
    for cand in (os.environ.get("SE2LAM_REFERENCE"), os.path.join(HERE, "..", "..", "reference")):
        if cand and os.path.isfile(os.path.join(cand, "Thirdparty", "DBoW2", "DBoW2", "ScoringObject.cpp")):
            return os.path.abspath(cand)
    return None


def make_ref():
    """Build oracle/_ref/libdbow2_l1.so from the reference tree when it is present; otherwise leave an existing library
    as it is. Returns the library's path, or None when there is none."""
    ref = reference_tree()
    if ref:
        subprocess.run(["make", "-C", HERE, "-s", "-f", "dbow2_ref.mk", "REF=" + ref], check=True)
    return REF_LIB if os.path.exists(REF_LIB) else None


def lib():
    global _lib
    if _lib is None:
        L = C.CDLL(make())
        vp, i, d = C.c_void_p, C.c_int, C.c_double
        L.loop_oracle_score.argtypes = [vp, vp, i, vp, vp, i]
        L.loop_oracle_score.restype = d
        L.loop_oracle_detect.argtypes = [i, vp, vp, vp, i, i, vp, vp, vp, i, vp, vp, i, d, vp, vp, vp]
        L.loop_oracle_detect.restype = None
        L.loop_oracle_verify_tail.argtypes = [i, vp, vp, vp, i, vp, i, i, i, d, i, vp, vp]
        L.loop_oracle_verify_tail.restype = i
        _lib = L
    return _lib


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def _bow(w, v):
    w = np.ascontiguousarray(w, np.int32); v = np.ascontiguousarray(v, np.float64)
    return (w if len(w) else np.zeros(1, np.int32)), (v if len(v) else np.zeros(1)), len(w)


def score(w1, v1, w2, v2):
    """L1Scoring::score(v1, v2) of two BowVectors given as ascending words and their values."""
    a, b = _bow(w1, v1), _bow(w2, v2)
    return lib().loop_oracle_score(_p(a[0]), _p(a[1]), a[2], _p(b[0]), _p(b[1]), b[2])


def dbow2_score(w1, v1, w2, v2):
    """DBoW2's own L1Scoring::score (oracle/_ref/libdbow2_l1.so), or None when that library is absent."""
    global _ref
    if _ref is None:
        if not os.path.exists(REF_LIB):
            return None
        _ref = C.CDLL(REF_LIB)
        _ref.dbow2_l1_score.argtypes = [C.c_void_p, C.c_void_p, C.c_int] * 2
        _ref.dbow2_l1_score.restype = C.c_double
    a, b = _bow(w1, v1), _bow(w2, v2)
    return _ref.dbow2_l1_score(_p(a[0]), _p(a[1]), a[2], _p(b[0]), _p(b[1]), b[2])


def dbow2_detect_ms(qw, qv, db_word, db_value, db_n, reps=3):
    """DetectLoopClose's loop with DBoW2's own score on one core (the BowVector copy included): (ms per query, best score),
    or None when oracle/_ref/libdbow2_l1.so is absent."""
    if dbow2_score([], [], [], []) is None:
        return None
    c = np.ascontiguousarray
    a, b = _bow(qw, qv)[:2], (c(db_word, np.int32), c(db_value, np.float64), c(db_n, np.int32))
    _ref.dbow2_l1_detect_ms.argtypes = [C.c_void_p, C.c_void_p, C.c_int] + [C.c_void_p] * 3 + [C.c_int] * 3 + [C.c_void_p]
    _ref.dbow2_l1_detect_ms.restype = C.c_double
    best = C.c_double(0)
    ms = _ref.dbow2_l1_detect_ms(_p(a[0]), _p(a[1]), len(qw), _p(b[0]), _p(b[1]), _p(b[2]), b[0].shape[1], len(b[2]), reps, C.byref(best))
    return ms, best.value


def detect(q_word, q_value, q_n, db_word, db_value, db_n, q_id=None, db_id=None, params=DETECT_GLOBAL_MAPPER):
    """DetectLoopClose for B queries ([B, cap_q] arrays, counts [B]) against N keyframes ([N, cap_db], [N]) in slot
    order. Returns (scores [B, N] f8, loop [B] i4, best [B] f8)."""
    c = np.ascontiguousarray
    qw, qv, qn = c(q_word, np.int32), c(q_value, np.float64), c(q_n, np.int32)
    dw, dv, dn = c(db_word, np.int32), c(db_value, np.float64), c(db_n, np.int32)
    B, cap_q = qw.shape; N, cap_db = dw.shape
    qi = c(q_id if q_id is not None else np.zeros(B), np.int32)
    di = c(db_id if db_id is not None else np.zeros(N), np.int32)
    scores = np.zeros((B, N)); loop = np.zeros(B, np.int32); best = np.zeros(B)
    keep = [qw, qv, dw, dv]
    pp = [(_p(a) if a.size else None) for a in keep]
    lib().loop_oracle_detect(B, pp[0], pp[1], _p(qn), cap_q, N, pp[2], pp[3], _p(dn) if N else None, cap_db, _p(qi),
                             _p(di) if N else None, int(params[0]), float(params[1]), _p(scores) if scores.size else None,
                             _p(loop), _p(best))
    return scores, loop, best


def remove_match_outlier_ransac(xy_cur, xy_loop, matches):
    """GlobalMapper::RemoveMatchOutlierRansac (src/GlobalMapper.cpp:1207-1248) on matches [n1] (-1 = none): fewer than 10
    clear everything; else findFundamentalMat(FM_RANSAC, 3, 0.99) on the pairs in ascending current index, the mask's
    matches kept (none when OpenCV never creates the mask)."""
    m = np.asarray(matches, np.int32)
    good = np.full(len(m), -1, np.int32)
    idx = np.flatnonzero(m >= 0)
    if len(idx) < 10:
        return good
    mask, _, _ = pyfundam.find_fundamental_mat(np.asarray(xy_cur, np.float32)[idx], np.asarray(xy_loop, np.float32)[m[idx]])
    if mask is not None:
        keep = idx[mask.astype(bool)]
        good[keep] = m[keep]
    return good


def verify(cur, loop, params=VERIFY_GLOBAL_MAPPER, n_mps_cur=0):
    """VerifyLoopClose for one pair. cur / loop: dict(angle, desc, node, ptr, feat, x, y (keyPointsUn), obs
    (hasObservation(idx))). Returns (raw, good, mp [n1] i4, counts (raw, good, MP), verdict)."""
    n1, n2 = len(cur["angle"]), len(loop["angle"])
    k1 = dict(cur, has_mp=np.zeros(n1, np.uint8)); k2 = dict(loop, has_mp=np.zeros(n2, np.uint8))
    _, raw = pyoracle.search_by_bow(k1, k2, False, 0.6, True)
    raw = np.asarray(raw, np.int32)
    good = remove_match_outlier_ransac(np.stack([cur["x"], cur["y"]], 1), np.stack([loop["x"], loop["y"]], 1), raw)
    mp = np.zeros(max(n1, 1), np.int32); counts = np.zeros(3, np.int32)
    o1 = np.ascontiguousarray(cur["obs"], np.uint8); o2 = np.ascontiguousarray(loop["obs"], np.uint8)
    r, g = np.ascontiguousarray(raw), np.ascontiguousarray(good)
    z = lambda a: a if len(a) else np.zeros(1, a.dtype)
    ok = lib().loop_oracle_verify_tail(n1, _p(z(r)), _p(z(g)), _p(z(o1)), n2, _p(z(o2)), int(params[0]), int(params[1]), int(params[2]),
                                       float(params[3]), int(n_mps_cur), _p(mp), _p(counts))
    return raw, good, mp[:n1].copy(), counts, bool(ok)
