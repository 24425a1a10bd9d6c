"""Pins the two-view geometry oracle (oracle/geom_oracle.cpp) against the cv2 calls its restated primitives resolve to, bit
for bit, and writes tests/golden/geom_golden.npz. Needs cv2; not run on the GPU machines. DESIGN.md section 8 states
what each pin covers and on which host arithmetic it depends.

    python oracle/pin_geom_against_cv2.py [--check]     (--check: compare with the committed fixture, write nothing)
"""
from __future__ import annotations

import ctypes
import math
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import cv2  # noqa: E402

from oracle import pygeom  # noqa: E402
from tools import geom_scenes as gs  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "geom_golden.npz")
f32 = np.float32


def a_matrices():
    """4x4 A matrices of cvu::triangulate: real two-view systems, then the degenerate families."""
    rng = np.random.default_rng(2024)
    out, kind = [], []
    sc = gs.triangulate_scene(200, seed=7)
    for i in range(200):
        out.append(pygeom.build_a(sc["pt1"][i], sc["pt2"][i], sc["P"][sc["idx1"][i]], sc["P"][sc["idx2"][i]])); kind.append(0)
    P0 = (gs.K.astype(np.float64) @ np.eye(3, 4)).astype(f32)
    for t in range(40):                                                    # zero baseline: P2 = K [R | 0]
        th = rng.uniform(-0.3, 0.3)
        R = np.array([[np.cos(th), 0, np.sin(th)], [0, 1, 0], [-np.sin(th), 0, np.cos(th)]])
        P2 = (gs.K.astype(np.float64) @ np.hstack([R, np.zeros((3, 1))])).astype(f32)
        p = rng.uniform(0, 640, 2).astype(f32)
        out.append(pygeom.build_a(p, p + f32(rng.normal(0, 2)), P0, P2)); kind.append(1)
    for t in range(40):                                                    # identical points in both views, same P
        p = rng.uniform(0, 640, 2).astype(f32)
        out.append(pygeom.build_a(p, p, sc["P"][t % 8], sc["P"][t % 8])); kind.append(2)
    for t in range(40):                                                    # repeated singular values
        Q, _ = np.linalg.qr(rng.normal(size=(4, 4)))
        s = [rng.choice([1.0, 2.0, 100.0])] * 2 + [rng.choice([0.5, 1.0])] * 2
        out.append((Q @ np.diag(s) @ np.linalg.qr(rng.normal(size=(4, 4)))[0]).astype(f32)); kind.append(3)
    for t in range(20):
        out.append(np.diag([1, 1, 1, 1]).astype(f32) * f32(rng.choice([1, 3]))); kind.append(3)
        out.append(np.zeros((4, 4), f32)); kind.append(3)
    for t in range(40):                                                    # point at infinity: A's null vector has w = 0
        d = np.append(rng.normal(size=3), 0.0)
        M = rng.normal(size=(4, 4)); M -= np.outer(M @ d, d) / (d @ d)
        out.append(M.astype(f32)); kind.append(4)
    for t in range(40):                                                    # a point behind the camera
        X = np.array([rng.uniform(-1, 1), rng.uniform(-1, 1), -rng.uniform(0.5, 5)])
        P2 = sc["P"][1 + t % 7]
        p1 = gs.project(P0.astype(np.float64), X).astype(f32); p2 = gs.project(P2.astype(np.float64), X).astype(f32)
        out.append(pygeom.build_a(p1, p2, P0, P2)); kind.append(5)
    return np.stack(out).astype(f32), np.array(kind, np.int32)


def asinf_restated(x):
    """glibc 2.39 __ieee754_asinf on float32 arrays in [0, 1] (the branch structure of sysdeps/ieee754/flt-32/e_asinf.c)."""
    x = np.asarray(x, f32)
    p0, p1, p2, p3, p4 = f32(1.666675248e-1), f32(7.495297643e-2), f32(4.547037598e-2), f32(2.417951451e-2), f32(4.216630880e-2)
    pio2_hi, pio2_lo, pio4_hi = f32(1.57079637050628662109375), f32(-4.37113900018624283e-8), f32(0.785398185253143310546875)
    ix = x.view(np.uint32) & np.uint32(0x7FFFFFFF)
    with np.errstate(all="ignore"):
        t = x * x
        small = x + x * (t * (p0 + t * (p1 + t * (p2 + t * (p3 + t * p4)))))
        t = (f32(1) - np.abs(x)) * f32(0.5)
        p = t * (p0 + t * (p1 + t * (p2 + t * (p3 + t * p4))))
        s = np.sqrt(t)
        near1 = pio2_hi - (f32(2) * (s + s * p) - pio2_lo)
        w = (s.view(np.uint32) & np.uint32(0xFFFFF000)).view(f32)
        c = (t - w * w) / (s + w)
        mid = pio4_hi - ((f32(2) * s * p - (pio2_lo - f32(2) * c)) - (pio4_hi - f32(2) * w))
        r = np.where(ix >= 0x3F79999A, near1, mid)
        r = np.where(ix < 0x3F000000, np.where(ix < 0x32000000, x, small), r)
        r = np.where(ix == 0x3F800000, x * pio2_hi + x * pio2_lo, r)
    return r.astype(f32)


def main():
    check = "--check" in sys.argv
    rng = np.random.default_rng(99)
    res = {}
    bad = {}

    # SVD::compute(A, w, u, vt, MODIFY_A | FULL_UV) -> cv2.SVDecomp with the same flags
    A, kind = a_matrices()
    w_cv = np.zeros((len(A), 4), f32); vt_cv = np.zeros((len(A), 4, 4), f32)
    for i, a in enumerate(A):
        w, _, vt = cv2.SVDecomp(a.copy(), flags=cv2.SVD_MODIFY_A | cv2.SVD_FULL_UV)
        w_cv[i] = w.ravel(); vt_cv[i] = vt
    w_o, vt_o = pygeom.svd4(A)
    bad["svd4"] = int((w_o.view(np.uint32) != w_cv.view(np.uint32)).sum() + (vt_o.view(np.uint32) != vt_cv.view(np.uint32)).sum())
    res.update(svd_A=A, svd_kind=kind, svd_w=w_cv, svd_vt=vt_cv)

    # A.row(r) = x * P.row(2) - P.row(0) -> cv2.addWeighted(P.row(2), x, P.row(0), -1, 0)
    rows_P = (rng.normal(size=(500, 2, 4)) * [[300], [1]]).astype(f32)
    rows_x = rng.uniform(0, 640, 500).astype(f32)
    rows_cv = np.stack([cv2.addWeighted(rows_P[i, 1:2], float(rows_x[i]), rows_P[i, 0:1], -1.0, 0.0).ravel() for i in range(500)])
    rows_o = np.zeros_like(rows_cv)
    for i in range(500):
        P = np.zeros((3, 4), f32); P[0] = rows_P[i, 0]; P[2] = rows_P[i, 1]
        rows_o[i] = pygeom.build_a(np.array([rows_x[i], 0], f32), np.zeros(2, f32), P, P)[0]
    bad["addWeighted_row"] = int((rows_o.view(np.uint32) != rows_cv.view(np.uint32)).sum())
    res.update(row_P=rows_P, row_x=rows_x, row_out=rows_cv)

    # Kcam * T.rowRange(0,3) and -RT * t -> cv2.gemm (small-matrix path); R.t() * info -> cv2.gemm(..., GEMM_1_T)
    gA = (rng.normal(size=(300, 3, 3)) * 200).astype(f32); gB = rng.normal(size=(300, 3, 4)).astype(f32)
    g34 = np.stack([cv2.gemm(gA[i], gB[i], 1, None, 0) for i in range(300)])
    g31 = np.stack([cv2.gemm(gA[i], gB[i, :, 3:4].copy(), -1, None, 0) for i in range(300)])
    gD = np.stack([np.diag(rng.uniform(1, 1e5, 3)) for _ in range(300)]).astype(f32)
    gT = np.stack([cv2.gemm(gA[i], gD[i], 1, None, 0, flags=cv2.GEMM_1_T) for i in range(300)])
    o34 = np.stack([pygeom.gemm3(gA[i], gB[i]) for i in range(300)])
    o31 = np.stack([pygeom.gemm3(gA[i], gB[i, :, 3:4], -1.0) for i in range(300)])
    oT = np.stack([pygeom.gemm3_at_b(gA[i], gD[i]) for i in range(300)])
    bad["gemm_3x4"] = int((o34.view(np.uint32) != g34.view(np.uint32)).sum())
    bad["gemm_3x1_alpha-1"] = int((o31.view(np.uint32) != g31.view(np.uint32)).sum())
    bad["gemm_1T"] = int((oT.view(np.uint32) != gT.view(np.uint32)).sum())
    res.update(gemm_A=gA, gemm_B=gB, gemm_D=gD, gemm_34=g34, gemm_31=g31, gemm_1T=gT)

    # cv::Rodrigues of a float 3x1 vector
    rv = (rng.normal(size=(500, 3)) * rng.choice([1e-4, 0.05, 0.5, 2.0], (500, 1))).astype(f32)
    rv[:5] = 0
    R_cv = np.stack([cv2.Rodrigues(rv[i].reshape(3, 1))[0] for i in range(500)])
    R_o = np.stack([pygeom.rodrigues(rv[i]) for i in range(500)])
    bad["rodrigues"] = int((R_o.view(np.uint32) != R_cv.view(np.uint32)).sum())
    res.update(rod_v=rv, rod_R=R_cv)

    # cv::norm(Point3f) = sqrt of the double sum of squares -> cv2.norm of a 3-vector (NORM_L2)
    pts = (rng.normal(size=(500, 3)) * 5).astype(f32)
    n_cv = np.array([cv2.norm(p.reshape(3, 1)) for p in pts])
    n_o = np.array([math.sqrt(float(p[0]) * float(p[0]) + float(p[1]) * float(p[1]) + float(p[2]) * float(p[2])) for p in pts])
    bad["norm_point3f"] = int((n_cv != n_o).sum())

    # host libm: std::asin(float) is glibc's asinf; the device restates its algorithm (geom.cu asinf_host), checked here
    # in numpy float32 against libm on every 257th float of [0, 1]
    libm = ctypes.CDLL("libm.so.6")
    libm.asinf.restype = ctypes.c_float; libm.asinf.argtypes = [ctypes.c_float]
    xs = np.arange(0, 0x3F800001, 257, dtype=np.uint32).view(f32)
    bad["asinf_restated"] = int(np.count_nonzero(np.array([libm.asinf(float(x)) for x in xs], f32).view(np.uint32)
                                                 != asinf_restated(xs).view(np.uint32)))
    # hypot: JacobiSVDImpl_ calls lapack.cpp's inline template, not libm (cv2 imports hypotf but no double hypot), so cv2
    # cannot reach it alone. It is pinned through the SVD: 20 000 more two-view A matrices against cv2.SVDecomp, and the
    # same sample run with libm's hypot instead shows whether the sample tells the two apart (reported, not required).
    big = []
    for seed in range(100):
        sc = gs.triangulate_scene(200, seed=1000 + seed)
        for i in range(200):
            big.append(pygeom.build_a(sc["pt1"][i], sc["pt2"][i], sc["P"][sc["idx1"][i]], sc["P"][sc["idx2"][i]]))
    big = np.stack(big)
    wb = np.zeros((len(big), 4), f32); vb = np.zeros((len(big), 4, 4), f32)
    for i, a in enumerate(big):
        w, _, vt = cv2.SVDecomp(a.copy(), flags=cv2.SVD_MODIFY_A | cv2.SVD_FULL_UV)
        wb[i] = w.ravel(); vb[i] = vt

    def n_diff(w, v):
        return int(((w.view(np.uint32) != wb.view(np.uint32)).any(1) | (v.view(np.uint32) != vb.view(np.uint32)).reshape(len(big), -1).any(1)).sum())
    bad["svd4_20000_matrices"] = n_diff(*pygeom.svd4(big))
    print(f"{'(libm hypot instead)':28s} matrices differing: {n_diff(*pygeom.svd4(big, libm_hypot=True))} of {len(big)}")

    for k, v in bad.items():
        print(f"{k:28s} differing values: {v}")
    total = sum(bad.values())
    if check:
        g = np.load(OUT)
        diff = sum(int(not np.array_equal(np.asarray(g[k]).view(np.uint8), np.asarray(v).view(np.uint8))) for k, v in res.items())
        print("fixture arrays differing from this run:", diff)
        total += diff
    else:
        np.savez_compressed(OUT, **res)
        print("wrote", OUT)
    print("cv2", cv2.__version__, "total differing:", total)
    return 0 if total == 0 else 1


if __name__ == "__main__":
    sys.exit(main())
