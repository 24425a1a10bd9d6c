"""Pins the OpenCV pieces the map-point oracle (oracle/mappoint_oracle.cpp) adds to the geometry oracle's against cv2, bit
for bit: the two chained float gemms of Rcw^T * M * Rcw (cv::gemm with GEMM_1_T, then the small-matrix path) and
Rcw * M * Rcw^T (the small-matrix path, then GEMM_2_T), cv::norm of a Point3f, and Point3f * double. Needs cv2 (4.13);
not run on the GPU machines. Exits non-zero on any mismatch.

A MatExpr A.t() * B * C evaluates A.t() * B as one cv::gemm with GEMM_1_T into a temporary and multiplies the temporary
by C with a second cv::gemm; A * B * C.t() is gemm(A, B) then gemm(tmp, C, GEMM_2_T). cv2 exposes cv::gemm, so the two
chains are pinned through it. cv::norm(Point3f) is pinned through cv2.norm of the same three floats, and Point3f * double
(each coordinate times the double, rounded once to float) through cv2.multiply of a float column by ones with that scale.

    python oracle/pin_mappoint_against_cv2.py
"""
from __future__ import annotations

import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import cv2  # noqa: E402

from oracle import pymappoint as pm  # noqa: E402

f32 = np.float32


def rotations(rng, n):
    out = []
    for _ in range(n):
        rv = rng.normal(0, 1.0, 3).astype(f32)
        R, _ = cv2.Rodrigues(rv.astype(np.float64))
        out.append(R.astype(f32))
    return out


def main():
    rng = np.random.default_rng(2026)
    bad = {"RtMR": 0, "RMRt": 0, "gemm_2T": 0, "norm": 0, "mul_pd": 0}
    for R in rotations(rng, 2000):
        M = np.diag(rng.uniform(1, 1e5, 3)).astype(f32)
        M += (rng.normal(0, 1, (3, 3)) * rng.uniform(0, 50)).astype(f32) * (rng.random() < 0.5)
        want = cv2.gemm(cv2.gemm(R, M, 1, None, 0, flags=cv2.GEMM_1_T), R, 1, None, 0)
        bad["RtMR"] += int((pm.rt_m_r(R, M).view(np.uint32) != want.view(np.uint32)).sum())
        want = cv2.gemm(cv2.gemm(R, M, 1, None, 0), R, 1, None, 0, flags=cv2.GEMM_2_T)
        bad["RMRt"] += int((pm.r_m_rt(R, M).view(np.uint32) != want.view(np.uint32)).sum())
        A = (rng.normal(0, 1, (3, 3)) * 10 ** rng.uniform(-2, 4)).astype(f32)
        bad["gemm_2T"] += int((pm.gemm3_a_bt(A, M).view(np.uint32) != cv2.gemm(A, M, 1, None, 0, flags=cv2.GEMM_2_T).view(np.uint32)).sum())
    for _ in range(20000):
        p = (rng.normal(size=3) * 10 ** rng.uniform(-3, 4)).astype(f32)
        n = pm.norm3(p)
        bad["norm"] += int(n != cv2.norm(p))
        s = 1.0 / n
        want = cv2.multiply(p.reshape(3, 1), np.ones((3, 1), f32), scale=s).reshape(3)
        bad["mul_pd"] += int((pm.mul_pd(p, s).view(np.uint32) != want.view(np.uint32)).sum())
    print(bad)
    return 0 if not any(bad.values()) else 1


if __name__ == "__main__":
    sys.exit(main())
