"""Pins the outlier-rejection oracle (oracle/fundam_oracle.cpp) against cv2.findFundamentalMat and writes
tests/golden/fundam_golden.npz: every scene's point pairs, cv2's mask (None when cv2 never creates it), cv2's F for the
7-pair scenes and the oracle's hypothesis counts. Needs cv2 (4.13); the tests only read the fixture.

Coordinates are multiples of 1/8 px (stored as int16 eighths), like keypoints on a scaled pyramid level, which keeps the
fixture small and makes exact collinearity and duplicates representable.

    python -m oracle.pin_fundam_against_cv2
"""
from __future__ import annotations

import os

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
OUT = os.path.join(HERE, "..", "tests", "golden", "fundam_golden.npz")

# scene kinds
RANDOM, COLLINEAR, DUPLICATE, STATIC, PLANAR, NOISE = range(6)
KIND_NAMES = ["random", "collinear", "duplicate", "static", "planar", "noise"]


def _q(x):
    return np.clip(np.round(np.asarray(x, np.float64) * 8), -32000, 32000).astype(np.int16)


def two_view(rng, n, outliers, noise=0.7, planar=False, static=False):
    """n pairs of a camera moving past a 3-D (or planar) scene, 640x480, with a share of random outlier pairs."""
    f, cx, cy = 400.0, 320.0, 240.0
    X = np.c_[rng.uniform(-3, 3, n), rng.uniform(-2, 2, n), np.full(n, 8.0) if planar else rng.uniform(4, 12, n)]
    a = rng.uniform(-0.1, 0.1, 3)
    th = np.linalg.norm(a); k = a / th
    Kx = np.array([[0, -k[2], k[1]], [k[2], 0, -k[0]], [-k[1], k[0], 0]])
    R = np.eye(3) + np.sin(th) * Kx + (1 - np.cos(th)) * Kx @ Kx
    t = rng.uniform(-0.5, 0.5, 3)
    if static:
        R, t = np.eye(3), np.zeros(3)
    Y = X @ R.T + t
    x1 = np.c_[f * X[:, 0] / X[:, 2] + cx, f * X[:, 1] / X[:, 2] + cy]
    x2 = np.c_[f * Y[:, 0] / Y[:, 2] + cx, f * Y[:, 1] / Y[:, 2] + cy]
    x1 += rng.normal(0, noise, x1.shape); x2 += rng.normal(0, noise, x2.shape)
    if static:
        x2 = x1.copy()
    k = int(round(outliers * n))
    o = rng.choice(n, k, replace=False)
    x2[o] = np.c_[rng.uniform(0, 640, k), rng.uniform(0, 480, k)]
    return np.c_[_q(x1), _q(x2)]


def scenes(seed=20261016):
    rng = np.random.default_rng(seed)
    out = []   # (kind, int16 [n,4])
    edges = [0, 6, 7, 8, 13, 14, 15, 16, 30, 100, 1000, 2000]
    for n in edges:
        for r in (0.0, 0.1, 0.3, 0.5):
            out.append((RANDOM, two_view(rng, n, r)))
    for _ in range(120):                                  # 7 pairs: the kernel alone
        out.append((RANDOM, two_view(rng, 7, 0.0)))
    for _ in range(240):                                  # LMedS
        out.append((RANDOM, two_view(rng, int(rng.integers(8, 15)), float(rng.choice([0, 0.1, 0.2, 0.3])))))
    for _ in range(2000):                                 # RANSAC, 0 - 70 % outliers
        n = int(rng.choice([15, 16, 20, 25, 30, 40, 50, 70, 100, 150]))
        out.append((RANDOM, two_view(rng, n, float(rng.choice([0, 0.1, 0.2, 0.3, 0.4, 0.5, 0.6, 0.7])))))
    for n, r in [(300, 0.5), (300, 0.6), (300, 0.7), (1000, 0.5), (1000, 0.6), (1000, 0.7), (2000, 0.5), (300, 0.3),
                 (1000, 0.1), (1000, 0.3)]:
        out.append((RANDOM, two_view(rng, n, r)))
    for n in (8, 12, 15, 40, 300):                        # every point on one line: getSubset exhausts its attempts
        x = np.sort(rng.uniform(0, 600, n))
        a = np.c_[x, 0.5 * x + 20]; b = np.c_[x * 0.9 + 5, 0.45 * x + 30]
        out.append((COLLINEAR, np.c_[_q(a), _q(b)]))
    for n in (8, 14, 20, 60, 300):                        # duplicated points
        p = two_view(rng, n // 2, 0.2)
        out.append((DUPLICATE, np.concatenate([p, p[: n - n // 2]])[rng.permutation(n)]))
    for n in (8, 15, 50, 300):
        out.append((STATIC, two_view(rng, n, 0.0, static=True)))
    for n in (8, 15, 50, 300, 1000):
        out.append((PLANAR, two_view(rng, n, 0.2, planar=True)))
    for n in (8, 10, 15, 20, 30, 50, 100):                # pure noise: few or no consistent models
        out.append((NOISE, np.c_[_q(rng.uniform(0, 640, (n, 2))), _q(rng.uniform(0, 480, (n, 2)))]))
    return out


def main():
    import cv2
    from . import pyfundam
    assert cv2.__version__.startswith("4.13"), cv2.__version__
    sc = scenes()
    pts, off, kinds, created, masks, f7, f7_off, iters = [], [0], [], [], [], [], [0], []
    agree = {}
    for kind, p in sc:
        q = p.astype(np.float32) / np.float32(8)
        p1, p2 = q[:, :2].copy(), q[:, 2:].copy()
        n = len(p)
        try:
            F, m = cv2.findFundamentalMat(p1, p2) if n else (None, None)
        except cv2.error:
            # OpenCV's own assertion (a degenerate 7-point solve): the reference would throw, there is nothing to pin
            print("cv2 raised on a", KIND_NAMES[kind], "scene of", n, "pairs; left out")
            continue
        mo, Fo, it = pyfundam.find_fundamental_mat(p1, p2)
        pts.append(p); off.append(off[-1] + n); kinds.append(kind); created.append(m is not None)
        masks.append(np.zeros(n, np.uint8) if m is None else m.ravel().astype(np.uint8))
        iters.append(it)
        if n == 7 and F is not None:
            f7.append(F.reshape(-1, 3, 3))
        f7_off.append(f7_off[-1] + (len(f7[-1]) if n == 7 and F is not None else 0))
        branch = "empty" if n < 7 else "7" if n == 7 else "lmeds" if n < 15 else "ransac"
        same = (m is None) == (mo is None) and (m is None or np.array_equal(m.ravel(), mo))
        a = agree.setdefault(branch, [0, 0]); a[0] += same; a[1] += 1
    np.savez_compressed(
        OUT, pts=np.concatenate(pts), off=np.array(off, np.int64), kind=np.array(kinds, np.int8),
        mask_created=np.array(created), mask_bits=np.packbits(np.concatenate(masks)),
        f7=np.concatenate(f7) if f7 else np.zeros((0, 3, 3)), f7_off=np.array(f7_off, np.int64),
        oracle_iters=np.array(iters, np.int32), cv2_version=np.array(cv2.__version__))
    print("wrote", OUT, "scenes", len(sc), "mask agreement per branch", agree)


if __name__ == "__main__":
    main()
