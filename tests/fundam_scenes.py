"""Seeded scene families for Track::removeOutliers beyond the cv2-pinned fixture (tests/golden/fundam_golden.npz): inputs
cv2 refuses or never produced, which the oracle (oracle/fundam_oracle.cpp) is defined on all the same.

  static     zero motion (x2 == x1), float and integer coordinates; half static, half moving; a pure image shift
  lattice    a rigid point set seen from two SE(2) poses, each image point snapped to the float32 lattice of an ORB
             octave (k * 1.2^l), with 0-60 % outliers drawn from the same lattices
  collinear  every pair on one exactly representable line: getSubset gives up on the first draw
  duplicate  most pairs stacked on a few coordinates
  giveup     collinear but for 1-3 points in frame 1: getSubset gives up after some hypotheses, before niters is reached

Numpy only. Each scene turns into a frame pair (kp1, kp2, matches12) with fundam_cases.frame_pair: unmatched keypoints
interleaved in frame 1, frame 2 permuted. `expect` names the estimator branch a scene is there for;
tests/test_fundam_scenes_oracle.py checks that the oracle takes it.
"""
from __future__ import annotations

import numpy as np

from tests.fundam_cases import frame_pair
from tools import geom_scenes as gs

KP_DTYPE = gs.KP_DTYPE
MAX_PAIRS = 8192                      # the device's keypoint capacity per frame
SCALE = np.float32(1.2)               # ORB's scale factor: octave l has lattice step float32(1.2 ** l)
SHIFT = np.array([3.5, -2.25], np.float32)

STATIC_N = [7, 8, 13, 14, 15, 16, 100, 1000, 8192]
LATTICE_N = [15, 16, 31, 32, 33, 255, 256, 257, 1000, 4095, 4096, 8191, 8192]
LATTICE_LMEDS_N = [8, 11, 14]
COLLINEAR_N = [8, 12, 14, 15, 40, 1000]
# zero motion at n = 1000: whether some 7-point elimination gets past its |pivot| < DBL_EPSILON test is decided by
# round-off, so these seeds were picked with the oracle for each outcome
STATIC_1000_SEEDS = {"none": [(False, 100), (True, 100), (False, 102)],
                     "model": [(False, 111), (False, 121), (True, 101), (True, 113)]}
# (n, points off the line, seed): picked with the oracle so that getSubset's 10 000 attempts run out after 1, 3, 31,
# 432, 720 and 893 hypotheses, before niters
GIVEUP = [(6000, 1, 11), (3000, 1, 4), (2000, 1, 2), (4000, 2, 0), (5000, 3, 2), (6000, 3, 0)]


class Scene:
    def __init__(self, family, name, p1, p2, seed, expect, cap=MAX_PAIRS):
        self.family, self.name, self.seed, self.expect, self.cap = family, name, seed, expect, cap
        self.p1 = np.ascontiguousarray(p1, np.float32); self.p2 = np.ascontiguousarray(p2, np.float32)
        self.n = len(self.p1)

    @property
    def branch(self):
        return "empty" if self.n < 7 else "7" if self.n == 7 else "lmeds" if self.n < 15 else "ransac"

    def keypoints(self, kp_dtype=KP_DTYPE, variant=0):
        """The frame pair; another `variant` interleaves other unmatched keypoints around the same matched pairs."""
        return frame_pair(self.p1, self.p2, kp_dtype, np.random.default_rng([self.seed, variant]), cap=self.cap)

    def __repr__(self):
        return f"{self.family}/{self.name}"


def _uniform(rng, n, integer):
    if integer:
        return np.stack([rng.integers(0, 640, n), rng.integers(0, 480, n)], 1).astype(np.float32)
    return np.stack([rng.uniform(0, 640, n), rng.uniform(0, 480, n)], 1).astype(np.float32)


def snap(xy, octave):
    """Each point to the float32 lattice of its octave: round(x / s_l) * s_l, s_l = float32(1.2 ** l)."""
    s = (np.float64(SCALE) ** np.asarray(octave, np.float64)).astype(np.float32)[:, None]
    xy = np.asarray(xy, np.float32)
    return (np.round(xy / s).astype(np.float32) * s).astype(np.float32)


def two_view(n, rng):
    """Image points of n world points seen from two SE(2) poses of the base: forward 0.1-0.4 m, turn within 0.15 rad."""
    T1 = gs.tcw_of_odom(0.0, 0.0, 0.0).astype(np.float64)
    d, th = rng.uniform(0.1, 0.4), rng.uniform(-0.15, 0.15)
    T2 = gs.tcw_of_odom(d * np.cos(th / 2), d * np.sin(th / 2), th).astype(np.float64)
    K = gs.K.astype(np.float64)
    z = rng.uniform(1.0, 8.0, n)
    u, v = rng.uniform(0, gs.W, n), rng.uniform(0, gs.H, n)
    Xc = np.stack([(u - K[0, 2]) / K[0, 0] * z, (v - K[1, 2]) / K[1, 1] * z, z, np.ones(n)], 1)
    Xw = (np.linalg.inv(T1) @ Xc.T).T[:, :3]
    P1, P2 = K @ T1[:3], K @ T2[:3]
    return np.array([gs.project(P1, X) for X in Xw]), np.array([gs.project(P2, X) for X in Xw])


def lattice_pairs(n, seed, outliers):
    rng = np.random.default_rng(seed)
    q1, q2 = two_view(n, rng)
    octave = rng.integers(0, 8, n)
    p1, p2 = snap(q1, octave), snap(q2, octave)
    k = rng.choice(n, int(round(outliers * n)), replace=False)
    p2[k] = snap(_uniform(rng, len(k), False), rng.integers(0, 8, len(k)))
    return p1, p2


def static_scenes():
    out = []
    for integer in (False, True):
        kind = "int" if integer else "float"
        for n in STATIC_N:
            p = _uniform(np.random.default_rng(n), n, integer)
            out.append(Scene("static", f"{kind} n{n}", p, p, 10_000 + n + integer, "static"))
    for outcome, seeds in STATIC_1000_SEEDS.items():
        for integer, seed in seeds:
            p = _uniform(np.random.default_rng(seed), 1000, integer)
            out.append(Scene("static", f"{'int' if integer else 'float'} n1000 seed {seed}", p, p, 20_000 + seed + integer,
                             "static-" + outcome))
    for n in (100, 1000):
        p1, p2 = lattice_pairs(n, 30_000 + n, 0.0)
        p2[: n // 2] = p1[: n // 2]
        out.append(Scene("static", f"half static n{n}", p1, p2, 31_000 + n, "ransac"))
        p = _uniform(np.random.default_rng(32_000 + n), n, False)
        out.append(Scene("static", f"shift n{n}", p, p + SHIFT, 33_000 + n, "ransac"))
    return out


def lattice_scenes():
    fracs = [0.0, 0.1, 0.2, 0.3, 0.4, 0.5, 0.6]
    out = []
    for i, n in enumerate(LATTICE_N):
        f = fracs[i % len(fracs)]
        p1, p2 = lattice_pairs(n, 40_000 + n, f)
        out.append(Scene("lattice", f"n{n} {int(f * 100)}% out", p1, p2, 41_000 + n, "ransac"))
    for n in LATTICE_LMEDS_N:                        # the LMedS median over lattice-tied errors
        p1, p2 = lattice_pairs(n, 42_000 + n, 0.2)
        out.append(Scene("lattice", f"n{n} 20% out", p1, p2, 43_000 + n, "lmeds"))
    return out


def collinear_scenes():
    out = []
    for n in COLLINEAR_N:
        rng = np.random.default_rng(50_000 + n)
        x1 = rng.permutation(np.arange(-400, 400 + n))[:n]
        x2 = rng.permutation(np.arange(-400, 400 + n))[:n]
        p1 = np.stack([x1, 2 * x1 + 11], 1).astype(np.float32)
        p2 = np.stack([x2, 2 * x2 - 5], 1).astype(np.float32)
        out.append(Scene("collinear", f"n{n}", p1, p2, 51_000 + n, "first-draw"))
    for n in (20, 200, 1000):
        rng = np.random.default_rng(52_000 + n)
        p1, p2 = lattice_pairs(n, 53_000 + n, 0.1)
        stack = rng.random(n) < 0.8                  # 80 % of the pairs on one of three coordinate pairs
        which = rng.integers(0, 3, n)
        c1, c2 = _uniform(rng, 3, True), _uniform(rng, 3, True)
        p1[stack] = c1[which[stack]]; p2[stack] = c2[which[stack]]
        out.append(Scene("duplicate", f"n{n}", p1, p2, 54_000 + n, "any"))
    return out


def giveup_pairs(n, off, seed):
    rng = np.random.default_rng(seed * 1000 + n + off)
    x = rng.permutation(np.arange(-2000, 2000 + n))[:n]
    p1 = np.stack([x, 2 * x + 7], 1).astype(np.float32)
    p2 = _uniform(rng, n, False)
    k = rng.choice(n, off, replace=False)
    p1[k] = rng.uniform(0, 480, (off, 2)).astype(np.float32)
    return p1, p2


def giveup_scenes():
    return [Scene("giveup", f"n{n} off {off} seed {seed}", *giveup_pairs(n, off, seed), 60_000 + n + off, "giveup")
            for n, off, seed in GIVEUP]


def all_scenes():
    return static_scenes() + lattice_scenes() + collinear_scenes() + giveup_scenes()


def sparse_capacity_pair(seed=70_000, matched=20):
    """cap1 = 8192 keypoints of which only `matched` are matched (a lattice scene with 2 outliers)."""
    rng = np.random.default_rng(seed)
    p1, p2 = lattice_pairs(matched, seed, 0.1)
    kp1 = np.zeros(MAX_PAIRS, KP_DTYPE); kp2 = np.zeros(MAX_PAIRS, KP_DTYPE)
    for kp in (kp1, kp2):
        kp["x"], kp["y"] = snap(_uniform(rng, MAX_PAIRS, False), rng.integers(0, 8, MAX_PAIRS)).T
    slots = np.sort(rng.choice(MAX_PAIRS, matched, replace=False))
    perm = rng.permutation(MAX_PAIRS)[:matched]
    kp1["x"][slots], kp1["y"][slots] = p1.T
    kp2["x"][perm], kp2["y"][perm] = p2.T
    m = np.full(MAX_PAIRS, -1, np.int32)
    m[slots] = perm
    return kp1, kp2, m
