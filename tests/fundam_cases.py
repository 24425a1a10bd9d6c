"""The scenes of tests/golden/fundam_golden.npz (written by oracle/pin_fundam_against_cv2.py)."""
from __future__ import annotations

import os

import numpy as np

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "fundam_golden.npz")
KIND_NAMES = ["random", "collinear", "duplicate", "static", "planar", "noise"]


class Scene:
    def __init__(self, i, kind, p, created, mask, f7, iters):
        self.i, self.kind, self.created, self.mask, self.f7, self.iters = i, KIND_NAMES[kind], created, mask, f7, iters
        q = p.astype(np.float32) / np.float32(8)
        self.p1, self.p2 = q[:, :2].copy(), q[:, 2:].copy()
        self.n = len(p)

    @property
    def branch(self):
        return "empty" if self.n < 7 else "7" if self.n == 7 else "lmeds" if self.n < 15 else "ransac"

    def keypoints(self, kp_dtype, rng=None):
        return frame_pair(self.p1, self.p2, kp_dtype, rng or np.random.default_rng(self.i))


def frame_pair(p1, p2, kp_dtype, rng, max_extra=4, cap=None):
    """A frame pair whose matched pairs, taken in ascending order, are (p1[k], p2[k]): kp1 with 0..max_extra unmatched
    keypoints interleaved, kp2 a permutation of the frame-2 points with as many extra ones, matches12 pointing into it.
    cap bounds both keypoint counts (the extras are cut first)."""
    n = len(p1)
    extra1, extra2 = int(rng.integers(0, max_extra + 1)), int(rng.integers(0, max_extra + 1))
    n1, n2 = n + extra1, n + extra2
    if cap is not None:
        n1, n2 = min(n1, max(cap, n)), min(n2, max(cap, n))
    kp1 = np.zeros(n1, kp_dtype); kp2 = np.zeros(n2, kp_dtype)
    slots = np.sort(rng.choice(n1, n, replace=False))
    perm = rng.permutation(n2)[:n]
    kp1["x"] = rng.uniform(0, 640, n1); kp1["y"] = rng.uniform(0, 480, n1)
    kp2["x"] = rng.uniform(0, 640, n2); kp2["y"] = rng.uniform(0, 480, n2)
    kp1["x"][slots] = p1[:, 0]; kp1["y"][slots] = p1[:, 1]
    kp2["x"][perm] = p2[:, 0]; kp2["y"][perm] = p2[:, 1]
    m = np.full(n1, -1, np.int32)
    m[slots] = perm
    return kp1, kp2, m


def load():
    z = np.load(GOLDEN)
    bits = np.unpackbits(z["mask_bits"])
    off, f7o = z["off"], z["f7_off"]
    out = []
    for i in range(len(z["kind"])):
        a, b = int(off[i]), int(off[i + 1])
        out.append(Scene(i, int(z["kind"][i]), z["pts"][a:b], bool(z["mask_created"][i]), bits[a:b].astype(np.uint8),
                         z["f7"][f7o[i]:f7o[i + 1]], int(z["oracle_iters"][i])))
    return out
