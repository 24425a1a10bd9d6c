#!/usr/bin/env python
"""Pins the HARRIS_SCORE ORB oracle (oracle/orb_harris_oracle.cpp) against REAL OpenCV code (the cv2 wheel in the build container)
and writes tests/golden/orb_harris_golden.npz.

Run in the build container only (needs cv2):   python oracle/pin_orb_harris_against_cv2.py [--write]

  1. orb_harris_oracle_responses (HarrisResponses, reference src/ORBextractor.cpp:85-126)
                                    == KeyPoint.response of cv2.ORB_create(nlevels=1, scoreType=ORB_HARRIS_SCORE) at cv2's
                                       own keypoints, on blurred noise and on saturated block images (where a = sum Ix^2
                                       exceeds 2^24 and (float)a rounds), bit for bit; and == harris_np below
  2. whole HARRIS_SCORE extractor   == pin_orb_against_cv2.py's composition of the reference orchestration over cv2
     (orb_harris_oracle.cpp)           primitives, run with its cv2 FAST detector wrapped so that every cell's keypoints carry
                                       harris_np of that cell (HarrisResponses follows the FAST / FAST(7) fallback, :625-629),
                                       on the image set of the FAST pin: keypoints (response bits included) and descriptors
The FAST-score pin (pin_orb_against_cv2.py) and orb_golden.npz are not touched.
"""
import os
import sys

import cv2
import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import pin_orb_against_cv2 as pin  # noqa: E402
from pin_orb_against_cv2 import synth  # noqa: E402

from oracle import pyharris  # noqa: E402

f32 = np.float32


def harris_sums(img, x, y):
    """a = sum Ix^2, b = sum Iy^2, c = sum Ix*Iy over the 7x7 block around integer pixel (x, y) of a uint8 image."""
    P = img[y - 4:y + 5, x - 4:x + 5].astype(np.int64)
    Ix = (P[1:-1, 2:] - P[1:-1, :-2]) * 2 + (P[:-2, 2:] - P[:-2, :-2]) + (P[2:, 2:] - P[2:, :-2])
    Iy = (P[2:, 1:-1] - P[:-2, 1:-1]) * 2 + (P[2:, :-2] - P[:-2, :-2]) + (P[2:, 2:] - P[:-2, 2:])
    return int((Ix * Ix).sum()), int((Iy * Iy).sum()), int((Ix * Iy).sum())


def harris_np(img, x, y):
    """HarrisResponses' float32 expression, in C++ evaluation order, at integer pixel (x, y) of a uint8 image."""
    a, b, c = (f32(v) for v in harris_sums(img, x, y))
    s = f32(1) / f32(7140)
    s4 = ((s * s) * s) * s
    k = f32(0.04)
    return f32(f32(f32(a * b) - f32(c * c)) - f32(f32(k * f32(a + b)) * f32(a + b))) * s4


class HarrisCellCv2:
    """cv2 as pin_orb_against_cv2.py's composition uses it, except that FAST detection on a cell returns keypoints whose
    response is harris_np on the bordered level the cell is a view of (the 3x3 gradients reach one pixel beyond the cell)."""

    def __getattr__(self, name):
        return getattr(cv2, name)

    def FastFeatureDetector_create(self, *args):
        det = cv2.FastFeatureDetector_create(*args)

        class Detector:
            def detect(self, cell):
                plane = cell.base
                assert plane is not None and plane.ndim == 2 and plane.flags.c_contiguous
                oy, ox = divmod(cell.ctypes.data - plane.ctypes.data, plane.strides[0])
                kps = det.detect(cell)
                for k in kps:
                    k.response = float(harris_np(plane, ox + int(k.pt[0]), oy + int(k.pt[1])))
                return kps
        return Detector()


def py_extract_harris(img):
    pin.cv2 = HarrisCellCv2()
    try:
        return pin.py_extract(img)
    finally:
        pin.cv2 = cv2


def harris_images():
    rng = np.random.default_rng(11)
    imgs = []
    for _ in range(4):   # blurred noise
        imgs.append(cv2.GaussianBlur(rng.integers(0, 256, (480, 640), dtype=np.uint8), (5, 5), 1.5))
    for blk in (2, 2, 3, 4):  # saturated blocks: |Ix|, |Iy| up to 1020, a and b beyond 2^24
        g = rng.integers(0, 2, (480 // blk + 1, 640 // blk + 1)).astype(np.uint8) * 255
        imgs.append(np.ascontiguousarray(np.kron(g, np.ones((blk, blk), np.uint8))[:480, :640]))
    return imgs


def check_primitive():
    bad = total = big = 0
    for img in harris_images():
        kps = cv2.ORB_create(nfeatures=1500, nlevels=1, scoreType=cv2.ORB_HARRIS_SCORE).detect(img)
        xs = np.array([k.pt[0] for k in kps], f32); ys = np.array([k.pt[1] for k in kps], f32)
        ref = np.array([k.response for k in kps], f32)
        got = pyharris.harris(img, xs, ys)
        npy = np.array([harris_np(img, int(x), int(y)) for x, y in zip(xs, ys)], f32)
        bad += int((got.view(np.uint32) != ref.view(np.uint32)).sum()) + int((npy.view(np.uint32) != got.view(np.uint32)).sum())
        total += len(kps)
        big += sum(1 for x, y in zip(xs, ys) if max(harris_sums(img, int(x), int(y))[:2]) > 1 << 24)
    print(f"[h1] HarrisResponses vs cv2.ORB(HARRIS_SCORE): {bad} differing values over {total} keypoints "
          f"({big} with a or b above 2^24)")
    return bad == 0 and total > 2000


def cases():
    return [("synth1000", synth.orb_frame(1000)), ("synth1001", synth.orb_frame(1001)),
            ("constant", synth.orb_adversarial("constant")), ("noise", synth.orb_adversarial("noise")),
            ("lowcontrast", synth.orb_adversarial("lowcontrast")), ("gradient", synth.orb_adversarial("gradient")),
            ("small_320x240", synth.orb_frame(5, 320, 240)), ("odd_501x377", synth.orb_frame(6, 501, 377))]


def check_full(write):
    ok = True
    gold = {}
    for name, img in cases():
        k_or, d_or = pyharris.HarrisOrbOracle(1000, 1.2, 8, 20).extract(img)
        k_py, d_py = py_extract_harris(img)
        same = len(k_or) == len(k_py) and k_or.tobytes() == k_py.tobytes() and d_or.tobytes() == d_py.tobytes()
        nd = int((d_or != d_py).any(axis=1).sum()) if len(k_or) == len(k_py) else -1
        print(f"[h2] {name}: oracle {len(k_or)} kps, cv2-composition {len(k_py)} kps, identical={same}, differing desc rows={nd}")
        ok &= same
        gold[name + "_kps"] = k_or
        gold[name + "_desc"] = d_or
    if write and ok:
        out = os.path.join(HERE, "..", "tests", "golden", "orb_harris_golden.npz")
        np.savez_compressed(out, **gold)
        print("wrote", out, os.path.getsize(out), "bytes")
    return ok


if __name__ == "__main__":
    results = [check_primitive(), check_full("--write" in sys.argv)]
    print("ALL PINNED" if all(results) else "PIN FAILURES", results)
    sys.exit(0 if all(results) else 1)
