"""ctypes bindings of the HARRIS_SCORE ORB oracle (oracle/liborb_harris_oracle.so) — TEST INFRASTRUCTURE ONLY.

A library of its own next to liboracle.so, built with the same flags (oracle/Makefile: no -march, -ffp-contract=off);
oracle/orb_harris_oracle.cpp compiles orb_oracle.cpp into the same translation unit. The product package (se2lam_b200)
never imports this module.
"""
from __future__ import annotations

import ctypes as C

import numpy as np

from .pyoracle import KP_DTYPE, make


_lib = None


def lib():
    global _lib
    if _lib is None:
        L = C.CDLL(make("liborb_harris_oracle.so"))
        vp, i, f = C.c_void_p, C.c_int, C.c_float
        L.orb_harris_oracle_create.restype = vp
        L.orb_harris_oracle_create.argtypes = [i, f, i, i]
        L.orb_harris_oracle_destroy.argtypes = [vp]
        L.orb_harris_oracle_extract.argtypes = [vp, vp, i, i, i, vp, vp]
        L.orb_harris_oracle_responses.argtypes = [vp, i, vp, vp, i, vp]
        _lib = L
    return _lib


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


class HarrisOrbOracle:
    """ORBextractor(nfeatures, scaleFactor, nlevels, HARRIS_SCORE, fastTh)."""

    def __init__(self, nfeatures=1000, scale_factor=1.2, nlevels=8, fast_th=20):
        self.nfeatures = nfeatures
        self.h = lib().orb_harris_oracle_create(nfeatures, scale_factor, nlevels, fast_th)

    def __del__(self):
        if getattr(self, "h", None):
            lib().orb_harris_oracle_destroy(self.h)
            self.h = None

    def extract(self, img: np.ndarray):
        img = np.ascontiguousarray(img, np.uint8)
        kps = np.zeros(self.nfeatures + 8, KP_DTYPE)
        desc = np.zeros((self.nfeatures + 8, 32), np.uint8)
        n = lib().orb_harris_oracle_extract(self.h, _p(img), img.shape[1], img.shape[0], img.strides[0], _p(kps), _p(desc))
        return kps[:n].copy(), desc[:n].copy()


def harris(img, xs, ys):
    """HarrisResponses(img, pts, 7, 0.04f) (ORBextractor.cpp:85-126) at the points (xs[i], ys[i]) of a uint8 image."""
    img = np.ascontiguousarray(img, np.uint8)
    xs = np.ascontiguousarray(xs, np.float32); ys = np.ascontiguousarray(ys, np.float32)
    out = np.zeros(len(xs), np.float32)
    lib().orb_harris_oracle_responses(_p(img), img.strides[0], _p(xs), _p(ys), len(xs), _p(out))
    return out
