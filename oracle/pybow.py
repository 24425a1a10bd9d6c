"""CPU restatement of KeyFrame::ComputeBoW (reference src/KeyFrame.cpp:244-254) — TEST INFRASTRUCTURE ONLY.

`compute_bow` is DBoW2's transform(features, v, fv, levelsup): the per-feature descent of oracle/bow_oracle.cpp
(pyoracle.voc_transform), then the BowVector / FeatureVector assembly of oracle/bow_assembly_oracle.cpp (built by
oracle/bow_assembly.mk). The results are arrays in ascending key order, the layout se2gpu_voc_compute_bow_device writes.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

from oracle import pyoracle

HERE = os.path.dirname(os.path.abspath(__file__))
_lib = None


def make() -> str:
    """Bring oracle/libbow_assembly_oracle.so up to date with oracle/bow_assembly.mk and return its path."""
    env = {k: v for k, v in os.environ.items() if k not in ("CXX", "CXXFLAGS")}
    subprocess.run(["make", "-C", HERE, "-s", "-f", "bow_assembly.mk", "CXX=g++"], check=True, env=env)
    return os.path.join(HERE, "libbow_assembly_oracle.so")


def lib():
    global _lib
    if _lib is None:
        L = C.CDLL(make())
        L.bow_oracle_assemble.argtypes = [C.c_void_p] * 3 + [C.c_int] + [C.c_void_p] * 7
        L.bow_oracle_assemble.restype = None
        _lib = L
    return _lib


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def assemble(word, weight, node):
    """(word, weight, node) per feature -> dict(word [W] i4, value [W] f8, node [K] i4, ptr [K+1] i4, feat [F] i4)."""
    w = np.ascontiguousarray(word, np.int32); wt = np.ascontiguousarray(weight, np.float64); nd = np.ascontiguousarray(node, np.int32)
    n = len(w)
    bw, bv = np.zeros(max(n, 1), np.int32), np.zeros(max(n, 1))
    fn, fp, ff = np.zeros(max(n, 1), np.int32), np.zeros(n + 1, np.int32), np.zeros(max(n, 1), np.int32)
    nw, nn = C.c_int(0), C.c_int(0)
    lib().bow_oracle_assemble(_p(w), _p(wt), _p(nd), n, _p(bw), _p(bv), C.byref(nw), _p(fn), _p(fp), _p(ff), C.byref(nn))
    k = nn.value
    return dict(word=bw[:nw.value].copy(), value=bv[:nw.value].copy(), node=fn[:k].copy(), ptr=fp[:k + 1].copy(),
                feat=ff[:fp[k]].copy())


def compute_bow(voc, desc, levelsup=4):
    """transform(features, v, fv, levelsup) for one keyframe's descriptors [n, 32] over the vocabulary dict of
    tests/bow_cases.make_voc."""
    word, weight, node = pyoracle.voc_transform(voc, np.ascontiguousarray(desc, np.uint8).reshape(-1, 32), levelsup)
    return assemble(word, weight, node)
