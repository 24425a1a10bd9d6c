"""Host-side mirror of the bag-of-words front end over the C ABI (se2gpu_voc_*, se2gpu_median_descriptor).

`Vocabulary.transform(descriptors, levelsup)` is DBoW2's TemplatedVocabulary::transform(features, v, fv, levelsup)
(reference Thirdparty/DBoW2/DBoW2/TemplatedVocabulary.h:1150-1216) as KeyFrame::ComputeBoW calls it
(src/KeyFrame.cpp:244-254): the per-descriptor tree descent runs on the GPU, the BowVector / FeatureVector assembly (a
sorted-map accumulation in feature order + L1 normalisation, TF_IDF weighting: the ORBvoc settings) on the host.
`Vocabulary.compute_bow_device` runs both halves on the device for a batch of keyframes (se2gpu_voc_compute_bow_device).
"""
from __future__ import annotations

import ctypes as C

import numpy as np

from . import _capi
from ._capi import check, lib, ptr


class Vocabulary:
    def __init__(self, node_desc, child_ptr, children, word_id, weight, levels, device=0):
        c = np.ascontiguousarray
        self._keep = [c(node_desc, np.uint8).reshape(-1, 32), c(child_ptr, np.int32), c(children, np.int32), c(word_id, np.int32),
                      c(weight, np.float64)]
        self.levels = int(levels)
        self.h = lib().se2gpu_voc_create(len(self._keep[0]), *[ptr(a) for a in self._keep], self.levels, device)
        if not self.h:
            raise _capi.Se2GpuError("se2gpu_voc_create failed: " + _capi.last_error())

    def close(self):
        if getattr(self, "h", None):
            lib().se2gpu_voc_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def transform_features(self, descriptors, levelsup=4):
        """Per feature: (word id, weight, node id at level L - levelsup)."""
        d = np.ascontiguousarray(descriptors, np.uint8).reshape(-1, 32)
        n = len(d)
        word = np.zeros(n, np.int32); weight = np.zeros(n); node = np.zeros(n, np.int32)
        check(lib().se2gpu_voc_transform(self.h, ptr(d), n, int(levelsup), ptr(word), ptr(weight), ptr(node)), "se2gpu_voc_transform")
        return word, weight, node

    def transform(self, descriptors, levelsup=4):
        """(BowVector as {word: value}, FeatureVector as {node: [feature indices]}), TF_IDF + L1 like ORBvoc."""
        word, weight, node = self.transform_features(descriptors, levelsup)
        v, fv = {}, {}
        for i in range(len(word)):                       # :1176-1190, feature order (the float sums depend on it)
            if weight[i] > 0:
                v[int(word[i])] = v.get(int(word[i]), 0.0) + float(weight[i])
                fv.setdefault(int(node[i]), []).append(i)
        norm = 0.0
        for k in sorted(v):                              # BowVector::normalize(L1), map order
            norm += abs(v[k])
        if norm > 0.0:
            for k in v:
                v[k] /= norm
        return dict(sorted(v.items())), dict(sorted(fv.items()))

    def compute_bow_device(self, B, d_desc, cap, d_fv_node, d_fv_ptr, d_fv_feat, d_fv_n, d_bow_word=None, d_bow_value=None,
                           d_bow_n=None, d_n=None, levelsup=4, stream=0):
        """KeyFrame::ComputeBoW for B keyframes on device buffers (CUDA pointers: ints or torch tensors), asynchronous on
        `stream`. Keyframe b: descriptors d_desc + b*cap*32, d_n[b] of them (None: cap); BowVector d_bow_word / d_bow_value
        (float64) + b*cap, d_bow_n[b] words (all three None: FeatureVector only); FeatureVector d_fv_node + b*cap ascending,
        d_fv_ptr + b*(cap+1), d_fv_feat + b*cap, d_fv_n[b] nodes. See se2gpu_voc_compute_bow_device."""
        check(lib().se2gpu_voc_compute_bow_device(self.h, int(B), ptr(d_desc), int(cap), ptr(d_n), int(levelsup), ptr(d_bow_word),
                                                  ptr(d_bow_value), ptr(d_bow_n), ptr(d_fv_node), ptr(d_fv_ptr), ptr(d_fv_feat),
                                                  ptr(d_fv_n), C.c_void_p(int(stream) if stream else 0)), "se2gpu_voc_compute_bow_device")


def median_descriptor(desc, ptr_, device=0):
    """MapPoint::updateMainKFandDescriptor (src/MapPoint.cpp:228-272) for many map points: desc rows ptr[m]..ptr[m+1]) are
    map point m's observation descriptors. Returns (best index within each list, its median distance)."""
    d = np.ascontiguousarray(desc, np.uint8).reshape(-1, 32); p = np.ascontiguousarray(ptr_, np.int32)
    M = len(p) - 1
    idx = np.zeros(M, np.int32); med = np.zeros(M, np.int32)
    check(lib().se2gpu_median_descriptor(ptr(d), ptr(p), M, ptr(idx), ptr(med), device), "se2gpu_median_descriptor")
    return idx, med
