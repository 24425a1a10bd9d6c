"""Host-side mirror of se2lam::ORBextractor (reference include/se2lam/ORBextractor.h:36-84) over the C ABI.

    ext = ORBextractor(nfeatures=1000, scaleFactor=1.2, nlevels=8, scoreType=FAST_SCORE, fastTh=20)
    keypoints, descriptors = ext(image)             # operator()(image, mask, keypoints, descriptors)

`keypoints` is a structured array with cv::KeyPoint's exact 28-byte layout, `descriptors` an [N,32] uint8
array (CV_8U rows).  Batched and device-resident variants are `extract_batch` / `extract_device`.
With scoreType=HARRIS_SCORE each cell's FAST keypoints are ranked by their Harris response, which is also the
keypoints' `response` (reference src/ORBextractor.cpp:85-126, :625-629).
No CPU fallback: without the CUDA library or a GPU the constructor raises.
"""
from __future__ import annotations

import ctypes as C

import numpy as np

from . import _capi
from ._capi import KP_DTYPE, check, lib, ptr

HARRIS_SCORE, FAST_SCORE = 0, 1


class ORBextractor:
    def __init__(self, nfeatures=1000, scaleFactor=1.2, nlevels=8, scoreType=FAST_SCORE, fastTh=20,
                 max_width=640, max_height=480, max_batch=1, device=0):
        self.nfeatures, self.scaleFactor, self.nlevels, self.fastTh = nfeatures, scaleFactor, nlevels, fastTh
        self.scoreType = scoreType
        self.max_batch = max_batch
        self.h = lib().se2gpu_orb_create_scored(nfeatures, scaleFactor, nlevels, scoreType, fastTh, max_width, max_height,
                                                max_batch, device)
        if not self.h:
            raise _capi.Se2GpuError("se2gpu_orb_create_scored failed: " + _capi.last_error())

    def close(self):
        if getattr(self, "h", None):
            lib().se2gpu_orb_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:      # interpreter shutdown: module globals may already be gone
            pass

    def set_undistort(self, K=None, dist=None):
        """Fold cv::undistort(im, img, K, dist) (reference src/Frame.cpp:22) into level 0: subsequent calls take RAW frames.
        K 3x3 float32, dist 0/4/5/8/12 float32 coefficients; K=None switches it off."""
        if K is None:
            check(lib().se2gpu_orb_set_undistort(self.h, None, None, 0), "se2gpu_orb_set_undistort")
            return
        K = np.ascontiguousarray(K, np.float32).reshape(9)
        dist = np.zeros(0, np.float32) if dist is None else np.ascontiguousarray(dist, np.float32).ravel()
        check(lib().se2gpu_orb_set_undistort(self.h, ptr(K), ptr(dist) if dist.size else None, int(dist.size)), "se2gpu_orb_set_undistort")

    def GetLevels(self):
        return self.nlevels

    def GetScaleFactor(self):
        return self.scaleFactor

    def __call__(self, image, mask=None):
        """operator()(image, mask, keypoints, descriptors); mask must be empty (Frame.cpp:25 passes cv::Mat())."""
        if mask is not None and np.size(mask):
            raise _capi.Se2GpuError("masks are not supported (the reference never passes one)")
        image = np.asarray(image)
        if image.size == 0:
            return np.zeros(0, KP_DTYPE), np.zeros((0, 32), np.uint8)
        assert image.dtype == np.uint8 and image.ndim == 2, "image.type() == CV_8UC1"
        kps, desc, counts = self.extract_batch(image[None])
        return kps[0, :counts[0]].copy(), desc[0, :counts[0]].copy()

    def extract_batch(self, images: np.ndarray):
        """images [n,h,w] uint8 (host). Returns (kps [n,nfeatures], desc [n,nfeatures,32], counts [n])."""
        images = np.ascontiguousarray(images, np.uint8)
        n, h, w = images.shape
        kps = np.zeros((n, self.nfeatures), KP_DTYPE)
        desc = np.zeros((n, self.nfeatures, 32), np.uint8)
        counts = np.zeros(n, np.int32)
        check(lib().se2gpu_orb_extract(self.h, ptr(images), n, w, h, images.strides[1], images.strides[0], ptr(kps), ptr(desc),
                                       ptr(counts)), "se2gpu_orb_extract")
        return kps, desc, counts

    def submit(self, images: np.ndarray, kps: np.ndarray, desc: np.ndarray, counts: np.ndarray):
        """Asynchronous extract_batch into caller-owned buffers (se2gpu_orb_submit); at most two batches in flight."""
        n, h, w = images.shape
        check(lib().se2gpu_orb_submit(self.h, ptr(images), n, w, h, images.strides[1], images.strides[0], ptr(kps), ptr(desc), ptr(counts)),
              "se2gpu_orb_submit")

    def wait(self):
        """Blocks until the oldest submitted batch is complete (se2gpu_orb_wait)."""
        check(lib().se2gpu_orb_wait(self.h), "se2gpu_orb_wait")

    def extract_device(self, d_images, n, h, w, d_kps, d_desc, d_counts, stream=0, stride=None, frame_stride=None):
        """Device-resident variant: all pointers are CUDA device pointers (ints or torch tensors); asynchronous."""
        stride = w if stride is None else stride
        frame_stride = h * stride if frame_stride is None else frame_stride
        check(lib().se2gpu_orb_extract_device(self.h, ptr(d_images), n, w, h, stride, frame_stride, ptr(d_kps), ptr(d_desc),
                                              ptr(d_counts), C.c_void_p(int(stream) if stream else 0)), "se2gpu_orb_extract_device")

    def level(self, frame, level, blurred=False):
        w, h, p = C.c_int(), C.c_int(), C.c_int()
        check(lib().se2gpu_orb_level_dims(self.h, level, C.byref(w), C.byref(h), C.byref(p)), "se2gpu_orb_level_dims")
        out = np.zeros((h.value + 32, p.value), np.uint8)
        check(lib().se2gpu_orb_get_level(self.h, frame, level, int(blurred), ptr(out)), "se2gpu_orb_get_level")
        return out, w.value, h.value

    PROFILE_GROUPS = ("pyramid", "orb_fast_cells", "orb_select", "orb_blur", "orb_orient_describe")

    def profile(self, enable=True):
        check(lib().se2gpu_orb_profile(self.h, int(enable)), "se2gpu_orb_profile")

    def profile_read(self):
        ms = np.zeros(len(self.PROFILE_GROUPS)); n = np.zeros(len(self.PROFILE_GROUPS), np.int32)
        check(lib().se2gpu_orb_profile_read(self.h, ptr(ms), ptr(n)), "se2gpu_orb_profile_read")
        return {g: (float(ms[i]), int(n[i])) for i, g in enumerate(self.PROFILE_GROUPS)}
