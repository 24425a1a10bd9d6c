"""Host-side mirror of se2lam::ORBmatcher (reference include/se2lam/ORBmatcher.h:40-81) over the C ABI.

The reference's Frame / KeyFrame / MapPoint objects are flattened to arrays (see include/se2gpu.h);
`FrameView` carries what the matcher reads from a Frame: keyPointsUn, descriptors and the grid bounds.
"""
from __future__ import annotations

import ctypes as C
import dataclasses

import numpy as np

from . import _capi
from ._capi import BowBatchKF, BowKF, GridParams, KP_DTYPE, check, lib, ptr

FRAME_GRID_ROWS, FRAME_GRID_COLS = 48, 64   # Frame.h:26-27


@dataclasses.dataclass
class FrameView:
    keyPointsUn: np.ndarray      # KP_DTYPE [N]
    descriptors: np.ndarray      # [N,32] uint8
    minXUn: float = 0.0
    maxXUn: float = 640.0
    minYUn: float = 0.0
    maxYUn: float = 480.0

    @property
    def N(self):
        return len(self.keyPointsUn)

    def grid(self) -> GridParams:   # Frame.cpp:37-40
        f = np.float32
        return GridParams(f(self.minXUn), f(self.minYUn), f(f(FRAME_GRID_COLS) / f(f(self.maxXUn) - f(self.minXUn))),
                          f(f(FRAME_GRID_ROWS) / f(f(self.maxYUn) - f(self.minYUn))))


class ORBmatcher:
    """ORBmatcher(nnratio, checkOri). With `max_queries` / `max_db` it owns a matcher context (se2gpu_matcher_create_batch:
    all device buffers allocated once, for up to `max_batch` frame pairs per batched call) and offers the device-resident
    entry points; without, the per-device default context of the library is used."""
    TH_HIGH, TH_LOW, HISTO_LENGTH = 100, 75, 30   # ORBmatcher.cpp:45-47
    PROFILE_GROUPS = ("k_grid_build", "k_candidates", "k_resolve", "k_fallback")

    def __init__(self, nnratio=0.6, checkOri=True, device=0, max_queries=None, max_db=None, max_batch=1):
        self.mfNNratio, self.mbCheckOrientation, self.device = float(nnratio), bool(checkOri), device
        self.h = None
        if max_queries is not None or max_db is not None:
            self.h = lib().se2gpu_matcher_create_batch(int(max_queries or max_db), int(max_db or max_queries), int(max_batch), device)
            if not self.h:
                raise _capi.Se2GpuError("se2gpu_matcher_create_batch failed: " + _capi.last_error())

    def close(self):
        if getattr(self, "h", None):
            lib().se2gpu_matcher_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:      # interpreter shutdown
            pass

    # ---- device-resident entry points (pointers are CUDA device pointers: ints or torch tensors); asynchronous on `stream`
    def MatchByWindowDevice(self, d_kp1, d_desc1, n1, d_kp2, d_desc2, n2, d_prev, grid: GridParams, winSize, d_matches12,
                            d_nmatches=None, d_n1=None, d_n2=None, levelOffset=1, minLevel=0, maxLevel=8, stream=0):
        assert self.h, "device entry points need an owned context (pass max_queries / max_db)"
        check(lib().se2gpu_match_by_window_device(self.h, ptr(d_kp1), ptr(d_desc1), int(n1), ptr(d_n1), ptr(d_kp2), ptr(d_desc2), int(n2),
                                                  ptr(d_n2), ptr(d_prev), grid, int(winSize), levelOffset, minLevel, maxLevel,
                                                  self.mfNNratio, ptr(d_matches12), ptr(d_nmatches),
                                                  C.c_void_p(int(stream) if stream else 0)), "se2gpu_match_by_window_device")

    @staticmethod
    def KeypointsToPointsDevice(d_kp, n, d_xy, d_n=None, stream=0):
        check(lib().se2gpu_keypoints_to_points_device(ptr(d_kp), int(n), ptr(d_n), ptr(d_xy), C.c_void_p(int(stream) if stream else 0)),
              "se2gpu_keypoints_to_points_device")

    def MatchByProjectionDevice(self, d_kf_kp, d_kf_desc, n_kf, d_kf_observed, d_mp_valid, d_mp_uv, n_mp, d_mp_octave, d_mp_desc,
                                grid: GridParams, winSize, levelOffset, d_matches_idx_mp, d_nmatches=None, d_n_kf=None, stream=0):
        assert self.h, "device entry points need an owned context (pass max_queries / max_db)"
        check(lib().se2gpu_match_by_projection_device(self.h, ptr(d_kf_kp), ptr(d_kf_desc), int(n_kf), ptr(d_n_kf), ptr(d_kf_observed),
                                                      ptr(d_mp_valid), ptr(d_mp_uv), int(n_mp), ptr(d_mp_octave), ptr(d_mp_desc), grid,
                                                      int(winSize), int(levelOffset), self.mfNNratio, ptr(d_matches_idx_mp),
                                                      ptr(d_nmatches), C.c_void_p(int(stream) if stream else 0)),
              "se2gpu_match_by_projection_device")

    # ---- batched device entry points: B frame pairs, pair b at slot b of every array (see include/se2gpu.h)
    def MatchByWindowBatchDevice(self, B, d_kp1, d_desc1, cap1, d_kp2, d_desc2, cap2, d_prev, grid: GridParams, winSize, d_matches12,
                                 d_nmatches=None, d_n1=None, d_n2=None, levelOffset=1, minLevel=0, maxLevel=8, stream=0):
        assert self.h, "device entry points need an owned context (pass max_queries / max_db)"
        check(lib().se2gpu_match_by_window_batch_device(self.h, int(B), ptr(d_kp1), ptr(d_desc1), int(cap1), ptr(d_n1), ptr(d_kp2),
                                                        ptr(d_desc2), int(cap2), ptr(d_n2), ptr(d_prev), grid, int(winSize), levelOffset,
                                                        minLevel, maxLevel, self.mfNNratio, ptr(d_matches12), ptr(d_nmatches),
                                                        C.c_void_p(int(stream) if stream else 0)), "se2gpu_match_by_window_batch_device")

    def MatchByProjectionBatchDevice(self, B, d_kf_kp, d_kf_desc, cap_kf, d_kf_observed, d_mp_valid, d_mp_uv, cap_mp, d_mp_octave,
                                     d_mp_desc, grid: GridParams, winSize, levelOffset, d_matches_idx_mp, d_nmatches=None, d_n_kf=None,
                                     stream=0):
        assert self.h, "device entry points need an owned context (pass max_queries / max_db)"
        check(lib().se2gpu_match_by_projection_batch_device(self.h, int(B), ptr(d_kf_kp), ptr(d_kf_desc), int(cap_kf), ptr(d_n_kf),
                                                            ptr(d_kf_observed), ptr(d_mp_valid), ptr(d_mp_uv), int(cap_mp),
                                                            ptr(d_mp_octave), ptr(d_mp_desc), grid, int(winSize), int(levelOffset),
                                                            self.mfNNratio, ptr(d_matches_idx_mp), ptr(d_nmatches),
                                                            C.c_void_p(int(stream) if stream else 0)),
              "se2gpu_match_by_projection_batch_device")

    @staticmethod
    def BowBatchSide(kp, desc, cap, fv_node, fv_ptr, fv_feat, fv_n, has_mp=None) -> BowBatchKF:
        """One side of SearchByBoWBatchDevice: keyframe k's keypoints, descriptors and has_mp in slot k of `cap`, and its
        FeatureVector as Vocabulary.compute_bow_device writes it (device pointers: ints or torch tensors)."""
        v = lambda a: ptr(a).value if a is not None else None
        return BowBatchKF(v(kp), v(desc), v(has_mp), int(cap), v(fv_node), v(fv_ptr), v(fv_feat), v(fv_n))

    def SearchByBoWBatchDevice(self, B, kf1: BowBatchKF, kf2: BowBatchKF, d_matches12, d_nmatches=None, d_slot2=None, bIfMPOnly=True,
                               stream=0):
        """SearchByBoW for B keyframe pairs: keyframe b of kf1 against keyframe d_slot2[b] of kf2 (None: b). Writes
        d_matches12 + b*kf1.cap (-1 = none) and d_nmatches[b]; asynchronous on `stream` (se2gpu_search_by_bow_batch_device)."""
        assert self.h, "device entry points need an owned context (pass max_queries / max_db)"
        check(lib().se2gpu_search_by_bow_batch_device(self.h, int(B), C.byref(kf1), C.byref(kf2), ptr(d_slot2), int(bIfMPOnly),
                                                      self.mfNNratio, int(self.mbCheckOrientation), ptr(d_matches12), ptr(d_nmatches),
                                                      C.c_void_p(int(stream) if stream else 0)), "se2gpu_search_by_bow_batch_device")

    def profile(self, enable=True):
        check(lib().se2gpu_matcher_profile(self.h, int(enable)), "se2gpu_matcher_profile")

    def profile_read(self):
        ms = np.zeros(len(self.PROFILE_GROUPS)); n = np.zeros(len(self.PROFILE_GROUPS), np.int32)
        check(lib().se2gpu_matcher_profile_read(self.h, ptr(ms), ptr(n)), "se2gpu_matcher_profile_read")
        return {g: (float(ms[i]), int(n[i])) for i, g in enumerate(self.PROFILE_GROUPS)}

    def last_rounds(self):
        r, f = C.c_int(), C.c_int()
        check(lib().se2gpu_matcher_last_rounds(self.h, C.byref(r), C.byref(f)), "se2gpu_matcher_last_rounds")
        return r.value, bool(f.value)

    def last_rounds_batch(self, B):
        """(rounds [B] int32, used_fallback [B] bool) of every pair of the last batched call."""
        r, f = np.zeros(B, np.int32), np.zeros(B, np.int32)
        check(lib().se2gpu_matcher_last_rounds_batch(self.h, int(B), ptr(r), ptr(f)), "se2gpu_matcher_last_rounds_batch")
        return r, f.astype(bool)

    @staticmethod
    def DescriptorDistance(a, b, device=0):
        a = np.ascontiguousarray(a, np.uint8).reshape(-1, 32); b = np.ascontiguousarray(b, np.uint8).reshape(-1, 32)
        out = np.zeros(len(a), np.int32)
        check(lib().se2gpu_hamming_distance(ptr(a), ptr(b), len(a), ptr(out), device), "se2gpu_hamming_distance")
        return int(out[0]) if len(out) == 1 else out

    def MatchByWindow(self, frame1: FrameView, frame2: FrameView, vbPrevMatched, winSize, levelOffset=1, minLevel=0, maxLevel=8):
        """Returns (nmatches, vnMatches12); vbPrevMatched [N1,2] float32 is updated in place."""
        kp1 = np.ascontiguousarray(frame1.keyPointsUn, KP_DTYPE); kp2 = np.ascontiguousarray(frame2.keyPointsUn, KP_DTYPE)
        d1 = np.ascontiguousarray(frame1.descriptors, np.uint8); d2 = np.ascontiguousarray(frame2.descriptors, np.uint8)
        assert vbPrevMatched.dtype == np.float32 and vbPrevMatched.flags.c_contiguous
        m = np.full(len(kp1), -1, np.int32)
        if self.h:
            n = check(lib().se2gpu_matcher_match_by_window(self.h, ptr(kp1), ptr(d1), len(kp1), ptr(kp2), ptr(d2), len(kp2),
                                                           ptr(vbPrevMatched), frame2.grid(), int(winSize), levelOffset, minLevel,
                                                           maxLevel, self.mfNNratio, ptr(m)), "se2gpu_matcher_match_by_window")
        else:
            n = check(lib().se2gpu_match_by_window(ptr(kp1), ptr(d1), len(kp1), ptr(kp2), ptr(d2), len(kp2), ptr(vbPrevMatched),
                                                   frame2.grid(), int(winSize), levelOffset, minLevel, maxLevel, self.mfNNratio,
                                                   ptr(m), self.device), "se2gpu_match_by_window")
        return n, m

    def MatchByProjection(self, kf: FrameView, kf_observed, mp_valid, mp_uv, mp_octave, mp_desc, winSize, levelOffset):
        kp = np.ascontiguousarray(kf.keyPointsUn, KP_DTYPE); d = np.ascontiguousarray(kf.descriptors, np.uint8)
        obs = np.ascontiguousarray(kf_observed, np.uint8); val = np.ascontiguousarray(mp_valid, np.uint8)
        uv = np.ascontiguousarray(mp_uv, np.float32); octv = np.ascontiguousarray(mp_octave, np.int32)
        md = np.ascontiguousarray(mp_desc, np.uint8)
        m = np.full(len(kp), -1, np.int32)
        if self.h:
            n = check(lib().se2gpu_matcher_match_by_projection(self.h, ptr(kp), ptr(d), len(kp), ptr(obs), ptr(val), ptr(uv), len(val),
                                                               ptr(octv), ptr(md), kf.grid(), int(winSize), int(levelOffset),
                                                               self.mfNNratio, ptr(m)), "se2gpu_matcher_match_by_projection")
        else:
            n = check(lib().se2gpu_match_by_projection(ptr(kp), ptr(d), len(kp), ptr(obs), ptr(val), ptr(uv), len(val), ptr(octv),
                                                       ptr(md), kf.grid(), int(winSize), int(levelOffset), self.mfNNratio, ptr(m),
                                                       self.device), "se2gpu_match_by_projection")
        return n, m

    def SearchByBoW(self, kf1: dict, kf2: dict, bIfMPOnly=True):
        """kf = dict(angle, desc, has_mp, node (ascending), ptr, feat). Returns (nmatches, matches12 [-1 = none])."""
        keep = []

        def pack(k):
            a = [np.ascontiguousarray(k["angle"], np.float32), np.ascontiguousarray(k["desc"], np.uint8),
                 np.ascontiguousarray(k["has_mp"], np.uint8), np.ascontiguousarray(k["node"], np.int32),
                 np.ascontiguousarray(k["ptr"], np.int32), np.ascontiguousarray(k["feat"], np.int32)]
            keep.append(a)
            return BowKF(ptr(a[0]).value, ptr(a[1]).value, ptr(a[2]).value, len(a[0]), ptr(a[3]).value, len(a[3]),
                         ptr(a[4]).value, ptr(a[5]).value)
        b1, b2 = pack(kf1), pack(kf2)
        m = np.full(b1.n, -1, np.int32)
        if self.h:
            n = check(lib().se2gpu_matcher_search_by_bow(self.h, C.byref(b1), C.byref(b2), int(bIfMPOnly), self.mfNNratio,
                                                         int(self.mbCheckOrientation), ptr(m)), "se2gpu_matcher_search_by_bow")
        else:
            n = check(lib().se2gpu_search_by_bow(C.byref(b1), C.byref(b2), int(bIfMPOnly), self.mfNNratio, int(self.mbCheckOrientation),
                                                 ptr(m), self.device), "se2gpu_search_by_bow")
        return n, m
