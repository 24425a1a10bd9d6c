"""Track::mTrack over the C ABI (include/se2gpu.h, se2gpu_tracker_*; DESIGN.md section 14): a tracker handle for B
independent camera streams whose tracking state (reference frame, mPrevMatched, mMatchIdx, mLocalMPs, mvbGoodPrl) stays
on the device between frames. One `step` takes one frame and one odometry reading per stream and returns the per-stream
record (counts and the two needNewKF flags); the caller makes the keyframes and calls `reset` for those streams.

Frames are uint8 arrays [B, h, w]: numpy (host) or torch CUDA tensors (device), read in place with their own row and
frame strides when the last axis has unit stride (frame_layout), packed into a copy otherwise. The keyframe side of stream b is a dict
    observed: device uint8 [nfeatures] (mpKF->hasObservation), view_mp: device float32 [nfeatures, 3] (mpKF->mViewMPs),
    n_obs_mp: int (getSizeObsMP), accept: bool (acceptNewKF), odom: (x, y, theta) (mpKF->odom)
"""
from __future__ import annotations

from ctypes import byref

import numpy as np

from ._capi import (KP_DTYPE, TRACK_RESULT_FIELDS, GridParams, TrackerParams, TrackKF, TrackResult, TrackState, check, lib,
                    ptr)

RESULT_DTYPE = np.dtype([(n, np.int32) for n in TRACK_RESULT_FIELDS])


def params(nfeatures, scale_factor, nlevels, K, grid, lower_depth, upper_depth, cTb, bTc, odo_noise, max_frames,
           min_frames=8, fast_th=20, dist=()) -> TrackerParams:
    """se2gpu_tracker_params from the reference's Config values (grid = (minX, minY, invW, invH))"""
    p = TrackerParams()
    p.nfeatures, p.scale_factor, p.nlevels, p.fast_th = int(nfeatures), float(scale_factor), int(nlevels), int(fast_th)
    p.K[:] = [float(v) for v in np.asarray(K, np.float32).ravel()]
    d = [float(v) for v in np.asarray(dist, np.float32).ravel()]
    p.ndist = len(d)
    p.dist[:len(d)] = d
    p.grid = GridParams(*[float(v) for v in grid])
    p.lower_depth, p.upper_depth = float(lower_depth), float(upper_depth)
    p.cTb[:] = [float(v) for v in np.asarray(cTb, np.float32).ravel()]
    p.bTc[:] = [float(v) for v in np.asarray(bTc, np.float32).ravel()]
    p.odo_noise[:] = [float(v) for v in odo_noise]
    p.min_frames, p.max_frames = int(min_frames), int(max_frames)
    return p


class _DevArray:
    """a view of device memory torch can adopt (__cuda_array_interface__)"""
    def __init__(self, addr, shape, typestr):
        self.__cuda_array_interface__ = {"shape": tuple(shape), "typestr": typestr, "data": (int(addr), False), "version": 2}


def _to_host(addr, shape, typestr):
    import torch
    if int(np.prod(shape)) == 0:
        return np.zeros(shape, np.dtype(typestr))
    return torch.as_tensor(_DevArray(addr, shape, typestr), device="cuda").cpu().numpy()


def _results(out, B):
    return np.frombuffer(bytes(out), RESULT_DTYPE, count=B).copy()


def frame_layout(frames):
    """(frames, on_device, B, h, w, stride, frame_stride) for a batch of frames [B, h, w]: a numpy array (host) or a torch
    CUDA tensor (device). A uint8 array whose last axis has unit stride, whose rows do not overlap and whose frames do not
    overlap (B = 1: any frame stride) is passed as it is, with its own row stride and frame stride in bytes, so a view
    such as big[:, y0:y0 + h, x0:x0 + w] is read where it lies. Any other array is first made a packed uint8 copy (a
    torch CPU tensor becomes a numpy array)."""
    if hasattr(frames, "data_ptr") and not frames.is_cuda:
        frames = frames.numpy()
    on_dev = hasattr(frames, "data_ptr")
    if on_dev:
        import torch
        ok = frames.dtype == torch.uint8 and frames.dim() == 3
        strides = frames.stride() if ok else ()
    else:
        frames = np.asarray(frames)
        ok = frames.dtype == np.uint8 and frames.ndim == 3
        strides = frames.strides if ok else ()
    if ok:
        B, hgt, w = frames.shape
        fs, rs, cs = strides
        ok = cs == 1 and rs >= w and (B == 1 or fs >= rs * (hgt - 1) + w) and fs >= 0
    if not ok:
        if on_dev:
            import torch
            frames = frames.to(torch.uint8).contiguous()
        else:
            frames = np.ascontiguousarray(frames, np.uint8)
        B, hgt, w = frames.shape
        fs, rs = w * hgt, w
    return frames, int(on_dev), B, hgt, w, int(rs), int(fs)


class Tracker:
    def __init__(self, max_streams, max_w, max_h, p: TrackerParams, device=0):
        self.p, self.cap, self.S = p, p.nfeatures, max_streams
        self.h = lib().se2gpu_tracker_create(max_streams, max_w, max_h, byref(p), device)
        if not self.h:
            check(-1, "se2gpu_tracker_create")

    def close(self):
        if getattr(self, "h", None):
            lib().se2gpu_tracker_destroy(self.h)
            self.h = None

    __del__ = close

    def first(self, frames, odom):
        """mCreateFrame for streams 0 .. B-1 (their reference frames dropped, frame ids restarted); frames as for
        frame_layout. The other streams are left as they are."""
        frames, on_dev, B, hgt, w, stride, fstride = frame_layout(frames)
        odom = np.ascontiguousarray(odom, np.float32).reshape(B, 3)
        out = (TrackResult * B)()
        check(lib().se2gpu_tracker_first(self.h, B, ptr(frames), on_dev, w, hgt, stride, fstride, ptr(odom), out),
              "se2gpu_tracker_first")
        return _results(out, B)

    def step(self, frames, odom, kf=None):
        """one frame per stream 0 .. B-1 (frames as for frame_layout; the other streams are left as they are); kf: one
        dict per stream (None for streams without a reference frame)"""
        frames, on_dev, B, hgt, w, stride, fstride = frame_layout(frames)
        odom = np.ascontiguousarray(odom, np.float32).reshape(B, 3)
        kfs = None
        if kf is not None:
            kfs = (TrackKF * B)()
            for b, k in enumerate(kf):
                if k is None:
                    continue
                kfs[b].d_observed, kfs[b].d_view_mp = ptr(k["observed"]), ptr(k["view_mp"])
                kfs[b].n_obs_mp, kfs[b].accept_new_kf = int(k["n_obs_mp"]), int(bool(k["accept"]))
                kfs[b].odom[:] = [float(v) for v in k["odom"]]
        out = (TrackResult * B)()
        check(lib().se2gpu_tracker_step(self.h, B, ptr(frames), on_dev, w, hgt, stride, fstride, ptr(odom), kfs, out),
              "se2gpu_tracker_step")
        return _results(out, B)

    def reset(self, streams, view_mps):
        """resetLocalTrack for `streams`, view_mps[j] a device float32 [nfeatures, 3] (the keyframe's mViewMPs)"""
        import ctypes as C
        n = len(streams)
        s = np.ascontiguousarray(streams, np.int32)
        v = (C.c_void_p * max(n, 1))(*[ptr(a).value for a in view_mps])
        check(lib().se2gpu_tracker_reset(self.h, n, ptr(s), v), "se2gpu_tracker_reset")

    def state(self, b):
        """stream b's state copied to the host: ref / cur keypoints and descriptors (count entries), prev [cap,2],
        matches [n_ref], local_mps [cap,3], good_prl [cap], Tcr [4,4], pre_meas [3], pre_cov [3,3] (column-major), ids"""
        st = TrackState()
        check(lib().se2gpu_tracker_state(self.h, b, byref(st)), "se2gpu_tracker_state")
        C_ = self.cap
        n_ref = int(_to_host(st.d_ref_n, (1,), "<i4")[0])
        n_cur = int(_to_host(st.d_cur_n, (1,), "<i4")[0])
        kp = lambda a, n: _to_host(a, (n * KP_DTYPE.itemsize,), "|u1").view(KP_DTYPE)
        return {
            "ref_kp": kp(st.d_ref_kp, n_ref), "ref_desc": _to_host(st.d_ref_desc, (n_ref, 32), "|u1"),
            "cur_kp": kp(st.d_cur_kp, n_cur), "cur_desc": _to_host(st.d_cur_desc, (n_cur, 32), "|u1"),
            "prev": _to_host(st.d_prev, (C_, 2), "<f4"), "matches": _to_host(st.d_matches, (n_ref,), "<i4"),
            "local_mps": _to_host(st.d_local_mps, (C_, 3), "<f4"), "good_prl": _to_host(st.d_good_prl, (C_,), "|u1"),
            "Tcr": np.array(st.Tcr, np.float32).reshape(4, 4), "pre_meas": np.array(st.pre_meas),
            "pre_cov": np.array(st.pre_cov).reshape(3, 3, order="F"), "frame_id": st.frame_id, "kf_id": st.kf_id,
            "has_ref": bool(st.has_ref), "n_good_prl": st.n_good_prl,
        }

    def graph_nodes(self):
        import ctypes as C
        k, n = C.c_int(), C.c_int()
        check(lib().se2gpu_tracker_graph_nodes(self.h, byref(k), byref(n)), "se2gpu_tracker_graph_nodes")
        return k.value, n.value

    def set_eager(self, eager: bool):
        """test hook: direct launches instead of the captured graph"""
        check(lib().se2gpu_tracker_debug_eager(self.h, int(eager)), "se2gpu_tracker_debug_eager")


def host_pose(p: TrackerParams, odom, kf_odom, last_odom, meas, cov):
    """updateFramePose's Tcr [4,4] and the pre-integration: returns (Tcr, meas, cov) with cov [9] column-major"""
    f = lambda a: np.ascontiguousarray(a, np.float32)
    Tcr = np.zeros(16, np.float32)
    meas = np.array(meas, np.float64); cov = np.array(cov, np.float64).ravel().copy()
    check(lib().se2gpu_track_host_pose(byref(p), ptr(f(odom)), ptr(f(kf_odom)), ptr(f(last_odom)), ptr(Tcr), ptr(meas), ptr(cov)),
          "se2gpu_track_host_pose")
    return Tcr.reshape(4, 4), meas, cov


def host_decide(p: TrackerParams, dframes, n_tracked_old, n_obs_mp, n_good_prl, n_inlier, odom, kf_odom, accept):
    """needNewKF: (new_kf, abort_ba)"""
    import ctypes as C
    f = lambda a: np.ascontiguousarray(a, np.float32)
    nk, ab = C.c_int(), C.c_int()
    check(lib().se2gpu_track_host_decide(byref(p), int(dframes), int(n_tracked_old), int(n_obs_mp), int(n_good_prl), int(n_inlier),
                                         ptr(f(odom)), ptr(f(kf_odom)), int(bool(accept)), byref(nk), byref(ab)),
          "se2gpu_track_host_decide")
    return bool(nk.value), bool(ab.value)
