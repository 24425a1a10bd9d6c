"""Localizer::run over the C ABI (include/se2gpu.h, se2gpu_loc_*; DESIGN.md section 15): a localization handle for B
camera streams against one static map uploaded once. One `step` takes one frame and one odometry reading per stream and
returns one record per stream; `relocalize` runs the verified loop-closure branch for streams the caller matched to a
map keyframe.

The map is a dict of numpy arrays (K keyframes, M map points):
    kf_Tcw [K,4,4] f4, kf_kp_ptr [K+1] i4, kf_obs_mp [kf_kp_ptr[K]] i4 (map point per keypoint slot, -1 for none),
    kf_obs_ptr [K+1] / kf_obs i4 (mObservations, ascending), kf_cov_ptr [K+1] / kf_cov i4 (covisible keyframes, ascending),
    mp_pos [M,3] f4, mp_null [M] u1, mp_good_prl [M] u1, mp_desc [M,32] u1, mp_octave [M] i4
"""
from __future__ import annotations

from ctypes import byref

import numpy as np

from ._capi import (KP_DTYPE, LOC_RESULT_FIELDS, GridParams, LocMap, LocParams, LocResult, LocStreamState, PoseBAParams, check,
                    lib, ptr)
from .track import _to_host, frame_layout

RESULT_DTYPE = np.dtype([(n, np.int32) for n in LOC_RESULT_FIELDS] + [("Tcw", np.float32, (4, 4))])
MAP_FIELDS = {"kf_Tcw": np.float32, "kf_kp_ptr": np.int32, "kf_obs_mp": np.int32, "kf_obs_ptr": np.int32, "kf_obs": np.int32,
              "kf_cov_ptr": np.int32, "kf_cov": np.int32, "mp_pos": np.float32, "mp_null": np.uint8, "mp_good_prl": np.uint8,
              "mp_desc": np.uint8, "mp_octave": np.int32}


def params(nfeatures, scale_factor, nlevels, K, grid, bounds, cTb, bTc, huber_delta, max_local_mps, fast_th=20, dist=(),
           xrot_info=1e6, yrot_info=1e6, z_info=1.0, iterations=30) -> LocParams:
    """se2gpu_loc_params from the reference's Config values: grid = (minX, minY, invW, invH), bounds = (minXUn, maxXUn,
    minYUn, maxYUn); mvInvLevelSigma2 follows from scale_factor as the extractor computes it"""
    p = LocParams()
    p.nfeatures, p.scale_factor, p.nlevels, p.fast_th = int(nfeatures), float(scale_factor), int(nlevels), int(fast_th)
    Kf = np.asarray(K, np.float32)
    p.K[:] = [float(v) for v in Kf.ravel()]
    d = [float(v) for v in np.asarray(dist, np.float32).ravel()]
    p.ndist = len(d)
    p.dist[:len(d)] = d
    p.grid = GridParams(*[float(v) for v in grid])
    p.min_x, p.max_x, p.min_y, p.max_y = (float(v) for v in bounds)
    p.cTb[:] = [float(v) for v in np.asarray(cTb, np.float32).ravel()]
    p.bTc[:] = [float(v) for v in np.asarray(bTc, np.float32).ravel()]
    ba = PoseBAParams()
    ba.fx, ba.cx, ba.cy = float(Kf[0, 0]), float(Kf[0, 2]), float(Kf[1, 2])
    ba.Tbc[:] = list(p.bTc)
    ba.huber_delta, ba.xrot_info, ba.yrot_info, ba.z_info, ba.iterations = float(huber_delta), xrot_info, yrot_info, z_info, iterations
    p.ba = ba
    p.inv_level_sigma2[:nlevels] = [float(v) for v in inv_level_sigma2(scale_factor, nlevels)]
    p.max_local_mps = int(max_local_mps)
    return p


def inv_level_sigma2(scale_factor, nlevels):
    """ORBextractor's mvInvLevelSigma2: 1 / (scale^l)^2 in float, the scale factors multiplied up in float"""
    s = [np.float32(1.0)]
    for _ in range(1, nlevels):
        s.append(np.float32(s[-1] * np.float32(scale_factor)))
    return np.array([np.float32(1.0) / np.float32(v * v) for v in s], np.float32)


def _map(m):
    arrs = {k: np.ascontiguousarray(m[k], t) for k, t in MAP_FIELDS.items()}
    c = LocMap()
    c.n_kf, c.n_mp = len(arrs["kf_kp_ptr"]) - 1, len(arrs["mp_null"])
    for k, a in arrs.items():
        setattr(c, k, ptr(a) if a.size else None)
    return c, arrs


def _results(out, n):
    r = np.zeros(n, RESULT_DTYPE)
    for b in range(n):
        for f in LOC_RESULT_FIELDS:
            r[b][f] = getattr(out[b], f)
        r[b]["Tcw"] = np.array(out[b].Tcw, np.float32).reshape(4, 4)
    return r


class Localizer:
    def __init__(self, max_streams, max_w, max_h, p: LocParams, map_, device=0):
        self.p, self.cap, self.S = p, p.nfeatures, max_streams
        self.n_kf = len(map_["kf_kp_ptr"]) - 1
        cm, keep = _map(map_)
        self.h = lib().se2gpu_loc_create(max_streams, max_w, max_h, byref(p), byref(cm), device)
        del keep
        if not self.h:
            check(-1, "se2gpu_loc_create")

    def close(self):
        if getattr(self, "h", None):
            lib().se2gpu_loc_destroy(self.h)
            self.h = None

    __del__ = close

    def step(self, frames, odom):
        """one frame per stream 0 .. B-1, the other streams left as they are: frames [B, h, w] (numpy or a CUDA tensor,
        read in place with its own strides when they allow it: se2lam_b200.track.frame_layout), odom [B, 3]"""
        frames, on_dev, B, hgt, w, stride, fstride = frame_layout(frames)
        odom = np.ascontiguousarray(odom, np.float32).reshape(B, 3)
        out = (LocResult * B)()
        check(lib().se2gpu_loc_step(self.h, B, ptr(frames), on_dev, w, hgt, stride, fstride, ptr(odom), out), "se2gpu_loc_step")
        return _results(out, B)

    def relocalize(self, streams, kf_loop, matches):
        """matches[j]: (idxCurr, idxLoop) pairs of stream streams[j] (the caller's verified mapMatchGood); returns (records,
        Tcw after the first BA [n, 4, 4])"""
        n = len(streams)
        s = np.ascontiguousarray(streams, np.int32)
        k = np.ascontiguousarray(kf_loop, np.int32)
        mp = np.zeros(n + 1, np.int32)
        for j, m in enumerate(matches):
            mp[j + 1] = mp[j] + len(m)
        pairs = np.concatenate([np.asarray(m, np.int32).reshape(-1, 2) for m in matches]) if n else np.zeros((0, 2), np.int32)
        cur, loop = np.ascontiguousarray(pairs[:, 0]), np.ascontiguousarray(pairs[:, 1])
        out = (LocResult * max(n, 1))()
        first = np.zeros((max(n, 1), 4, 4), np.float32)
        check(lib().se2gpu_loc_relocalize(self.h, n, ptr(s), ptr(k), ptr(mp), ptr(cur), ptr(loop), out, ptr(first)),
              "se2gpu_loc_relocalize")
        return _results(out, n), first[:n]

    def state(self, b):
        """stream b's state copied to the host: kp / desc (count entries), obs_mp [n], local_mps (count entries, at most
        max_local_mps), local_kfs / covis_kfs [K] u1, Tcw [4,4], flags"""
        st = LocStreamState()
        check(lib().se2gpu_loc_state(self.h, b, byref(st)), "se2gpu_loc_state")
        n = int(_to_host(st.d_n, (1,), "<i4")[0])
        nl = min(int(_to_host(st.d_n_local_mps, (1,), "<i4")[0]), self.p.max_local_mps)
        K = max(self.n_kf, 0)
        return {
            "kp": _to_host(st.d_kp, (n * KP_DTYPE.itemsize,), "|u1").view(KP_DTYPE), "desc": _to_host(st.d_desc, (n, 32), "|u1"),
            "obs_mp": _to_host(st.d_obs_mp, (n,), "<i4"), "local_mps": _to_host(st.d_local_mps, (nl,), "<i4"),
            "local_kfs": _to_host(st.d_local_kfs, (K,), "|u1"), "covis_kfs": _to_host(st.d_covis_kfs, (K,), "|u1"),
            "Tcw": np.array(st.Tcw, np.float32).reshape(4, 4), "has_frame": bool(st.has_frame), "tracked": bool(st.tracked),
            "overflow": bool(st.overflow),
        }

    def graph_nodes(self):
        import ctypes as C
        k, n = C.c_int(), C.c_int()
        check(lib().se2gpu_loc_graph_nodes(self.h, byref(k), byref(n)), "se2gpu_loc_graph_nodes")
        return k.value, n.value

    def set_eager(self, eager: bool):
        """test hook: direct launches instead of the captured graph"""
        check(lib().se2gpu_loc_debug_eager(self.h, int(eager)), "se2gpu_loc_debug_eager")


def host_pose(p: LocParams, odom, ref_odom, ref_Tcw):
    """UpdatePoseCurr's Tcw [4,4] for odometry odom after ref_odom, from the previous pose ref_Tcw"""
    f = lambda a: np.ascontiguousarray(a, np.float32)
    T = np.zeros(16, np.float32)
    check(lib().se2gpu_loc_host_pose(byref(p), ptr(f(odom)), ptr(f(ref_odom)), ptr(f(ref_Tcw)), ptr(T)), "se2gpu_loc_host_pose")
    return T.reshape(4, 4)
