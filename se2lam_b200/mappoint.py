"""Map-point updates (reference src/MapPoint.cpp) over the C ABI: MapPoint::addObservation, eraseObservation and
updateMeasureInKFs for many map points in one call, on the object graph flattened into arrays (include/se2gpu.h,
se2gpu_mp_*; DESIGN.md section 13).

The keyframe table `kf` and the point table `mp` are dicts of arrays:
    kf: kf_id [K] i4, kf_null [K] u1, Tcw [K,4,4] f4, kp_base [K] i4, kp [S] KP_DTYPE, desc [S,32] u1,
        view_mp [S,3] f4, view_info [S,3,3] f8
    mp: pos [M,3] f4, good_prl [M] u1, null [M] u1, main_kf [M] i4, main_desc [M,32] u1, main_octave [M] i4,
        main_measure [M,2] f4, level_scale [M] f4, normal [M,3] f4, min_dist [M] f4, max_dist [M] f4,
        obs_ptr [M+1] i4, obs_kf [n_obs] i4, obs_idx [n_obs] i4
`MapPoints` takes host (numpy) arrays and updates them in place; `keyframes`, `points` and `params` build the structs the
`_device` entry points take from device arrays (torch CUDA tensors) just as well.
"""
from __future__ import annotations

from ctypes import byref

import numpy as np

from ._capi import KP_DTYPE, MP_MAX_LEVELS, MpKeyframes, MpParams, MpPoints, check, lib, ptr

KF_FIELDS = {"kf_id": np.int32, "kf_null": np.uint8, "Tcw": np.float32, "kp_base": np.int32, "kp": KP_DTYPE,
             "desc": np.uint8, "view_mp": np.float32, "view_info": np.float64}
MP_FIELDS = {"pos": np.float32, "good_prl": np.uint8, "null": np.uint8, "main_kf": np.int32, "main_desc": np.uint8,
             "main_octave": np.int32, "main_measure": np.float32, "level_scale": np.float32, "normal": np.float32,
             "min_dist": np.float32, "max_dist": np.float32, "obs_ptr": np.int32, "obs_kf": np.int32, "obs_idx": np.int32}


def _rows(a):
    return int(a.shape[0])


def keyframes(kf) -> MpKeyframes:
    """se2gpu_mp_keyframes over the arrays of `kf` (host or device)"""
    return MpKeyframes(_rows(kf["kf_id"]), ptr(kf["kf_id"]), ptr(kf["kf_null"]), ptr(kf["Tcw"]), ptr(kf["kp_base"]),
                       _rows(kf["view_mp"]), ptr(kf["kp"]), ptr(kf["desc"]), ptr(kf["view_mp"]), ptr(kf["view_info"]))


def points(mp) -> MpPoints:
    """se2gpu_mp_points over the arrays of `mp` (host or device)"""
    return MpPoints(_rows(mp["obs_ptr"]) - 1, *[ptr(mp[k]) for k in list(MP_FIELDS)])


def params(K, lower_depth, upper_depth, fx, scale_factors) -> MpParams:
    """se2gpu_mp_params: Config::Kcam, LOWER/UPPER_DEPTH, fxCam and mvScaleFactors"""
    sf = np.asarray(scale_factors, np.float32).ravel()
    if not 1 <= len(sf) <= MP_MAX_LEVELS:
        raise ValueError(f"1 to {MP_MAX_LEVELS} scale factors")
    p = MpParams()
    p.K[:] = [float(v) for v in np.asarray(K, np.float32).ravel()]
    p.lower_depth, p.upper_depth, p.fx, p.nlevels = float(lower_depth), float(upper_depth), float(fx), len(sf)
    p.scale_factors[:len(sf)] = [float(v) for v in sf]
    return p


def _host(table, fields):
    for k, dt in fields.items():
        a = table[k]
        if not isinstance(a, np.ndarray) or a.dtype != np.dtype(dt) or not a.flags.c_contiguous:
            raise TypeError(f"{k} must be a C-contiguous {np.dtype(dt)} numpy array")


class MapPoints:
    """The map points of the tables `kf` and `mp` (host arrays, updated in place by every call)."""

    def __init__(self, kf, mp, K, lower_depth, upper_depth, fx, scale_factors, device=0):
        _host(kf, KF_FIELDS)
        _host(mp, MP_FIELDS)
        self.kf, self.mp, self.device = kf, mp, device
        self.params = params(K, lower_depth, upper_depth, fx, scale_factors)

    def _updates(self, fn, upd_ptr, upd_pos, name):
        upd_ptr = np.ascontiguousarray(upd_ptr, np.int32)
        upd_pos = np.ascontiguousarray(upd_pos, np.int32)
        k, p = keyframes(self.kf), points(self.mp)
        abandoned = np.zeros(p.n_mp, np.uint8)
        check(fn(byref(k), byref(p), ptr(upd_ptr), ptr(upd_pos), byref(self.params), ptr(abandoned), self.device), name)
        return abandoned.astype(bool)

    def addObservation(self, upd_ptr, upd_pos):
        """MapPoint::addObservation: point m inserts the list positions upd_pos[upd_ptr[m]:upd_ptr[m+1]], in order (its
        list in `mp` is the list after them). Returns the points updateParallax abandoned."""
        return self._updates(lib().se2gpu_mp_add_observations, upd_ptr, upd_pos, "se2gpu_mp_add_observations")

    def eraseObservation(self, upd_ptr, upd_pos):
        """MapPoint::eraseObservation of the list positions upd_pos[upd_ptr[m]:upd_ptr[m+1]] (its list in `mp` is the list
        before them). Returns the points left with no observation and set null."""
        return self._updates(lib().se2gpu_mp_erase_observations, upd_ptr, upd_pos, "se2gpu_mp_erase_observations")

    def updateMeasureInKFs(self, pts):
        """MapPoint::updateMeasureInKFs of the points `pts`"""
        pts = np.ascontiguousarray(pts, np.int32)
        k, p = keyframes(self.kf), points(self.mp)
        check(lib().se2gpu_mp_update_measure(byref(k), byref(p), len(pts), ptr(pts), self.device), "se2gpu_mp_update_measure")
