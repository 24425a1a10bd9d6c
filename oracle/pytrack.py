"""CPU restatement of Track (reference src/Track.cpp) — TEST INFRASTRUCTURE ONLY.

`pose` / `decide` bind oracle/libtrack_oracle.so (updateFramePose with the pre-integration, needNewKF). `TrackOracle` composes
them with the ORB, undistortion, MatchByWindow, removeOutliers and doTriangulate oracles into one camera stream's
mCreateFrame / mTrack / resetLocalTrack, with the same per-step record and state as se2lam_b200.track.Tracker.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

from oracle import pyfundam, pygeom, pyoracle

HERE = os.path.dirname(os.path.abspath(__file__))
_lib = None


def make() -> str:
    """Bring oracle/libtrack_oracle.so up to date with oracle/track.mk and return its path."""
    env = {k: v for k, v in os.environ.items() if k not in ("CXX", "CXXFLAGS")}
    subprocess.run(["make", "-C", HERE, "-s", "-f", "track.mk", "CXX=g++"], check=True, env=env)
    return os.path.join(HERE, "libtrack_oracle.so")


def lib():
    global _lib
    if _lib is None:
        L = C.CDLL(make())
        vp, i, f = C.c_void_p, C.c_int, C.c_float
        L.track_oracle_pose.argtypes = [vp] * 9
        L.track_oracle_pose.restype = None
        L.track_oracle_decide.argtypes = [vp, vp, f, i, i, i, i, i, i, i, i, vp, vp, i, vp]
        L.track_oracle_decide.restype = i
        for n in ("track_oracle_cosf", "track_oracle_sinf"):
            getattr(L, n).argtypes = [f]
            getattr(L, n).restype = f
        _lib = L
    return _lib


def _f(a):
    return np.ascontiguousarray(a, np.float32)


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def pose(cfg, odom, kf_odom, last_odom, meas, cov):
    """(Tcr [4,4] f4, meas [3], cov [9] column-major)"""
    Tcr = np.zeros(16, np.float32)
    meas = np.array(meas, np.float64); cov = np.array(cov, np.float64).ravel().copy()
    cTb, bTc, nz = _f(cfg["cTb"]), _f(cfg["bTc"]), _f(cfg["odo_noise"])
    o, k, l = _f(odom), _f(kf_odom), _f(last_odom)
    lib().track_oracle_pose(_p(cTb), _p(bTc), _p(nz), _p(o), _p(k), _p(l), _p(Tcr), _p(meas), _p(cov))
    return Tcr.reshape(4, 4), meas, cov


def decide(cfg, dframes, n_tracked_old, n_obs_mp, n_good_prl, n_inlier, odom, kf_odom, accept):
    """needNewKF: (new_kf, abort_ba)"""
    ab = C.c_int(0)
    cTb, bTc, o, k = _f(cfg["cTb"]), _f(cfg["bTc"]), _f(odom), _f(kf_odom)
    r = lib().track_oracle_decide(_p(cTb), _p(bTc), float(cfg["upper_depth"]), int(cfg["nfeatures"]), int(cfg["min_frames"]),
                                  int(cfg["max_frames"]), int(dframes), int(n_tracked_old), int(n_obs_mp), int(n_good_prl),
                                  int(n_inlier), _p(o), _p(k), int(bool(accept)), C.byref(ab))
    return bool(r), bool(ab.value)


class TrackOracle:
    """One camera stream of Track. cfg: nfeatures, scale_factor, nlevels, fast_th, K [3,3], dist, grid, lower_depth,
    upper_depth, cTb, bTc, odo_noise, min_frames, max_frames."""

    def __init__(self, cfg):
        self.cfg, self.cap = cfg, int(cfg["nfeatures"])
        self.orb = pyoracle.OrbOracle(cfg["nfeatures"], cfg["scale_factor"], cfg["nlevels"], cfg["fast_th"])
        self.next_id, self.frame_id, self.kf_id, self.has_ref = 0, -1, 0, False
        self.last_odom = np.zeros(3, np.float32)
        self.meas, self.cov, self.n_good_prl = np.zeros(3), np.zeros(9), 0
        self.Tcr = np.eye(4, dtype=np.float32)
        self.ref_kp = self.cur_kp = np.zeros(0, pyoracle.KP_DTYPE)
        self.ref_desc = self.cur_desc = np.zeros((0, 32), np.uint8)
        self.prev = np.zeros((self.cap, 2), np.float32)
        self.matches = np.full(self.cap, -1, np.int32)
        self.local = np.full((self.cap, 3), -1, np.float32)
        self.good = np.zeros(self.cap, np.uint8)

    def _extract(self, img):
        return self.orb.extract(pyoracle.frame_image(img, self.cfg["K"], self.cfg.get("dist", ())))

    def first(self, img, odom):
        self.has_ref, self.next_id = False, 0
        return self.step(img, odom, None)

    def step(self, img, odom, kf):
        """kf: dict(observed [cap] u1, view_mp [cap,3] f4, n_obs_mp, accept, odom) or None; returns the record dict"""
        cfg = self.cfg
        odom = _f(odom)
        fid = self.next_id
        self.next_id += 1
        self.frame_id = fid
        self.cur_kp, self.cur_desc = self._extract(img)
        r = dict(frame_id=fid, first=0, n_keypoints=len(self.cur_kp), n_matched=0, n_inlier=0, n_tracked_old=0, n_good_prl=0,
                 triangulated=0, new_kf=0, abort_ba=0)
        if not self.has_ref:                                   # mCreateFrame
            r["first"] = 1
            r["new_kf"] = int(len(self.cur_kp) > 100)
            if not r["new_kf"]:
                self.next_id = 0
            self.last_odom = odom
            return r
        n = len(self.ref_kp)
        nm, m, prev = pyoracle.match_by_window(self.ref_kp, self.ref_desc, self.cur_kp, self.cur_desc, self.prev[:n], cfg["grid"],
                                               20, 1, 0, 8, 0.9)
        self.prev[:n] = prev
        nin, m, _, _ = pyfundam.remove_outliers(self.ref_kp, self.cur_kp, m)
        self.Tcr, self.meas, self.cov = pose(cfg, odom, kf["odom"], self.last_odom, self.meas, self.cov)
        gate = not (fid - self.kf_id < cfg["min_frames"])
        nto = 0
        if gate:
            m, lm, good, (nto, ngp) = pygeom.track_triangulate(self.ref_kp, self.cur_kp, m, kf["observed"][:n], kf["view_mp"][:n],
                                                               self.Tcr, cfg["K"], cfg["lower_depth"], cfg["upper_depth"], 2,
                                                               self.local[:n])
            self.local[:n] = lm
            self.good[:n] = good
            self.n_good_prl = ngp
        self.matches[:n] = m
        new_kf, abort = decide(cfg, fid - self.kf_id, nto, kf["n_obs_mp"], self.n_good_prl, nin, odom, kf["odom"], kf["accept"])
        r.update(n_matched=nm, n_inlier=nin, n_tracked_old=nto, n_good_prl=self.n_good_prl, triangulated=int(gate),
                 new_kf=int(new_kf), abort_ba=int(abort))
        self.last_odom = odom
        return r

    def reset(self, view_mp):
        """resetLocalTrack after the caller made the current frame a keyframe; view_mp [cap,3] its mViewMPs"""
        n = len(self.cur_kp)
        self.ref_kp, self.ref_desc = self.cur_kp, self.cur_desc
        self.prev[:n, 0], self.prev[:n, 1] = self.cur_kp["x"], self.cur_kp["y"]
        self.local[:] = -1
        self.local[:n] = np.asarray(view_mp, np.float32)[:n]
        self.matches[:] = -1
        self.has_ref, self.kf_id = True, self.frame_id
        self.Tcr = np.eye(4, dtype=np.float32)
        self.meas, self.cov, self.n_good_prl = np.zeros(3), np.zeros(9), 0
