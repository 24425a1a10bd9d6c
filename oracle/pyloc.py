"""CPU restatement of Localizer::run (reference src/Localizer.cpp) over a flattened static map — TEST INFRASTRUCTURE ONLY.

`LocOracle` is one camera stream. It composes the ORB oracle, the MatchByProjection oracle and the pose-only BA oracle
with the Localizer's own logic (UpdatePoseCurr, the projection and inImgBound, UpdateCovisKFCurr, UpdateLocalMap,
MatchLoopClose), which comes from oracle/libloc_oracle.so (oracle/loc_oracle.cpp, built by oracle/loc.mk) or, with
logic="numpy", from its independent restatement oracle/loc_numpy.py. Map points are listed in ascending index, the order
the device handle uses (DESIGN.md section 15).
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

from oracle import loc_numpy, pyoracle, pypose

F = np.float32
HERE = os.path.dirname(os.path.abspath(__file__))
_lib = None


def make() -> str:
    """Bring oracle/libloc_oracle.so up to date with oracle/loc.mk and return its path."""
    env = {k: v for k, v in os.environ.items() if k not in ("CXX", "CXXFLAGS")}
    subprocess.run(["make", "-C", HERE, "-s", "-f", "loc.mk", "CXX=g++"], check=True, env=env)
    return os.path.join(HERE, "libloc_oracle.so")


def lib():
    global _lib
    if _lib is None:
        L = C.CDLL(make())
        vp, i = C.c_void_p, C.c_int
        L.loc_oracle_pose.argtypes = [vp] * 6
        L.loc_oracle_pose.restype = None
        L.loc_oracle_project.argtypes = [vp, vp, i, vp, vp, vp, vp]
        L.loc_oracle_project.restype = None
        L.loc_oracle_covis.argtypes = [vp, vp, vp, i, vp]
        L.loc_oracle_local_map.argtypes = [vp, vp, i, vp, vp, i]
        L.loc_oracle_loop_close.argtypes = [vp, i, i, vp, vp, vp, vp]
        _lib = L
    return _lib


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


class CppLogic:
    """the functions of oracle/loc_numpy.py, computed by oracle/loc_oracle.cpp"""

    def __init__(self, m):
        from se2lam_b200._capi import LocMap
        from se2lam_b200.loc import MAP_FIELDS
        self.m = m
        self.keep = {k: np.ascontiguousarray(m[k], t) for k, t in MAP_FIELDS.items()}
        c = LocMap()
        c.n_kf, c.n_mp = len(self.keep["kf_kp_ptr"]) - 1, len(self.keep["mp_null"])
        for k, a in self.keep.items():
            setattr(c, k, _p(a) if a.size else None)
        self.cmap = c

    @staticmethod
    def pose(cfg, odom, ref_odom, ref_Tcw):
        f = lambda a: np.ascontiguousarray(a, F)
        T = np.zeros(16, F)
        cTb, bTc, o, r, t = f(cfg["cTb"]), f(cfg["bTc"]), f(odom), f(ref_odom), f(ref_Tcw)
        lib().loc_oracle_pose(_p(cTb), _p(bTc), _p(o), _p(r), _p(t), _p(T))
        return T.reshape(4, 4)

    @staticmethod
    def project(K, T, pos, bounds):
        P = np.ascontiguousarray(pos, F).reshape(-1, 3)
        n = len(P)
        ok, uv = np.zeros(n, np.uint8), np.zeros((n, 2), F)
        Kf, Tf, b = np.ascontiguousarray(K, F), np.ascontiguousarray(T, F), np.ascontiguousarray(bounds, F)
        if n:
            lib().loc_oracle_project(_p(Kf), _p(Tf), n, _p(P), _p(b), _p(ok), _p(uv))
        return ok, uv

    def covis(self, m, local_kfs, obs_mp, cov):
        lk, o = np.ascontiguousarray(local_kfs, np.uint8), np.ascontiguousarray(obs_mp, np.int32)
        return lib().loc_oracle_covis(C.byref(self.cmap), _p(lk), _p(o), len(o), _p(cov))

    def local_map(self, m, cov, hops, cap):
        K, M = self.cmap.n_kf, self.cmap.n_mp
        lk, lst = np.zeros(max(K, 1), np.uint8), np.zeros(max(M, 1), np.int32)
        c = np.ascontiguousarray(cov, np.uint8)
        n = lib().loc_oracle_local_map(C.byref(self.cmap), _p(c), int(hops), _p(lk), _p(lst), M)
        return lk[:K], [int(v) for v in lst[:min(n, cap)]], n

    def loop_close(self, m, kf, pairs, obs_mp):
        cur = np.ascontiguousarray([p[0] for p in pairs], np.int32)
        loop = np.ascontiguousarray([p[1] for p in pairs], np.int32)
        bad = C.c_int(0)
        nulls = lib().loc_oracle_loop_close(C.byref(self.cmap), int(kf), len(cur), _p(cur), _p(loop), _p(obs_mp), C.byref(bad))
        return nulls, bad.value


def host_pose(cfg, odom, ref_odom, ref_Tcw):
    """UpdatePoseCurr, from the C++ oracle"""
    return CppLogic.pose(cfg, odom, ref_odom, ref_Tcw)


class LocOracle:
    """One camera stream of the Localizer over the map dict m. cfg: the tools/loc_scenes.py configuration; isig:
    mvInvLevelSigma2; logic: "cpp" (oracle/loc_oracle.cpp) or "numpy" (oracle/loc_numpy.py), or an object with their
    functions (one CppLogic may be shared by many streams)."""

    def __init__(self, cfg, m, isig, logic="cpp"):
        self.cfg, self.m, self.isig = cfg, m, np.asarray(isig, F)
        self.L = CppLogic(m) if logic == "cpp" else loc_numpy if logic == "numpy" else logic
        self.K = len(m["kf_kp_ptr"]) - 1
        self.cap = int(cfg["max_local_mps"])
        self.orb = pyoracle.OrbOracle(cfg["nfeatures"], cfg["scale_factor"], cfg["nlevels"], cfg["fast_th"])
        self.has_frame = self.tracked = self.first = False
        self.Tcw = np.asarray(cfg["cTb"], F).copy()
        self.odom = np.zeros(3, F)
        self.kp = np.zeros(0, pyoracle.KP_DTYPE)
        self.desc = np.zeros((0, 32), np.uint8)
        self.obs_mp = np.zeros(0, np.int32)
        self.covis = np.zeros(self.K, np.uint8)
        self.local_kfs = set()
        self.local_kf_mask = np.zeros(self.K, np.uint8)
        self.local_mps, self.n_local_mps = [], 0
        self.branches = []

    # KeyFrame::getSizeObsMP
    def n_obs(self):
        return len(set(int(v) for v in self.obs_mp if v >= 0))

    def step(self, img, odom, Tcw_prev=None):
        """one Localizer::run iteration; Tcw_prev (teacher forcing) replaces the previous pose. Returns the record dict."""
        odom = np.asarray(odom, F)
        if Tcw_prev is not None:
            self.Tcw = np.asarray(Tcw_prev, F).copy()
        img = pyoracle.frame_image(img, self.cfg["K"], self.cfg.get("dist", ()))   # ReadFrameInfo builds a Frame, which undistorts
        self.kp, self.desc = self.orb.extract(img)
        self.obs_mp = np.full(len(self.kp), -1, np.int32)
        self.covis = np.zeros(self.K, np.uint8)
        r = dict(tracked=0, first=0, n_keypoints=len(self.kp), n_matched=0, n_obs_mp=0, ba_status=1, ba_iterations=0,
                 n_local_kfs=0, n_local_mps=0, overflow=0)
        if not self.has_frame:                                             # mpKFRef == NULL: continue
            self.Tcw = np.asarray(self.cfg["cTb"], F).copy()
            self.has_frame, self.first = True, True
            self.odom = odom
            r["first"] = 1
            self.branches.append("first")
            return r
        self.first = False
        self.Tcw = self.L.pose(self.cfg, odom, self.odom, self.Tcw)       # UpdatePoseCurr
        self.odom = odom
        if self.tracked:
            r["n_matched"] = self.match_local_map()
            n = self.n_obs()
            r["n_obs_mp"] = n
            if n > 30:
                r["ba_status"], r["ba_iterations"] = self.local_ba()
            else:
                r["ba_status"] = 3
                self.branches.append("gated")
            if self.L.covis(self.m, self.local_kf_mask, self.obs_mp, self.covis):   # UpdateCovisKFCurr
                self.branches.append("covis_edge")
            self.update_local_map(1)
            self.tracked = len(self.local_kfs) > 0                         # DetectIfLost
            self.branches.append("tracked" if self.tracked else "lost_now")
            r.update(n_local_kfs=len(self.local_kfs), n_local_mps=self.n_local_mps)
        else:
            self.branches.append("lost")
        r["tracked"] = int(self.tracked)
        r["overflow"] = int(self.n_local_mps > self.cap)
        if r["overflow"]:
            self.branches.append("overflow")
        return r

    def match_local_map(self):
        """MatchLocalMap over the local list (at most max_local_mps of it)"""
        cfg, m = self.cfg, self.m
        L = np.asarray(self.local_mps, np.int64)
        Q = len(L)
        if len(self.kp) == 0 or Q == 0:
            return 0
        has = np.zeros(len(m["mp_null"]), bool)
        has[self.obs_mp[self.obs_mp >= 0]] = True
        use = (m["mp_null"][L] == 0) & (m["mp_good_prl"][L] != 0) & ~has[L]   # !isNull && isGoodPrl && !hasObservation
        inb, uv = self.L.project(cfg["K"], self.Tcw, m["mp_pos"][L], cfg["bounds"])
        valid = (use & (inb != 0)).astype(np.uint8)
        uv = np.where(valid[:, None] != 0, uv, F(0)).astype(F)
        octv = np.where(valid != 0, m["mp_octave"][L], 0).astype(np.int32)
        mdesc = np.where(valid[:, None] != 0, m["mp_desc"][L], 0).astype(np.uint8)
        observed = (self.obs_mp >= 0).astype(np.uint8)
        n, mt = pyoracle.match_by_projection(self.kp, self.desc, observed, valid, uv, octv, mdesc, cfg["grid"], 15, 2, 0.9)
        for i, q in enumerate(mt):                                         # KeyFrame::addObservation in idxKPCurr order
            if q >= 0:
                self.obs_mp[i] = L[q]
        return int(n)

    def local_ba(self):
        """DoLocalBA: edges in ascending map-point index, uv of the last keypoint that observed the point, octave-0 information"""
        cfg, m = self.cfg, self.m
        xyz, uvs, ws = [], [], []
        w0 = self.isig[int(self.kp["octave"][0])] if len(self.kp) else F(0)
        for j in sorted(set(int(v) for v in self.obs_mp if v >= 0)):
            if m["mp_null"][j] or not m["mp_good_prl"][j]:
                continue
            i = int(np.flatnonzero(self.obs_mp == j).max())
            xyz.append(m["mp_pos"][j]); uvs.append((self.kp["x"][i], self.kp["y"][i])); ws.append(w0)
        if not xyz:
            return 1, 0
        K = np.asarray(cfg["K"], F)
        o = pypose.run(self.Tcw, np.array(xyz, F), np.array(uvs, F), np.array(ws, F), K[0, 0], K[0, 2], K[1, 2], cfg["bTc"],
                       cfg["huber"], iterations=30)
        self.Tcw = o["Tcw"].astype(F)
        return int(o["status"]), int(o["iterations"])

    def update_local_map(self, level):
        self.local_kf_mask, self.local_mps, self.n_local_mps = self.L.local_map(self.m, self.covis, level, self.cap)
        self.local_kfs = {int(k) for k in np.flatnonzero(self.local_kf_mask)}

    def relocalize(self, kf, pairs, Tcw_first=None):
        """the verified branch (Localizer.cpp:123-139), then DetectIfLost; Tcw_first replaces the pose after the first BA"""
        self.Tcw = np.asarray(self.m["kf_Tcw"][kf], F).copy()
        self.covis = np.zeros(self.K, np.uint8)
        self.covis[kf] = 1
        self.update_local_map(3)
        nulls, bad = self.L.loop_close(self.m, kf, pairs, self.obs_mp)    # MatchLoopClose
        if nulls:
            self.branches.append("loop_null")
        if bad:
            self.branches.append("loop_badprl")
        if len({p[1] for p in pairs}) < len(pairs):
            self.branches.append("loop_repeat")
        self.local_ba()
        first = self.Tcw.copy()
        if Tcw_first is not None:
            self.Tcw = np.asarray(Tcw_first, F).copy()
        n_matched = self.match_local_map()
        st, it = self.local_ba()
        self.tracked = len(self.local_kfs) > 0
        self.branches.append("relocalized")
        return dict(tracked=int(self.tracked), first=0, n_keypoints=len(self.kp), n_matched=n_matched, n_obs_mp=self.n_obs(),
                    ba_status=st, ba_iterations=it, n_local_kfs=len(self.local_kfs), n_local_mps=self.n_local_mps,
                    overflow=int(self.n_local_mps > self.cap)), first
