"""An independent numpy restatement of the map-point updates (MapPoint::addObservation / eraseObservation /
updateMeasureInKFs, reference src/MapPoint.cpp) - TEST INFRASTRUCTURE ONLY, checked against oracle/mappoint_oracle.cpp.

It works on the same tables (dicts of numpy arrays, updated in place) but holds each point's list as a Python list and
writes the control flow out again from the reference. The two-view pieces it shares with the geometry oracle
(cvu::triangulate, Track::calcSE3toXYZInfo, cv::gemm's small path) come from oracle/pygeom.py, which
tests/test_geom_oracle.py checks on its own; the rest is numpy float32 / float64 scalar arithmetic in the reference's order,
so the results are bit-exact. Every call also records which branches it took (`trace`), so tests can see that each case
reaches the branch it was built for.
"""
from __future__ import annotations

import numpy as np

from oracle import pygeom

f32, f64 = np.float32, np.float64


def _norm3(v):
    return np.sqrt(f64(v[0]) * f64(v[0]) + f64(v[1]) * f64(v[1]) + f64(v[2]) * f64(v[2]))


def _unit(v):
    s = f64(1.0) / _norm3(v)
    return np.array([f32(f64(v[k]) * s) for k in range(3)], f32)


def _gemm_dbl(A, B):
    """3x3 float product with double sums (cv::gemm's generic path, GEMM_1_T / GEMM_2_T applied by the caller)"""
    D = np.zeros((3, 3), f32)
    for i in range(3):
        for j in range(3):
            s = f64(0)
            for k in range(3):
                s = s + f64(A[i, k]) * f64(B[k, j])
            D[i, j] = f32(s * 1.0)
    return D


class Restatement:
    def __init__(self, kf, mp, params):
        self.kf, self.mp, self.p = kf, mp, params
        self.trace = []
        self.pkf0 = []                                     # (m, q, j0) of every updateParallax that chose a pKF0
        self.sf = np.asarray(params["scale_factors"], f32)

    # ------------------------------------------------------------------ helpers over list entries (positions j of point m)
    def _kf(self, m, j): return int(self.mp["obs_kf"][self.mp["obs_ptr"][m] + j])
    def _slot(self, m, j): return int(self.kf["kp_base"][self._kf(m, j)] + self.mp["obs_idx"][self.mp["obs_ptr"][m] + j])
    def _id(self, m, j): return int(self.kf["kf_id"][self._kf(m, j)])
    def _T(self, m, j): return self.kf["Tcw"][self._kf(m, j)]

    def _ev(self, m, what):
        self.trace.append((m, what))

    def _main(self, m, obs):
        kf, mp = self.kf, self.mp
        if mp["null"][m] or not obs:
            return
        v = [j for j in obs if not kf["kf_null"][self._kf(m, j)]]
        if len(v) < len(obs):
            self._ev(m, "null_kf_skipped")
        if len(v) <= 32 < int(mp["obs_ptr"][m + 1] - mp["obs_ptr"][m]):
            self._ev(m, "short_median_of_long_list")
        if not v:
            return
        d = [kf["desc"][self._slot(m, j)] for j in v]
        N = len(v)
        D = np.array([[int(np.unpackbits(d[a] ^ d[b]).sum()) for b in range(N)] for a in range(N)])
        med = [int(np.sort(D[i])[int(0.5 * (N - 1))]) for i in range(N)]
        best = int(np.argmin(med))                         # first index of the least median
        if med.count(med[best]) > 1:
            self._ev(m, "median_tie")
        jb = v[best]; s = self._slot(m, jb); k = self._kf(m, jb)
        mp["main_desc"][m] = kf["desc"][s]
        mp["main_measure"][m] = (kf["kp"]["x"][s], kf["kp"]["y"][s])
        if mp["main_kf"][m] >= 0 and kf["kf_id"][mp["main_kf"][m]] == kf["kf_id"][k]:
            self._ev(m, "main_unchanged")
            return
        self._ev(m, "main_changed")
        if len(self.sf) != 8:
            self._ev(m, "range_of_other_nlevels")
        mp["main_kf"][m] = k
        o = int(kf["kp"]["octave"][s])
        mp["main_octave"][m] = o
        mp["level_scale"][m] = self.sf[o]
        dist = f32(_norm3(kf["view_mp"][s]))
        mp["max_dist"][m] = f32(dist * self.sf[o])
        mp["min_dist"][m] = f32(mp["max_dist"][m] / self.sf[-1])

    def _set_view(self, m, j, pos, info):
        s = self._slot(m, j)
        self.kf["view_mp"][s] = pos
        self.kf["view_info"][s] = info

    def _parallax(self, m, obs, q):
        kf, mp, p = self.kf, self.mp, self.p
        if mp["good_prl"][m]:
            self._ev(m, "already_good"); return False
        if len(obs) <= 2:
            self._ev(m, "short_list"); return False
        idn = self._id(m, q)
        j0 = None
        for j in obs:
            if idn - self._id(m, j) > 6:
                continue
            if j0 is None or self._id(m, j) < self._id(m, j0):
                j0 = j
        self._ev(m, "pkf0_self" if j0 == q else "pkf0_older")
        self.pkf0.append((m, q, j0))
        if any(idn - self._id(m, j) > 6 for j in obs):
            self._ev(m, "observer_beyond_6")
        T0, T1 = self._T(m, j0), self._T(m, q)
        Kc = np.asarray(p["K"], f32)
        P = np.stack([pygeom.gemm3(Kc, T0[:3]), pygeom.gemm3(Kc, T1[:3])])
        s0, s1 = self._slot(m, j0), self._slot(m, q)
        pt0 = np.array([kf["kp"]["x"][s0], kf["kp"]["y"][s0]], f32)
        pt1 = np.array([kf["kp"]["x"][s1], kf["kp"]["y"][s1]], f32)
        posW = pygeom.triangulate(pt0[None], pt1[None], P, np.array([0], np.int32), np.array([1], np.int32))[0]

        def se3map(T, x):
            r = [f32(f32(f32(f32(0) + f32(T[i, 0] * x[0])) + f32(T[i, 1] * x[1])) + f32(T[i, 2] * x[2])) for i in range(3)]
            return np.array([f32(r[i] + T[i, 3]) for i in range(3)], f32)

        pos0, pos1 = se3map(T0, posW), se3map(T1, posW)
        lo, hi = f32(p["lower_depth"]), f32(p["upper_depth"])
        ok = False
        if not (lo <= pos0[2] <= hi and lo <= pos1[2] <= hi):
            self._ev(m, "depth_below" if min(pos0[2], pos1[2]) < lo else "depth_above")
        else:
            O0, O1 = pygeom.inv(T0)[:3, 3], pygeom.inv(T1)[:3, 3]
            ok = pygeom.check_parallax(O0, O1, posW, 2)
            self._ev(m, "triangulated" if ok else "parallax_rejected")
        if ok:
            mp["pos"][m] = posW
            mp["good_prl"][m] = 1
            Tt = np.stack([T0, T1])
            info0, info1 = pygeom.xyz_info(pos0[None], np.array([0], np.int32), np.array([1], np.int32), Tt, p["fx"])
            self._set_view(m, j0, pos0, info0[0])
            self._set_view(m, q, pos1, info1[0])
            R0 = np.ascontiguousarray(T0[:3, :3])
            W = pygeom.gemm3(_gemm_dbl(R0.T, info0[0].astype(f32)), R0)
            for j in obs:
                if self._id(m, j) in (idn, self._id(m, j0)):
                    continue
                Rk = np.ascontiguousarray(self._T(m, j)[:3, :3])
                Wk = _gemm_dbl(pygeom.gemm3(Rk, W), Rk.T)
                self._set_view(m, j, se3map(self._T(m, j), posW), Wk.astype(f64))
        if idn - self._id(m, j0) >= 6 and not mp["good_prl"][m]:
            self._ev(m, "abandoned")
            mp["null"][m] = 1; mp["good_prl"][m] = 0
            obs.clear()
            return True
        return False

    # ------------------------------------------------------------------ the three operations
    def add(self, upd_ptr, upd_pos):
        mp = self.mp
        M = len(mp["obs_ptr"]) - 1
        ab = np.zeros(M, bool)
        for m in range(M):
            ups = [int(x) for x in upd_pos[upd_ptr[m]:upd_ptr[m + 1]]]
            L = int(mp["obs_ptr"][m + 1] - mp["obs_ptr"][m])
            obs = [j for j in range(L) if j not in ups]
            if len(ups) > 1:
                self._ev(m, "two_adds")
            for q in ups:
                old = len(obs)
                obs.append(q); obs.sort()
                was_null = bool(mp["null"][m])
                self._main(m, obs)
                if ab[m] and not mp["good_prl"][m] and len(obs) > 2:
                    self._ev(m, "parallax_after_abandon")
                ab[m] |= self._parallax(m, obs, q)
                nn = _unit(self.kf["view_mp"][self._slot(m, q)])
                n = mp["normal"][m]
                f = f32(f32(1) / f32(old + 1))
                mp["normal"][m] = [f32(f32(f32(n[k] * f32(old)) + nn[k]) * f) for k in range(3)]
                if mp["null"][m] or was_null:
                    self._ev(m, "null_reset")
                mp["null"][m] = 0
        return ab

    def erase(self, upd_ptr, upd_pos):
        mp = self.mp
        M = len(mp["obs_ptr"]) - 1
        ab = np.zeros(M, bool)
        for m in range(M):
            obs = list(range(int(mp["obs_ptr"][m + 1] - mp["obs_ptr"][m])))
            for q in [int(x) for x in upd_pos[upd_ptr[m]:upd_ptr[m + 1]]]:
                npos = _unit(self.kf["view_mp"][self._slot(m, q)])
                if mp["main_kf"][m] == self._kf(m, q):
                    self._ev(m, "erase_main")
                obs.remove(q)
                if not mp["null"][m] and not obs:
                    self._ev(m, "erased_to_empty")
                    mp["null"][m] = 1; mp["good_prl"][m] = 0
                    ab[m] = True
                    continue
                before = int(mp["main_kf"][m])
                self._main(m, obs)
                if mp["main_kf"][m] != before:
                    self._ev(m, "erase_main_changed")
                size = len(obs)
                n = mp["normal"][m]
                with np.errstate(divide="ignore", invalid="ignore"):
                    f = f32(f32(1) / f32(size))
                    mp["normal"][m] = [f32(f32(f32(n[k] * f32(size + 1)) - npos[k]) * f) for k in range(3)]
        return ab

    def update_measure(self, points):
        kf, mp = self.kf, self.mp
        for m in points:
            pos = mp["pos"][m]
            for j in range(int(mp["obs_ptr"][m + 1] - mp["obs_ptr"][m])):
                k = self._kf(m, j)
                if kf["kf_null"][k]:
                    continue
                T = kf["Tcw"][k]
                r = [f32(f32(f32(f32(0) + f32(T[i, 0] * pos[0])) + f32(T[i, 1] * pos[1])) + f32(T[i, 2] * pos[2])) for i in range(3)]
                kf["view_mp"][self._slot(m, j)] = [f32(r[i] + T[i, 3]) for i in range(3)]
