"""ctypes bindings of the CPU oracle (oracle/liboracle.so) — TEST INFRASTRUCTURE ONLY.

Importable from tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs.
The product package (se2lam_b200) never imports this module.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))

KP_DTYPE = np.dtype([("x", "f4"), ("y", "f4"), ("size", "f4"), ("angle", "f4"), ("response", "f4"),
                     ("octave", "i4"), ("class_id", "i4")])
BA_STATS_DTYPE = np.dtype([("chi2_before", "f8"), ("chi2_after", "f8"), ("lambda", "f8"), ("rho", "f8"),
                           ("trials", "i4"), ("accepted", "i4"), ("terminate", "i4"), ("pad", "i4")])


def make(lib: str = "") -> str:
    """Bring oracle/<lib> (every oracle library when lib is empty) up to date with oracle/Makefile, which decides what is
    stale, and return its path. g++ with the Makefile's flags, whatever CXX / CXXFLAGS the environment holds."""
    env = {k: v for k, v in os.environ.items() if k not in ("CXX", "CXXFLAGS")}
    subprocess.run(["make", "-C", HERE, "-s", "CXX=g++"] + ([lib] if lib else []), check=True, env=env)
    return os.path.join(HERE, lib)


_lib = None


def lib():
    global _lib
    if _lib is None:
        L = C.CDLL(make("liboracle.so"))
        vp, i, f, d = C.c_void_p, C.c_int, C.c_float, C.c_double
        L.orb_oracle_create.restype = vp
        L.orb_oracle_create.argtypes = [i, f, i, i]
        L.orb_oracle_destroy.argtypes = [vp]
        L.orb_oracle_extract.argtypes = [vp, vp, i, i, i, vp, vp]
        L.orb_oracle_get_level.argtypes = [vp, i, i, vp]
        L.orb_oracle_level_dims.argtypes = [vp, i] + [C.POINTER(i)] * 3
        L.orb_oracle_retain_best.argtypes = [vp, i, i, vp]
        L.orb_oracle_nth_element.argtypes = [vp, i, i, vp]
        L.orb_oracle_tables.argtypes = [vp] * 6
        L.undistort_oracle.argtypes = [vp, i, i, i, vp, vp, i, vp]
        L.undistort_oracle_map.argtypes = [vp, vp, i, i, i, vp, vp]
        L.ba_oracle_create.restype = vp
        L.ba_oracle_create.argtypes = [i, i, i, i] + [vp] * 11 + [d, d, d, vp, d]
        L.ba_oracle_destroy.argtypes = [vp]
        L.ba_oracle_optimize.argtypes = [vp, i, vp, vp, vp, vp]
        L.ba_oracle_get.argtypes = [vp, vp, vp]
        L.ba_oracle_set.argtypes = [vp, vp, vp]
        L.ba_oracle_num_free.argtypes = [vp]
        L.ba_oracle_chi2.restype = d
        L.ba_oracle_chi2.argtypes = [vp]
        L.ba_oracle_linearize.restype = d
        L.ba_oracle_linearize.argtypes = [vp] * 6
        L.ba_oracle_schur_solve.argtypes = [vp, d, vp, vp, vp, vp]
        L.ba_oracle_edge_xyz.argtypes = [vp, i, vp, vp, vp]
        L.ba_oracle_edge_odo.argtypes = [vp, i, vp, vp, vp]
        L.ba_oracle_edge_information.argtypes = [i, vp, vp, vp, vp, vp, vp, vp, vp, f, f, f, vp]
        L.ba_oracle_writeback_f32.argtypes = [vp, vp, vp]
        L.voc_oracle_transform.argtypes = [i, vp, vp, vp, vp, vp, i, vp, i, i, vp, vp, vp]
        L.median_descriptor_oracle.argtypes = [vp, vp, i, vp, vp]
        if hasattr(L, "matcher_oracle_distance"):
            L.matcher_oracle_distance.argtypes = [vp, vp]
            L.matcher_oracle_match_by_window.argtypes = [vp, vp, i, vp, vp, i, vp, f, f, f, f, f, i, i, i, i, f, vp]
            L.matcher_oracle_match_by_projection.argtypes = [vp, vp, i, vp, vp, vp, i, vp, vp, i, f, f, f, f, i, f, vp]
            L.matcher_oracle_search_by_bow.argtypes = [vp, vp, vp, i, vp, i, vp, vp] * 2 + [i, f, i, vp]
        _lib = L
    return _lib


def _p(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


# ------------------------------------------------------------------------------------------ ORB
class OrbOracle:
    def __init__(self, nfeatures=1000, scale_factor=1.2, nlevels=8, fast_th=20):
        self.nfeatures, self.nlevels = nfeatures, nlevels
        self.h = lib().orb_oracle_create(nfeatures, scale_factor, nlevels, fast_th)

    def __del__(self):
        if getattr(self, "h", None):
            lib().orb_oracle_destroy(self.h)
            self.h = None

    def extract(self, img: np.ndarray):
        img = np.ascontiguousarray(img, np.uint8)
        kps = np.zeros(self.nfeatures + 8, KP_DTYPE)
        desc = np.zeros((self.nfeatures + 8, 32), np.uint8)
        n = lib().orb_oracle_extract(self.h, _p(img), img.shape[1], img.shape[0], img.strides[0], _p(kps), _p(desc))
        return kps[:n].copy(), desc[:n].copy()

    def level(self, level: int, blurred: bool):
        w, hh, p = C.c_int(), C.c_int(), C.c_int()
        lib().orb_oracle_level_dims(self.h, level, C.byref(w), C.byref(hh), C.byref(p))
        out = np.zeros((hh.value + 32, p.value), np.uint8)
        rc = lib().orb_oracle_get_level(self.h, level, int(blurred), _p(out))
        return (out if rc == 0 else None), w.value, hh.value

    def tables(self):
        fpl = np.zeros(self.nlevels, np.int32); sc = np.zeros(self.nlevels, np.float32)
        isc = np.zeros(self.nlevels, np.float32); umax = np.zeros(16, np.int32); gk = np.zeros(7, np.float32)
        lib().orb_oracle_tables(self.h, _p(fpl), _p(sc), _p(isc), _p(umax), _p(gk))
        return dict(features_per_level=fpl, scale=sc, inv_scale=isc, umax=umax, gauss=gk)


def retain_best(responses, n_points):
    r = np.ascontiguousarray(responses, np.float32)
    ids = np.zeros(len(r), np.int32)
    m = lib().orb_oracle_retain_best(_p(r), len(r), n_points, _p(ids))
    return ids[:m].copy()


def nth_element(responses, nth):
    r = np.ascontiguousarray(responses, np.float32)
    ids = np.zeros(len(r), np.int32)
    lib().orb_oracle_nth_element(_p(r), len(r), nth, _p(ids))
    return ids


def undistort(img, K, dist):
    """cv::undistort(img, K, dist) (reference src/Frame.cpp:22): K 3x3 float32, dist 4/5/8/12 float32 coefficients."""
    img = np.ascontiguousarray(img, np.uint8)
    K = np.ascontiguousarray(K, np.float32).reshape(9)
    dist = np.ascontiguousarray(dist, np.float32).ravel()
    out = np.zeros_like(img)
    rc = lib().undistort_oracle(_p(img), img.shape[1], img.shape[0], img.strides[0], _p(K), _p(dist), len(dist), _p(out))
    if rc != 0:
        raise ValueError("singular camera matrix")
    return out


def undistort_map(K, dist, w, h):
    K = np.ascontiguousarray(K, np.float32).reshape(9)
    dist = np.ascontiguousarray(dist, np.float32).ravel()
    m1 = np.zeros((h, w, 2), np.int16); m2 = np.zeros((h, w), np.uint16)
    rc = lib().undistort_oracle_map(_p(K), _p(dist), len(dist), w, h, _p(m1), _p(m2))
    if rc != 0:
        raise ValueError("singular camera matrix")
    return m1, m2


# ------------------------------------------------------------------------------------------ BA
class BAOracle:
    def __init__(self, prob):
        self.prob = prob
        self._keep = [np.ascontiguousarray(a) for a in (
            prob.poses.astype(np.float64), prob.fixed.astype(np.uint8), prob.points.astype(np.float64),
            prob.edge_pose.astype(np.int32), prob.edge_point.astype(np.int32), prob.uv.astype(np.float64),
            prob.info.astype(np.float64), prob.odo_i.astype(np.int32), prob.odo_j.astype(np.int32),
            prob.odo_meas.astype(np.float64), prob.odo_info.astype(np.float64))]
        tcb = np.ascontiguousarray(prob.Tcb, np.float64)
        self.h = lib().ba_oracle_create(prob.P, prob.L, prob.E, prob.O, *[_p(a) for a in self._keep],
                                        prob.fx, prob.cx, prob.cy, _p(tcb), prob.huber_delta)
        self.nf = lib().ba_oracle_num_free(self.h)

    def __del__(self):
        if getattr(self, "h", None):
            lib().ba_oracle_destroy(self.h)
            self.h = None

    def optimize(self, iters, trace=False):
        st = np.zeros(iters, BA_STATS_DTYPE)
        tp = np.zeros((iters, self.prob.P, 3)) if trace else None
        tl = np.zeros((iters, self.prob.L, 3)) if trace else None
        n = lib().ba_oracle_optimize(self.h, iters, _p(st), _p(tp), _p(tl), None)
        if trace:
            return n, st[:n], tp[:n], tl[:n]
        return n, st[:n]

    def get(self):
        poses = np.zeros((self.prob.P, 3)); pts = np.zeros((self.prob.L, 3))
        lib().ba_oracle_get(self.h, _p(poses), _p(pts))
        return poses, pts

    def set(self, poses, pts):
        poses = np.ascontiguousarray(poses, np.float64); pts = np.ascontiguousarray(pts, np.float64)
        lib().ba_oracle_set(self.h, _p(poses), _p(pts))

    def chi2(self):
        return lib().ba_oracle_chi2(self.h)

    def linearize(self):
        n = 3 * self.nf
        out = dict(Hpp=np.zeros((n, n)), bp=np.zeros(n), Hll=np.zeros((self.prob.L, 3, 3)),
                   bl=np.zeros((self.prob.L, 3)), Hpl=np.zeros((self.prob.E, 3, 3)))
        out["chi2"] = lib().ba_oracle_linearize(self.h, _p(out["Hpp"]), _p(out["bp"]), _p(out["Hll"]), _p(out["bl"]), _p(out["Hpl"]))
        return out

    def schur_solve(self, lam):
        n = 3 * self.nf
        out = dict(S=np.zeros((n, n)), bs=np.zeros(n), dx_p=np.zeros(n), dx_l=np.zeros((self.prob.L, 3)))
        out["ok"] = lib().ba_oracle_schur_solve(self.h, lam, _p(out["S"]), _p(out["bs"]), _p(out["dx_p"]), _p(out["dx_l"]))
        return out

    def writeback_f32(self):
        poses = np.zeros((self.prob.P, 3), np.float32); pts = np.zeros((self.prob.L, 3), np.float32)
        lib().ba_oracle_writeback_f32(self.h, _p(poses), _p(pts))
        return poses, pts

    def edge_xyz(self, e):
        err = np.zeros(2); Ji = np.zeros((2, 3)); Jj = np.zeros((2, 3))
        lib().ba_oracle_edge_xyz(self.h, e, _p(err), _p(Ji), _p(Jj))
        return err, Ji, Jj

    def edge_odo(self, o):
        err = np.zeros(3); Ji = np.zeros((3, 3)); Jj = np.zeros((3, 3))
        lib().ba_oracle_edge_odo(self.h, o, _p(err), _p(Ji), _p(Jj))
        return err, Ji, Jj


# ------------------------------------------------------------------------------------------ matcher
def descriptor_distance(a, b):
    a = np.ascontiguousarray(a, np.uint8); b = np.ascontiguousarray(b, np.uint8)
    return lib().matcher_oracle_distance(_p(a), _p(b))


def match_by_window(kp1, d1, kp2, d2, prev, grid, win_size=20, level_offset=1, min_level=0, max_level=8, nnratio=0.9):
    """grid = (minX, minY, invW, invH). Returns (nmatches, matches12, prev_updated)."""
    kp1 = np.ascontiguousarray(kp1); kp2 = np.ascontiguousarray(kp2)
    d1 = np.ascontiguousarray(d1, np.uint8); d2 = np.ascontiguousarray(d2, np.uint8)
    prev = np.ascontiguousarray(prev, np.float32).copy()
    m = np.zeros(len(kp1), np.int32)
    n = lib().matcher_oracle_match_by_window(_p(kp1), _p(d1), len(kp1), _p(kp2), _p(d2), len(kp2), _p(prev),
                                             grid[0], grid[1], grid[2], grid[3], float(win_size), level_offset,
                                             min_level, max_level, 1, nnratio, _p(m))
    return n, m, prev


def match_by_projection(kfkp, kfdesc, kf_observed, mp_valid, mp_uv, mp_octave, mp_desc, grid, win_size=15,
                        level_offset=2, nnratio=0.6):
    kfkp = np.ascontiguousarray(kfkp); kfdesc = np.ascontiguousarray(kfdesc, np.uint8)
    kf_observed = np.ascontiguousarray(kf_observed, np.uint8); mp_valid = np.ascontiguousarray(mp_valid, np.uint8)
    mp_uv = np.ascontiguousarray(mp_uv, np.float32); mp_octave = np.ascontiguousarray(mp_octave, np.int32)
    mp_desc = np.ascontiguousarray(mp_desc, np.uint8)
    m = np.zeros(len(kfkp), np.int32)
    n = lib().matcher_oracle_match_by_projection(_p(kfkp), _p(kfdesc), len(kfkp), _p(kf_observed), _p(mp_valid), _p(mp_uv),
                                                 len(mp_valid), _p(mp_octave), _p(mp_desc), win_size, grid[0], grid[1],
                                                 grid[2], grid[3], level_offset, nnratio, _p(m))
    return n, m


def search_by_bow(kf1, kf2, mp_only=True, nnratio=0.6, check_ori=True):
    """kf = dict(angle[f4 N], desc[N,32], has_mp[u8 N], node[i4 K] ascending, ptr[i4 K+1], feat[i4])."""
    def args(k):
        a = [np.ascontiguousarray(k["angle"], np.float32), np.ascontiguousarray(k["desc"], np.uint8),
             np.ascontiguousarray(k["has_mp"], np.uint8), np.ascontiguousarray(k["node"], np.int32),
             np.ascontiguousarray(k["ptr"], np.int32), np.ascontiguousarray(k["feat"], np.int32)]
        return a, [_p(a[0]), _p(a[1]), _p(a[2]), len(a[0]), _p(a[3]), len(a[3]), _p(a[4]), _p(a[5])]
    k1, a1 = args(kf1); k2, a2 = args(kf2)
    m = np.zeros(len(k1[0]), np.int32)
    n = lib().matcher_oracle_search_by_bow(*a1, *a2, int(mp_only), nnratio, int(check_ori), _p(m))
    return n, m


def edge_information(view_mp, edge_pose, edge_point, octave, kf_Rcw, kf_twb_xy, mp_pos, level_sigma2, fx, xrot_info=1e6, z_info=1.0):
    """Per-edge information of Map::loadLocalGraph (Map.cpp:1024-1049) from float inputs. Returns [E,3] (xx, xy, yy)."""
    c = np.ascontiguousarray
    view_mp = c(view_mp, np.float32); edge_pose = c(edge_pose, np.int32); edge_point = c(edge_point, np.int32); octave = c(octave, np.int32)
    kf_Rcw = c(kf_Rcw, np.float32); kf_twb_xy = c(kf_twb_xy, np.float32); mp_pos = c(mp_pos, np.float32); level_sigma2 = c(level_sigma2, np.float32)
    info = np.zeros((len(edge_pose), 3))
    lib().ba_oracle_edge_information(len(edge_pose), _p(view_mp), _p(edge_pose), _p(edge_point), _p(octave), _p(kf_Rcw), _p(kf_twb_xy),
                                     _p(mp_pos), _p(level_sigma2), float(fx), float(xrot_info), float(z_info), _p(info))
    return info


# ------------------------------------------------------------------------------------------ bag of words
def voc_transform(voc, feats, levelsup):
    """voc = dict(desc [n,32] u8, child_ptr [n+1], children, word_id [n], weight [n] f8, levels). Returns (word, weight, node)."""
    c = np.ascontiguousarray
    desc = c(voc["desc"], np.uint8); cp = c(voc["child_ptr"], np.int32); ch = c(voc["children"], np.int32)
    wid = c(voc["word_id"], np.int32); wt = c(voc["weight"], np.float64); feats = c(feats, np.uint8)
    n = len(feats)
    word = np.zeros(n, np.int32); weight = np.zeros(n); node = np.zeros(n, np.int32)
    lib().voc_oracle_transform(len(desc), _p(desc), _p(cp), _p(ch), _p(wid), _p(wt), int(voc["levels"]), _p(feats), n, int(levelsup),
                               _p(word), _p(weight), _p(node))
    return word, weight, node


def median_descriptor(desc, ptr):
    desc = np.ascontiguousarray(desc, np.uint8); ptr = np.ascontiguousarray(ptr, np.int32)
    M = len(ptr) - 1
    idx = np.zeros(M, np.int32); med = np.zeros(M, np.int32)
    lib().median_descriptor_oracle(_p(desc), _p(ptr), M, _p(idx), _p(med))
    return idx, med
