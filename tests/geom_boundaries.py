"""Boundary pairs of the two-view geometry and map-point decisions (tests/test_geom_boundaries_oracle.py,
tests/test_geom_paths_gpu.py).

A pair is two inputs that differ in one value and on which the oracle takes the two sides of one comparison, every other
condition being comfortably met on both. Float pairs are adjacent floats: either a bound set to a value the oracle computed
(a depth or a distance read from its output with wide bounds, and the next float beyond it), or the two floats that a
bisection over an input's bit patterns leaves when the oracle's decision differs at its ends (a keypoint coordinate for the
parallax cosine, one normal component for acceptNewObserve's 30 degree cosine). Integer pairs take the exact differences
the reference compares: octaves 2 and 3 apart, keyframe ids 5, 6 and 7 apart.

Every pair is built from public inputs and the oracles alone (oracle/pygeom.py, oracle/pymappoint.py).
"""
from __future__ import annotations

import numpy as np

from oracle import mappoint_numpy as mpn
from oracle import pygeom
from oracle import pymappoint as pm
from tools import geom_scenes as gs
from tools import mappoint_scenes as ms

f32, f64 = np.float32, np.float64
MIN_COS = tuple(f32(c) for c in (0.9998, 0.9994, 0.9986, 0.9976))     # cvu::checkParallax's minCos
COS30 = f32(0.866)                                                     # acceptNewObserve's c2
WIDE = (f32(-1e30), f32(1e30))


# ------------------------------------------------------------------------------------------ float bit patterns
def key(x):
    """float32 -> an integer that orders like the float (adjacent floats are adjacent integers)"""
    i = int(np.array(x, f32).view(np.int32))
    return i if i >= 0 else -(i & 0x7FFFFFFF)


def unkey(k):
    return np.array(k if k >= 0 else (-k) | -0x80000000, np.int32).view(f32)[()]


def bits(x):
    return f"0x{int(np.array(x, f32).view(np.uint32)):08x}"


def up(x):
    return np.nextafter(f32(x), f32(np.inf))


def down(x):
    return np.nextafter(f32(x), f32(-np.inf))


def bisect(decide, a, b):
    """adjacent floats (x0, x1) between a and b with decide(x0) != decide(x1); decide(a) != decide(b) is required"""
    ka, kb = key(a), key(b)
    da, db = decide(unkey(ka)), decide(unkey(kb))
    assert da != db, "the ends must decide differently"
    while abs(kb - ka) > 1:
        km = (ka + kb) // 2
        if decide(unkey(km)) == da:
            ka = km
        else:
            kb = km
    return (unkey(ka), unkey(kb)) if ka < kb else (unkey(kb), unkey(ka))


class Pair:
    """Two inputs (`a`, `b`: dicts of the call's arguments) on the two sides of one comparison. `what` names the decision,
    `field` the one input that differs, `values` its two values."""

    def __init__(self, kind, what, field, a, b):
        self.kind, self.what, self.field, self.a, self.b = kind, what, field, a, b

    @property
    def values(self):
        return get(self.a, self.field), get(self.b, self.field)

    def describe(self):
        va, vb = self.values
        if isinstance(va, (np.floating, float)):
            return f"{self.kind}:{self.what}: {self.field} = {va!r} ({bits(va)}) | {vb!r} ({bits(vb)})"
        return f"{self.kind}:{self.what}: {self.field} = {va} | {vb}"

    def __repr__(self):
        return f"Pair({self.kind}:{self.what})"


def get(d, path):
    for p in path.split("."):
        d = d[int(p)] if isinstance(d, (list, np.ndarray)) else d[p]
    return d


# ------------------------------------------------------------------------------------------ Track::doTriangulate
def _kp(xy, octave=0):
    kp = np.zeros(len(xy), gs.KP_DTYPE)
    kp["x"] = [p[0] for p in xy]; kp["y"] = [p[1] for p in xy]
    kp["size"] = 31; kp["octave"] = octave; kp["class_id"] = -1
    return kp


def _sideways_tcr(tx=-0.1):
    """a sideways step with a small yaw: epipolar lines close to the rows"""
    c, s = np.cos(0.02), np.sin(0.02)
    T = np.eye(4, dtype=np.float64)
    T[:3, :3] = [[c, 0, s], [0, 1, 0], [-s, 0, c]]
    T[:3, 3] = [tx, 0.004, 0.01]
    return T.astype(f32)


def track_case(X=(0.4, -0.2, 4.0), frame_x=None, lower=gs.LOWER_DEPTH, upper=gs.UPPER_DEPTH, deg=2):
    """one keyframe keypoint, the projection of X (reference-camera coordinates) matched to its projection in the frame;
    frame_x replaces the frame keypoint's x"""
    Tcr = _sideways_tcr()
    P0 = gs.K.astype(f64) @ np.eye(3, 4); P1 = gs.K.astype(f64) @ Tcr[:3].astype(f64)
    X = np.asarray(X, f64)
    pk, pf = gs.project(P0, X).astype(f32), gs.project(P1, X).astype(f32)
    if frame_x is not None:
        pf[0] = frame_x
    return dict(kp_kf=_kp([pk]), kp_frame=_kp([pf]), matches12=np.zeros(1, np.int32), kf_observed=np.zeros(1, np.uint8),
                kf_view_mp=np.full((1, 3), 5.0, f32), Tcr=Tcr, K=gs.K, lower=f32(lower), upper=f32(upper), deg=int(deg),
                local_mps=np.full((1, 3), 7.0, f32))


def track_oracle(c):
    return pygeom.track_triangulate(c["kp_kf"], c["kp_frame"], c["matches12"], c["kf_observed"], c["kf_view_mp"], c["Tcr"],
                                    c["K"], c["lower"], c["upper"], c["deg"], c["local_mps"])


def track_decisions(c):
    """(depth accepted, parallax good) of row 0"""
    m, _, good, _ = track_oracle(c)
    return bool(m[0] >= 0), bool(good[0])


def track_pairs():
    pairs = []
    base = track_case(lower=WIDE[0], upper=WIDE[1])
    z = track_oracle(base)[1][0, 2]
    ok = track_case()
    pairs.append(Pair("track", "depth_lower", "lower", dict(ok, lower=z), dict(ok, lower=up(z))))
    pairs.append(Pair("track", "depth_upper", "upper", dict(ok, upper=z), dict(ok, upper=down(z))))
    # parallax: slide the frame keypoint along its row between the projections of a near point (1 m, wide parallax) and
    # a far one (9 m, narrow), both well inside the depth window
    X = np.array([0.3, -0.2, 1.0])
    near = track_case(X=X)["kp_frame"]["x"][0]
    far = track_case(X=X * 9.0)["kp_frame"]["x"][0]
    for deg in (1, 2, 3, 4):
        mk = lambda x, deg=deg: track_case(X=X, frame_x=x, deg=deg)
        x0, x1 = bisect(lambda x: track_decisions(mk(x)), near, far)
        pairs.append(Pair("track", f"parallax_deg{deg}", "kp_frame.0.x", _kp_set(mk(x0), x0), _kp_set(mk(x1), x1)))
    return pairs


def _kp_set(c, x):
    c["kp_frame"]["x"][0] = x
    return c


# ------------------------------------------------------------------------------------------ findCorrespd's projection branch
def projection_case(octave_diff=0, normal_x=None, min_dist=WIDE[0], max_dist=WIDE[1], lower=gs.LOWER_DEPTH,
                    upper=gs.UPPER_DEPTH):
    """one new-keyframe keypoint matched to map point 0, whose main keyframe is pose 0 of a two-pose table; the normal is
    the point's bearing from the new keyframe (cosine 1), normal_x replaces its x component"""
    T0 = gs.tcw_of_odom(1.0, 0.2, 0.1)
    Tn = gs.tcw_of_odom(1.0, -0.1, 0.1)
    Xc = np.array([0.5, -0.3, 3.5])
    Xw = np.linalg.inv(Tn.astype(f64)) @ np.append(Xc, 1.0)
    meas = gs.project(gs.K.astype(f64) @ T0[:3].astype(f64), Xw[:3]).astype(f32)
    uv = gs.project(gs.K.astype(f64) @ Tn[:3].astype(f64), Xw[:3]).astype(f32)
    main_oct = 4
    nv = (Xc / np.linalg.norm(Xc)).astype(f32)
    if normal_x is not None:
        nv[0] = normal_x
    mp = dict(main_measure=meas[None], main_pose=np.zeros(1, np.int32), main_octave=np.array([main_oct], np.int32),
              normal=nv[None], min_dist=np.array([min_dist], f32), max_dist=np.array([max_dist], f32))
    return dict(kf_kp=_kp([uv], octave=main_oct - octave_diff), matches_idx_mp=np.zeros(1, np.int32), Tcw_new=Tn, mp=mp,
                Tcw_table=np.stack([T0, Tn]), K=gs.K, lower=f32(lower), upper=f32(upper), fx=gs.FX)


def projection_oracle(c):
    return pygeom.projection_observations(c["kf_kp"], c["matches_idx_mp"], c["Tcw_new"], c["mp"], c["Tcw_table"], c["K"],
                                          c["lower"], c["upper"], c["fx"])


def projection_accept(c):
    return bool(projection_oracle(c)[0][0])


def projection_pairs():
    pairs = []
    base = projection_case()
    pos = projection_oracle(base)[1][0]
    assert projection_accept(base)
    dist = f32(np.sqrt(f64(pos[0]) * f64(pos[0]) + f64(pos[1]) * f64(pos[1]) + f64(pos[2]) * f64(pos[2])))
    for sign in (1, -1):
        pairs.append(Pair("projection", f"c1_octave{'+' if sign > 0 else '-'}", "kf_kp.0.octave",
                          projection_case(octave_diff=2 * sign), projection_case(octave_diff=3 * sign)))
    nx = base["mp"]["normal"][0, 0]
    x0, x1 = bisect(lambda x: projection_accept(projection_case(normal_x=x)), nx, f32(nx + 2.0))
    pairs.append(Pair("projection", "c2_cos30", "mp.normal.0.0", _normal_set(x0), _normal_set(x1)))
    pairs.append(Pair("projection", "c3_min_dist", "mp.min_dist.0", projection_case(min_dist=dist),
                      projection_case(min_dist=up(dist))))
    pairs.append(Pair("projection", "c3_max_dist", "mp.max_dist.0", projection_case(max_dist=dist),
                      projection_case(max_dist=down(dist))))
    pairs.append(Pair("projection", "depth_lower", "lower", projection_case(lower=pos[2]), projection_case(lower=up(pos[2]))))
    pairs.append(Pair("projection", "depth_upper", "upper", projection_case(upper=pos[2]), projection_case(upper=down(pos[2]))))
    return pairs


def _normal_set(x):
    c = projection_case(normal_x=x)
    c["mp"]["normal"][0, 0] = x
    return c


# ------------------------------------------------------------------------------------------ updateParallax
def _tcw_at(x, z=0.0):
    """a camera at world (x, 0, z) looking along +z (camera axes = world axes)"""
    T = np.eye(4, dtype=f32)
    T[0, 3], T[2, 3] = -x, -z
    return T


def mp_case(ids, cams, q, X=(0.2, -0.1, 3.0), kp_dx=0.0, lower=gs.LOWER_DEPTH, upper=gs.UPPER_DEPTH, seed=0):
    """one map point observed once by each keyframe of `ids` (ids[j] = mIdKF of list entry j), camera j at world
    (cams[j][0], 0, cams[j][1]); the update inserts list position q. Keypoints are the exact projections of X; kp_dx shifts
    the x of entry q's keypoint. No good parallax yet, main keyframe entry 0."""
    rng = np.random.default_rng(seed)
    n = len(ids)
    Tcw = np.stack([_tcw_at(cx, cz) for cx, cz in cams])
    kp_base = (2 * np.arange(n)).astype(np.int32)
    slot = kp_base + 1
    kp = np.zeros(2 * n, gs.KP_DTYPE)
    kp["size"] = 31; kp["angle"] = -1; kp["class_id"] = -1
    X = np.asarray(X, f64)
    for j in range(n):
        uv = gs.project(gs.K.astype(f64) @ Tcw[j][:3].astype(f64), X).astype(f32)
        kp["x"][slot[j]], kp["y"][slot[j]] = uv
    kp["x"][slot[q]] = f32(kp["x"][slot[q]] + f32(kp_dx))
    desc = rng.integers(0, 256, (2 * n, 32), dtype=np.uint8)
    view_mp = np.zeros((2 * n, 3), f32)
    view_mp[slot] = [(Tcw[j][:3, :3].astype(f64) @ X + Tcw[j][:3, 3]).astype(f32) for j in range(n)]
    view_info = np.zeros((2 * n, 3, 3)); view_info[slot] = 100.0 * np.eye(3)
    kf = dict(kf_id=np.asarray(ids, np.int32), kf_null=np.zeros(n, np.uint8), Tcw=Tcw, kp_base=kp_base, kp=kp, desc=desc,
              view_mp=view_mp, view_info=view_info)
    d0 = f32(np.linalg.norm(view_mp[slot[0]].astype(f64)))
    nrm = (X / np.linalg.norm(X)).astype(f32)
    mp = dict(pos=X.astype(f32)[None].copy(), good_prl=np.zeros(1, np.uint8), null=np.zeros(1, np.uint8),
              main_kf=np.zeros(1, np.int32), main_desc=desc[slot[:1]].copy(), main_octave=np.zeros(1, np.int32),
              main_measure=np.array([[kp["x"][slot[0]], kp["y"][slot[0]]]], f32), level_scale=np.ones(1, f32),
              normal=nrm[None].copy(), min_dist=np.array([d0 / ms.SCALE_FACTORS[-1]], f32), max_dist=np.array([d0], f32),
              obs_ptr=np.array([0, n], np.int32), obs_kf=np.arange(n, dtype=np.int32), obs_idx=np.ones(n, np.int32))
    params = dict(K=gs.K, lower_depth=f32(lower), upper_depth=f32(upper), fx=gs.FX, scale_factors=ms.SCALE_FACTORS)
    return dict(kf=kf, mp=mp, upd_ptr=np.array([0, 1], np.int32), upd_pos=np.array([q], np.int32), params=params)


def mp_oracle(c):
    """the oracle's add; returns (kf, mp, abandoned) on copies of the tables"""
    kf, mp = ms.copy_tables(c)
    ab = pm.add_observations(kf, mp, c["upd_ptr"], c["upd_pos"], c["params"])
    return kf, mp, ab


def mp_restated(c):
    """the numpy restatement's add; returns (kf, mp, abandoned, restatement) with its trace and pKF0 choices"""
    kf, mp = ms.copy_tables(c)
    r = mpn.Restatement(kf, mp, c["params"])
    ab = r.add(c["upd_ptr"], c["upd_pos"])
    return kf, mp, ab, r


def mp_decisions(c):
    """(re-triangulated with good parallax, abandoned)"""
    _, mp, ab = mp_oracle(c)
    return bool(mp["good_prl"][0]), bool(ab[0])


# The list of the pKF0 and abandonment cases: entry 0 is the candidate `d` ids older than pKF (entry q = 3), entry 1 is 3
# ids older, entry 2 two ids later. Wide baselines re-triangulate; baselines of a millimetre fail the parallax test.
IDN = 20


def _window_case(d, wide):
    ids = [IDN - d, IDN - 3, IDN + 2, IDN]
    s = 1.0 if wide else 1e-3
    cams = [(-0.6 * s, 0.0), (-0.3 * s, 0.0), (0.2 * s, 0.0), (0.0, 0.0)]
    return mp_case(ids, cams, q=3)


def mp_pairs():
    pairs = []
    # depth of pos0 and pos1 at both ends: pKF0 (entry 0) behind pKF (entry 2) along the optical axis, so z0 > z1; and
    # the same list with the cameras' order along the axis reversed, z0 < z1
    for name, cams in (("z0_gt_z1", [(-0.5, -0.8), (-0.2, -0.4), (0.0, 0.0)]), ("z0_lt_z1", [(-0.5, 0.8), (-0.2, 0.4), (0.0, 0.0)])):
        ids = [IDN - 4, IDN - 2, IDN]
        wide = mp_case(ids, cams, q=2, lower=WIDE[0], upper=WIDE[1])
        kf, mp, _ = mp_oracle(wide)
        assert mp["good_prl"][0] == 1
        z0 = kf["view_mp"][1, 2]; z1 = kf["view_mp"][5, 2]
        lo_who, hi_who = ("pos1", "pos0") if z0 > z1 else ("pos0", "pos1")
        zlo, zhi = min(z0, z1), max(z0, z1)
        mk = lambda lo=gs.LOWER_DEPTH, hi=gs.UPPER_DEPTH: mp_case(ids, cams, q=2, lower=lo, upper=hi)
        pairs.append(Pair("mp", f"depth_lower_{lo_who}", "params.lower_depth", mk(lo=zlo), mk(lo=up(zlo))))
        pairs.append(Pair("mp", f"depth_upper_{hi_who}", "params.upper_depth", mk(hi=zhi), mk(hi=down(zhi))))
    # parallax: shift pKF's keypoint along its row from a wide-baseline pair towards the direction of a zero-baseline one
    ids = [IDN - 4, IDN - 2, IDN]
    cams = [(-0.3, 0.0), (-0.15, 0.0), (0.0, 0.0)]
    mk = lambda dx: mp_case(ids, cams, q=2, kp_dx=dx, upper=100.0)
    x0, x1 = bisect(lambda dx: mp_decisions(mk(dx))[0], f32(0.0), _no_parallax_shift(mk))
    pairs.append(Pair("mp", "parallax", "kf.kp.5.x", mk(x0), mk(x1)))          # slot 5: entry 2's keypoint
    # pKF0: the candidate 6 ids older is chosen, 7 ids older it is not (a later keyframe is in the list)
    pairs.append(Pair("mp", "pkf0_window", "kf.kf_id.0", _window_case(6, True), _window_case(7, True)))
    # abandonment without good parallax: pKF0 6 ids older abandons, 5 older does not, 7 older is out of the window
    pairs.append(Pair("mp", "abandon_6_vs_5", "kf.kf_id.0", _window_case(6, False), _window_case(5, False)))
    pairs.append(Pair("mp", "abandon_6_vs_7", "kf.kf_id.0", _window_case(6, False), _window_case(7, False)))
    return pairs


def _no_parallax_shift(mk):
    """a shift of pKF's keypoint (pixels) that leaves the two rays meeting far away, where the parallax cosine is near 1"""
    for dx in (16.0, 18.0, 20.0, 22.0, -16.0, -18.0, -20.0, -22.0):
        good, _ = mp_decisions(mk(f32(dx)))
        if not good:
            return f32(dx)
    raise AssertionError("no shift rejects the parallax")


def all_pairs():
    return track_pairs() + projection_pairs() + mp_pairs()
