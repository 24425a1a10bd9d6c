"""Host parts of the localization handle (no GPU): UpdatePoseCurr's pose composition against the oracle's restatement bit
for bit, and the map validation se2gpu_loc_create runs before it touches a device."""
import ctypes as C

import numpy as np
import pytest

from oracle import pyloc, pytrack
from tools import loc_scenes as ls
from tools import track_scenes as ts


def _cfg():
    c = ts.config()
    c.update(bounds=(0.0, 320.0, 0.0, 240.0), huber=2.0, max_local_mps=256)
    return c


def _params(c):
    from se2lam_b200 import loc
    return loc.params(c["nfeatures"], c["scale_factor"], c["nlevels"], c["K"], c["grid"], c["bounds"], c["cTb"], c["bTc"], c["huber"],
                      c["max_local_mps"])


@pytest.mark.parametrize("seed", range(6))
def test_host_pose_matches_oracle(seed):
    from se2lam_b200 import loc
    cfg = _cfg()
    p = _params(cfg)
    rng = np.random.default_rng(seed)
    T = ls.tcw(cfg, (0.3, -0.2, 0.4))
    for k in range(40):
        ref = rng.uniform(-2, 2, 3).astype(np.float32)
        if k % 5 == 0:                    # angle wrap at +-pi and near-zero motion
            ref[2] = np.float32(np.pi - 1e-4)
        odom = (ref + rng.normal(0, [0.05, 0.05, 0.02 if k % 7 else 1e-7])).astype(np.float32)
        if k % 5 == 0:
            odom[2] = np.float32(-np.pi + 1e-4)
        g = loc.host_pose(p, odom, ref, T)
        o = pyloc.host_pose(cfg, odom, ref, T)
        assert g.tobytes() == o.tobytes(), f"step {k}"
        T = g


@pytest.mark.parametrize("seed", range(3))
def test_numpy_pose_equals_cpp_oracle(seed):
    """UpdatePoseCurr restated in numpy float32 (oracle/loc_numpy.py) equals oracle/loc_oracle.cpp bit for bit"""
    from oracle import loc_numpy
    cfg = _cfg()
    rng = np.random.default_rng(100 + seed)
    T = ls.tcw(cfg, (0.1, 0.2, -0.3))
    for k in range(20):
        ref = rng.uniform(-3.5, 3.5, 3).astype(np.float32)
        odom = (ref + rng.normal(0, 0.05, 3)).astype(np.float32)
        a, b = pyloc.CppLogic.pose(cfg, odom, ref, T), loc_numpy.pose(cfg, odom, ref, T)
        assert a.tobytes() == b.tobytes(), f"step {k}"
        T = a


def _tiny_map():
    return dict(kf_Tcw=np.tile(np.eye(4, dtype=np.float32), (2, 1, 1)), kf_kp_ptr=np.array([0, 3, 5], np.int32),
                kf_obs_mp=np.array([0, -1, 1, 1, 2], np.int32), kf_obs_ptr=np.array([0, 2, 4], np.int32),
                kf_obs=np.array([0, 1, 1, 2], np.int32), kf_cov_ptr=np.array([0, 1, 2], np.int32), kf_cov=np.array([1, 0], np.int32),
                mp_pos=np.ones((3, 3), np.float32), mp_null=np.zeros(3, np.uint8), mp_good_prl=np.ones(3, np.uint8),
                mp_desc=np.zeros((3, 32), np.uint8), mp_octave=np.zeros(3, np.int32))


BAD = {
    "obs_mp out of range": ("kf_obs_mp", np.array([0, -1, 1, 1, 3], np.int32)),
    "obs_mp below -1": ("kf_obs_mp", np.array([0, -2, 1, 1, 2], np.int32)),
    "kp_ptr not monotone": ("kf_kp_ptr", np.array([0, 4, 3], np.int32)),
    "kp_ptr not from 0": ("kf_kp_ptr", np.array([1, 3, 5], np.int32)),
    "observations not ascending": ("kf_obs", np.array([1, 0, 1, 2], np.int32)),
    "observation out of range": ("kf_obs", np.array([0, 1, 1, 7], np.int32)),
    "covisibility out of range": ("kf_cov", np.array([1, 2], np.int32)),
    "octave past nlevels": ("mp_octave", np.array([0, 6, 0], np.int32)),
}


@pytest.mark.parametrize("case", sorted(BAD))
def test_malformed_maps_are_rejected(case):
    from se2lam_b200._capi import lib
    from se2lam_b200.loc import MAP_FIELDS, _map
    key, val = BAD[case]
    m = _tiny_map()
    m[key] = val
    cm, keep = _map({k: m[k] for k in MAP_FIELDS})
    L = lib()
    assert not L.se2gpu_loc_create(2, 320, 240, C.byref(_params(_cfg())), C.byref(cm), 0)
    msg = L.se2gpu_last_error().decode()
    assert "map" in msg or "CSR" in msg or "octave" in msg or "index" in msg, msg
    del keep


def test_bad_params_are_rejected():
    from se2lam_b200._capi import lib
    from se2lam_b200.loc import MAP_FIELDS, _map
    cm, keep = _map({k: v for k, v in _tiny_map().items() if k in MAP_FIELDS})
    for field, v in (("nlevels", 17), ("max_local_mps", 0), ("ndist", 3)):
        p = _params(_cfg())
        setattr(p, field, v)
        assert not lib().se2gpu_loc_create(2, 320, 240, C.byref(p), C.byref(cm), 0)
        assert "bad arguments" in lib().se2gpu_last_error().decode()
    del keep


# ---------------------------------------------------------------------------------------------- C++ oracle vs numpy
_MAP = {}


def _scene():
    if not _MAP:
        cfg = ls.config()
        _MAP.update(cfg=cfg, m=ls.build_map(3, cfg))
    return _MAP["cfg"], _MAP["m"]


@pytest.mark.parametrize("kind", ls.KINDS)
def test_cpp_oracle_equals_numpy_restatement_on_scene_families(kind):
    """Localizer::run over one stream of each family, once with oracle/loc_oracle.cpp's logic and once with
    oracle/loc_numpy.py's: every record, pose, observation and local set equal bit for bit"""
    from se2lam_b200.loc import inv_level_sigma2
    cfg, m = _scene()
    isig = inv_level_sigma2(cfg["scale_factor"], cfg["nlevels"])
    s = ls.stream(200 + ls.KINDS.index(kind), m, cfg, 30, kind)
    a, b = pyloc.LocOracle(cfg, m, isig, "cpp"), pyloc.LocOracle(cfg, m, isig, "numpy")
    for k in range(30):
        ra, rb = a.step(s[0][k], s[1][k]), b.step(s[0][k], s[1][k])
        if k == 1:
            pairs = ls.loop_matches(a.kp, a.desc, m, s[3])
            (ra, fa), (rb, fb) = a.relocalize(s[3], pairs), b.relocalize(s[3], pairs)
            assert fa.tobytes() == fb.tobytes()
        assert ra == rb, f"frame {k}: {ra} != {rb}"
        assert a.Tcw.tobytes() == b.Tcw.tobytes() and a.obs_mp.tobytes() == b.obs_mp.tobytes(), f"frame {k}"
        assert a.local_kfs == b.local_kfs and a.local_mps == b.local_mps and a.covis.tobytes() == b.covis.tobytes(), f"frame {k}"
    assert a.branches == b.branches
    assert {"first", "relocalized", "tracked", "loop_null", "loop_badprl", "loop_repeat"} <= set(a.branches), a.branches
    if kind == "leave":
        assert {"lost_now", "lost"} <= set(a.branches), a.branches
    if kind == "blank":
        assert "gated" in a.branches, a.branches


def test_set_logic_boundaries_cpp_equals_numpy():
    """the 0.1 covisibility threshold hit exactly (10 * count == getSizeObsMP: not covisible), one above it, and
    MatchLoopClose over null, not-good-parallax and repeated idxLoop entries"""
    from oracle import loc_numpy
    m = _tiny_map()
    m["kf_obs_ptr"] = np.array([0, 1, 3], np.int32); m["kf_obs"] = np.array([0, 0, 1], np.int32)
    cpp = pyloc.CppLogic(m)
    one = np.full(10, -1, np.int32); one[0] = 0          # one observed point, shared by both keyframes: 1 > 0.1
    ca, cb = np.zeros(2, np.uint8), np.zeros(2, np.uint8)
    ea = cpp.covis(m, np.ones(2, np.uint8), one, ca); eb = loc_numpy.covis(m, np.ones(2, np.uint8), one, cb)
    assert ca.tobytes() == cb.tobytes() and ea == eb == 0 and tuple(ca) == (1, 1)
    # ten observed points, keyframe 0 shares exactly one: 1 > 0.1 * 10 is false, the boundary
    big = _tiny_map()
    big["mp_pos"] = np.ones((12, 3), np.float32); big["mp_null"] = np.zeros(12, np.uint8); big["mp_good_prl"] = np.ones(12, np.uint8)
    big["mp_desc"] = np.zeros((12, 32), np.uint8); big["mp_octave"] = np.zeros(12, np.int32)
    big["kf_obs_ptr"] = np.array([0, 1, 3], np.int32); big["kf_obs"] = np.array([0, 0, 1], np.int32)
    cpp = pyloc.CppLogic(big)
    o = np.arange(10, dtype=np.int32)
    ca, cb = np.zeros(2, np.uint8), np.zeros(2, np.uint8)
    ea = cpp.covis(big, np.ones(2, np.uint8), o, ca); eb = loc_numpy.covis(big, np.ones(2, np.uint8), o, cb)
    assert ea == eb == 1 and ca.tobytes() == cb.tobytes() and tuple(ca) == (0, 1)
    # MatchLoopClose: slot 0 -> point 0 (null), slot 2 -> point 1 (no good parallax), slot 1 empty, slot 2 used twice
    lc = _tiny_map(); lc["mp_null"] = np.array([1, 0, 0], np.uint8); lc["mp_good_prl"] = np.array([1, 0, 1], np.uint8)
    cpp = pyloc.CppLogic(lc)
    pairs = [(0, 0), (1, 1), (3, 2), (4, 2)]
    oa, ob = np.full(6, -1, np.int32), np.full(6, -1, np.int32)
    assert cpp.loop_close(lc, 0, pairs, oa) == loc_numpy.loop_close(lc, 0, pairs, ob) == (1, 2)
    assert oa.tobytes() == ob.tobytes() and oa.tolist() == [-1, -1, -1, 1, 1, -1]


@pytest.mark.parametrize("n", sorted(ts.DISTORTION))
def test_oracle_extracts_from_the_undistorted_frame(n):
    """ReadFrameInfo builds a Frame, and Frame::Frame runs cv::undistort before extracting (reference Frame.cpp:22): with
    4, 5, 8 and 12 coefficients, LocOracle's keypoints and descriptors after one step are those of the undistorted frame"""
    from oracle import pyoracle
    from se2lam_b200.loc import inv_level_sigma2
    cfg = ls.config(dist=ts.DISTORTION[n])
    img = ts.stream(40 + n, 2, "normal", cfg)[0][0]
    o = pyloc.LocOracle(cfg, {"kf_kp_ptr": np.zeros(1, np.int32)}, inv_level_sigma2(cfg["scale_factor"], cfg["nlevels"]), "numpy")
    o.step(img, np.zeros(3, np.float32))
    orb = pyoracle.OrbOracle(cfg["nfeatures"], cfg["scale_factor"], cfg["nlevels"], cfg["fast_th"])
    kp, desc = orb.extract(pyoracle.undistort(img, cfg["K"], np.asarray(cfg["dist"], np.float32)))
    assert len(kp) > 100
    assert o.kp.tobytes() == kp.tobytes() and o.desc.tobytes() == desc.tobytes()
    raw, _ = orb.extract(img)                            # the distortion moves the keypoints: the comparison can tell
    assert raw.tobytes() != kp.tobytes()
