"""The map-point update oracle (oracle/mappoint_oracle.cpp) against the numpy restatement (oracle/mappoint_numpy.py), bit
for bit on every table (NaNs compared as one canonical NaN), on seeded scenes that reach every branch of addObservation and
eraseObservation; and the pin of the OpenCV pieces the oracle restates."""
import os
import subprocess
import sys

import numpy as np
import pytest

from oracle import mappoint_numpy as mpn
from oracle import pymappoint as pm
from tests import mappoint_cases as mc
from tools import mappoint_scenes as ms

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def canon(a):
    a = np.array(a, copy=True)
    if a.dtype.kind == "f":
        a[np.isnan(a)] = np.nan
    return a.tobytes()


def same_tables(a, b):
    return [k for k in a if canon(a[k]) != canon(b[k])]


def run_both(sc, mode):
    kf_o, mp_o = ms.copy_tables(sc)
    kf_n, mp_n = ms.copy_tables(sc)
    r = mpn.Restatement(kf_n, mp_n, sc["params"])
    if mode == "add":
        ab_o = pm.add_observations(kf_o, mp_o, sc["upd_ptr"], sc["upd_pos"], sc["params"])
        ab_n = r.add(sc["upd_ptr"], sc["upd_pos"])
    else:
        ab_o = pm.erase_observations(kf_o, mp_o, sc["upd_ptr"], sc["upd_pos"], sc["params"])
        ab_n = r.erase(sc["upd_ptr"], sc["upd_pos"])
    return (kf_o, mp_o, ab_o), (kf_n, mp_n, ab_n), {e for _, e in r.trace}


def test_pin_against_cv2():
    pytest.importorskip("cv2")
    out = subprocess.run([sys.executable, os.path.join(ROOT, "oracle", "pin_mappoint_against_cv2.py")], capture_output=True, text=True)
    assert out.returncode == 0, out.stdout + out.stderr


@pytest.mark.parametrize("i", range(len(mc.add_scenes())))
def test_add_matches_numpy(i):
    _, sc = mc.add_scenes()[i]
    (kf_o, mp_o, ab_o), (kf_n, mp_n, ab_n), _ = run_both(sc, "add")
    assert not same_tables(kf_o, kf_n) and not same_tables(mp_o, mp_n)
    assert np.array_equal(ab_o, ab_n)


@pytest.mark.parametrize("i", range(len(mc.erase_scenes())))
def test_erase_matches_numpy(i):
    _, sc = mc.erase_scenes()[i]
    (kf_o, mp_o, ab_o), (kf_n, mp_n, ab_n), _ = run_both(sc, "erase")
    assert not same_tables(kf_o, kf_n) and not same_tables(mp_o, mp_n)
    assert np.array_equal(ab_o, ab_n)


def test_every_add_branch_is_reached():
    events = set()
    for _, sc in mc.add_scenes():
        events |= run_both(sc, "add")[2]
    assert mc.ADD_EVENTS <= events, mc.ADD_EVENTS - events


def test_every_erase_branch_is_reached():
    events = set()
    for _, sc in mc.erase_scenes():
        events |= run_both(sc, "erase")[2]
    assert mc.ERASE_EVENTS <= events, mc.ERASE_EVENTS - events


@pytest.mark.parametrize("mode", ["add", "erase"])
def test_long_lists_match_numpy(mode):
    sc = mc.long_scene(mode)
    (kf_o, mp_o, ab_o), (kf_n, mp_n, ab_n), _ = run_both(sc, mode)
    assert not same_tables(kf_o, kf_n) and not same_tables(mp_o, mp_n)
    assert np.array_equal(ab_o, ab_n)


def test_abandoned_point_ends_non_null_with_an_empty_list():
    """setNull inside updateParallax, then addObservation's final mbNull = false (MapPoint.cpp:119-121)"""
    _, sc = mc.add_scenes()[1]
    kf, mp = ms.copy_tables(sc)
    ab = pm.add_observations(kf, mp, sc["upd_ptr"], sc["upd_pos"], sc["params"])
    assert ab.any()
    assert not mp["null"][ab].any() and not mp["good_prl"][ab].any()


def test_two_adds_in_one_call_equal_two_single_calls():
    """findCorrespd's third loop: addObservation(pPrefKF) then addObservation(mNewKF) in one call"""
    _, sc = mc.add_scenes()[0]
    assert (np.diff(sc["upd_ptr"]) == 2).any()
    kf1, mp1 = ms.copy_tables(sc)
    ab1 = pm.add_observations(kf1, mp1, sc["upd_ptr"], sc["upd_pos"], sc["params"])
    (ptr, okf, oidx, u1p, u1), (u2p, u2) = mc.split_updates(sc)
    kf2, mp2 = ms.copy_tables(sc)
    first = dict(mp2, obs_ptr=ptr, obs_kf=okf, obs_idx=oidx)
    ab_a = pm.add_observations(kf2, first, u1p, u1, sc["params"])
    mp2 = {k: (first[k] if k not in ("obs_ptr", "obs_kf", "obs_idx") else mp2[k]) for k in mp2}
    ab_b = pm.add_observations(kf2, mp2, u2p, u2, sc["params"])
    two = np.diff(sc["upd_ptr"]) == 2
    # a point the first call abandons starts its second insertion from an empty list, which two calls over the same
    # flattened list cannot express: those are compared by the one-call path only
    sel = two & ~ab_a
    for k in mp1:
        if k in ("obs_ptr", "obs_kf", "obs_idx"):
            continue
        assert canon(mp1[k][sel]) == canon(mp2[k][sel]), k
    assert np.array_equal(ab1[sel], (ab_a | ab_b)[sel])


def test_update_measure_matches_numpy():
    sc = ms.scene(500, seed=401)
    pts = np.arange(0, 500, 3, dtype=np.int32)
    kf_o, mp_o = ms.copy_tables(sc)
    kf_n, mp_n = ms.copy_tables(sc)
    pm.update_measure(kf_o, mp_o, pts)
    mpn.Restatement(kf_n, mp_n, sc["params"]).update_measure(pts)
    assert not same_tables(kf_o, kf_n)
    assert canon(kf_o["view_mp"]) != canon(sc["kf"]["view_mp"])


def test_host_entries_check_their_input_before_the_device():
    """malformed tables are SE2GPU_ERR_INVALID whether or not a device is present, and nothing is written"""
    from se2lam_b200 import _capi, build, mappoint
    build.build_lib()
    sc = ms.scene(40, seed=701)
    bad = sc["upd_pos"].copy(); bad[0] = 10 ** 6
    kf, mp = ms.copy_tables(sc)
    with pytest.raises(_capi.Se2GpuError, match="-3"):
        mappoint.MapPoints(kf, mp, **sc["params"]).addObservation(sc["upd_ptr"], bad)
    assert not same_tables(kf, sc["kf"]) and not same_tables(mp, sc["mp"])
    with pytest.raises(_capi.Se2GpuError, match="-3"):
        mappoint.MapPoints(kf, mp, **sc["params"]).updateMeasureInKFs([40])
