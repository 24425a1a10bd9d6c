"""The depth, parallax and acceptNewObserve decisions at their thresholds, on the oracles (no GPU).

tests/geom_boundaries.py builds pairs of inputs that differ in one value and sit on the two sides of one comparison. Here
each pair is checked three ways: the two inputs differ in that value alone; the oracle's decisions differ in the targeted
one alone; and an independent numpy restatement of that one comparison, written as the reference writes it, straddles the
threshold on the oracle's own intermediate values. Run with -s to see every pair and the bit patterns of its two sides.

The second half holds the map-point scenes of tests/mappoint_cases.py that the random families never build (long update
runs, erasure of the main keyframe down to an empty list, long lists with null keyframes, other pyramid level counts) to
the numpy restatement, and checks that they reach the branch events they were built for."""
import numpy as np
import pytest

from oracle import pygeom
from tests import geom_boundaries as gb
from tests import mappoint_cases as mc
from tests.test_mappoint_oracle import run_both, same_tables

f32, f64 = np.float32, np.float64


@pytest.fixture(scope="module")
def pairs():
    return gb.all_pairs()


def by_kind(pairs, kind):
    return [p for p in pairs if p.kind == kind]


def leaves(d, prefix=""):
    out = {}
    for k, v in d.items():
        if isinstance(v, dict):
            out.update(leaves(v, prefix + k + "."))
        else:
            out[prefix + k] = np.asarray(v)
    return out


def differing(a, b):
    """the paths (array path, flat index) at which two argument dicts differ"""
    la, lb = leaves(a), leaves(b)
    assert la.keys() == lb.keys()
    out = []
    for k in la:
        x, y = la[k], lb[k]
        assert x.dtype == y.dtype and x.shape == y.shape, k
        if x.dtype.names:
            for i in range(len(x)):
                out += [f"{k}.{i}.{name}" for name in x.dtype.names if x[i][name].tobytes() != y[i][name].tobytes()]
        elif x.ndim == 0:
            if x.tobytes() != y.tobytes():
                out.append(k)
        else:
            xs = x.reshape(x.shape[0], -1) if x.ndim > 1 else x.reshape(-1, 1)
            ys = y.reshape(y.shape[0], -1) if y.ndim > 1 else y.reshape(-1, 1)
            for i in range(xs.shape[0]):
                for j in range(xs.shape[1]):
                    if xs[i, j].tobytes() != ys[i, j].tobytes():
                        out.append(f"{k}.{i}" + (f".{j}" if x.ndim > 1 else ""))
    return out


# ------------------------------------------------------------------------------------------ restatements of one comparison
def norm3(p):
    return np.sqrt(f64(p[0]) * f64(p[0]) + f64(p[1]) * f64(p[1]) + f64(p[2]) * f64(p[2]))


def dot_f(a, b):
    return f32(f32(f32(a[0]) * f32(b[0]) + f32(a[1]) * f32(b[1])) + f32(a[2]) * f32(b[2]))


def cos_parallax(o1, o2, p):
    """cvutil.cpp:92-98: Point3f differences, the float dot product, the double norms, the double quotient rounded to float"""
    p1 = [f32(f32(p[k]) - f32(o1[k])) for k in range(3)]
    p2 = [f32(f32(p[k]) - f32(o2[k])) for k in range(3)]
    return f32(abs(f64(dot_f(p1, p2))) / (norm3(p1) * norm3(p2)))


def cos_normal(pos, nv):
    """MapPoint.cpp:203-204: float dist = cv::norm(posKF); cv::norm(posKF.dot(n)) / (dist * cv::norm(n)) in double"""
    dist = f32(norm3(pos))
    return f32(abs(f64(dot_f(pos, nv))) / (f64(dist) * norm3(nv))), dist


def accept_depth(z, lo, hi):
    """Config.cpp:188-190, inclusive at both ends"""
    return bool(f32(z) >= f32(lo) and f32(z) <= f32(hi))


# ------------------------------------------------------------------------------------------ every pair
def test_pairs_are_adjacent_and_printed(pairs):
    assert {p.kind for p in pairs} == {"track", "projection", "mp"}
    assert len(pairs) == 21
    for p in pairs:
        print(p.describe())
        va, vb = p.values
        assert differing(p.a, p.b) == [p.field], p
        if isinstance(va, np.floating):
            assert abs(gb.key(va) - gb.key(vb)) == 1, p


def test_track_pairs(pairs):
    ps = by_kind(pairs, "track")
    assert [p.what for p in ps] == ["depth_lower", "depth_upper"] + [f"parallax_deg{d}" for d in (1, 2, 3, 4)]
    for p in ps:
        (m_a, lm_a, g_a, _), (m_b, lm_b, g_b, _) = gb.track_oracle(p.a), gb.track_oracle(p.b)
        if p.what.startswith("depth"):
            # accepted on side a, rejected on side b; the position is the same triangulation on both sides
            assert m_a[0] == 0 and m_b[0] == -1, p
            assert lm_b.tobytes() == p.b["local_mps"].tobytes() and not g_b[0]
            z = lm_a[0, 2]
            assert accept_depth(z, p.a["lower"], p.a["upper"]) and not accept_depth(z, p.b["lower"], p.b["upper"])
        else:
            deg = int(p.what[-1])
            assert m_a[0] == 0 and m_b[0] == 0, p
            assert accept_depth(lm_a[0, 2], p.a["lower"], p.a["upper"]) and accept_depth(lm_b[0, 2], p.b["lower"], p.b["upper"])
            assert g_a[0] != g_b[0], p
            O = pygeom.inv(p.a["Tcr"])[:3, 3]
            ca, cb = cos_parallax(np.zeros(3, f32), O, lm_a[0]), cos_parallax(np.zeros(3, f32), O, lm_b[0])
            assert (ca < gb.MIN_COS[deg - 1]) == bool(g_a[0]) and (cb < gb.MIN_COS[deg - 1]) == bool(g_b[0]), p
            assert min(ca, cb) < gb.MIN_COS[deg - 1] <= max(ca, cb)
            print(p.what, "cos", gb.bits(ca), gb.bits(cb), "threshold", gb.bits(gb.MIN_COS[deg - 1]))


def test_track_parallax_pairs_differ_between_degrees(pairs):
    """each degree's pair sits at its own threshold: the neighbouring degrees decide both of its sides alike"""
    ps = {p.what: p for p in by_kind(pairs, "track")}
    for deg in (1, 2, 3, 4):
        p = ps[f"parallax_deg{deg}"]
        for other in {1, 2, 3, 4} - {deg}:
            da = gb.track_decisions(dict(p.a, deg=other)); db = gb.track_decisions(dict(p.b, deg=other))
            assert da == db, (deg, other)


def test_projection_pairs(pairs):
    ps = by_kind(pairs, "projection")
    assert [p.what for p in ps] == ["c1_octave+", "c1_octave-", "c2_cos30", "c3_min_dist", "c3_max_dist", "depth_lower",
                                    "depth_upper"]
    for p in ps:
        acc_a, pos_a, _ = gb.projection_oracle(p.a)
        acc_b, pos_b, _ = gb.projection_oracle(p.b)
        assert acc_a[0] == 1 and acc_b[0] == 0, p
        assert not pos_b.any()                       # written only where accepted
        pos = pos_a[0]                               # the triangulation is the same on both sides
        conds = []
        for side in (p.a, p.b):
            mp = side["mp"]
            cos, dist = cos_normal(pos, mp["normal"][0])
            conds.append(dict(c1=abs(int(mp["main_octave"][0]) - int(side["kf_kp"]["octave"][0])) <= 2,
                              c2=bool(cos >= gb.COS30),
                              c3=bool(dist >= mp["min_dist"][0] and dist <= mp["max_dist"][0]),
                              depth=accept_depth(pos[2], side["lower"], side["upper"])))
        target = p.what.split("_")[0]
        assert all(conds[0].values()), p
        assert [k for k in conds[1] if not conds[1][k]] == [target], p
        if target == "c2":
            ca, _ = cos_normal(pos, p.a["mp"]["normal"][0]); cb, _ = cos_normal(pos, p.b["mp"]["normal"][0])
            print(p.what, "cos", gb.bits(ca), gb.bits(cb), "threshold", gb.bits(gb.COS30))
    oct_a = [p for p in ps if p.what.startswith("c1")]
    assert sorted(int(p.a["mp"]["main_octave"][0]) - int(p.a["kf_kp"]["octave"][0]) for p in oct_a) == [-2, 2]
    assert sorted(int(p.b["mp"]["main_octave"][0]) - int(p.b["kf_kp"]["octave"][0]) for p in oct_a) == [-3, 3]


def test_mp_pairs(pairs):
    ps = by_kind(pairs, "mp")
    assert sorted(p.what for p in ps) == sorted(["depth_lower_pos1", "depth_upper_pos0", "depth_lower_pos0", "depth_upper_pos1",
                                                 "parallax", "pkf0_window", "abandon_6_vs_5", "abandon_6_vs_7"])
    for p in ps:
        res = []
        for side in (p.a, p.b):
            kf_o, mp_o, ab_o = gb.mp_oracle(side)
            kf_n, mp_n, ab_n, r = gb.mp_restated(side)
            assert not same_tables(kf_o, kf_n) and not same_tables(mp_o, mp_n) and np.array_equal(ab_o, ab_n), p
            res.append((bool(mp_o["good_prl"][0]), bool(ab_o[0]), r.pkf0, kf_o, mp_o))
        (g_a, ab_a, c_a, kf_a, mp_a), (g_b, ab_b, c_b, _, _) = res
        ids = [list(p.a["kf"]["kf_id"]), list(p.b["kf"]["kf_id"])]
        if p.what.startswith("depth") or p.what == "parallax":
            assert (g_a, g_b, ab_a, ab_b) == (True, False, False, False), p
            assert c_a == c_b == [(0, 2, 0)]
        if p.what.startswith("depth"):
            who = p.what.split("_")[-1]
            z = kf_a["view_mp"][1 if who == "pos0" else 5, 2]          # setViewMP of pKF0 (slot 1) and pKF (slot 5)
            prm_a, prm_b = p.a["params"], p.b["params"]
            assert accept_depth(z, prm_a["lower_depth"], prm_a["upper_depth"])
            assert not accept_depth(z, prm_b["lower_depth"], prm_b["upper_depth"])
            other = kf_a["view_mp"][5 if who == "pos0" else 1, 2]
            assert accept_depth(other, prm_b["lower_depth"], prm_b["upper_depth"])
        if p.what == "parallax":
            cos = []
            for side in (p.a, p.b):
                kf = side["kf"]
                P = np.stack([pygeom.gemm3(side["params"]["K"], kf["Tcw"][j][:3]) for j in (0, 2)])
                pt = np.array([[kf["kp"]["x"][s], kf["kp"]["y"][s]] for s in (1, 5)], f32)
                posW = pygeom.triangulate(pt[:1], pt[1:], P, [0], [1])[0]
                cos.append(cos_parallax(pygeom.inv(kf["Tcw"][0])[:3, 3], pygeom.inv(kf["Tcw"][2])[:3, 3], posW))
                if side is p.a:
                    assert posW.tobytes() == mp_a["pos"][0].tobytes()
            assert cos[0] < gb.MIN_COS[1] <= cos[1]
            print(p.what, "cos", gb.bits(cos[0]), gb.bits(cos[1]), "threshold", gb.bits(gb.MIN_COS[1]))
        if p.what == "pkf0_window":
            # entry 0 is 6 ids older on side a, 7 on side b; both re-triangulate, against entry 0 and entry 1
            assert (g_a, g_b, ab_a, ab_b) == (True, True, False, False)
            assert c_a == [(0, 3, 0)] and c_b == [(0, 3, 1)]
            assert [gb.IDN - i <= 6 for i in (ids[0][0], ids[1][0])] == [True, False]
            assert ids[0][2] > gb.IDN and ids[1][2] > gb.IDN                    # a later keyframe is present
        if p.what.startswith("abandon"):
            assert (g_a, g_b, ab_a, ab_b) == (False, False, True, False), p
            id0 = [ids[k][c[0][2]] for k, c in ((0, c_a), (1, c_b))]
            assert [gb.IDN - i >= 6 for i in id0] == [True, False]
            assert c_a == [(0, 3, 0)] and c_b == ([(0, 3, 0)] if p.what.endswith("5") else [(0, 3, 1)])


# ------------------------------------------------------------------------------------------ map-point scenes
def events_of(sc, mode):
    (kf_o, mp_o, ab_o), (kf_n, mp_n, ab_n), ev = run_both(sc, mode)
    assert not same_tables(kf_o, kf_n) and not same_tables(mp_o, mp_n)
    assert np.array_equal(ab_o, ab_n)
    return ev


def test_many_updates_reach_parallax_on_a_rebuilt_list():
    sc = mc.many_updates_scene()
    n = np.diff(sc["upd_ptr"])
    assert n.min() >= 3 and n.max() == 8
    assert {"abandoned", "parallax_after_abandon", "triangulated", "parallax_rejected"} <= events_of(sc, "add")


def test_erase_runs_remove_the_main_keyframe_down_to_an_empty_list():
    from oracle import mappoint_numpy as mpn
    from tools import mappoint_scenes as ms
    sc = mc.erase_main_scene()
    kf, mp = ms.copy_tables(sc)
    r = mpn.Restatement(kf, mp, sc["params"])
    ab = r.erase(sc["upd_ptr"], sc["upd_pos"])
    per = {}
    for m, e in r.trace:
        per.setdefault(m, []).append(e)
    repeated = [m for m, ev in per.items() if ev.count("erase_main") >= 3 and "erased_to_empty" in ev]
    assert len(repeated) > 50 and ab[repeated].all()
    assert {"erase_main_changed", "null_kf_skipped"} <= events_of(sc, "erase")


@pytest.mark.parametrize("mode", ["add", "erase"])
def test_list_lengths_around_the_shared_memory_list(mode):
    """lists of 31 to 257 entries (the 1 000 and 4 000 entry lists run against the oracle alone, in the GPU tests)"""
    sc = mc.list_length_scene(mode, (31, 32, 33, 255, 256, 257))
    assert "short_median_of_long_list" in events_of(sc, mode)


@pytest.mark.parametrize("nlevels", mc.NLEVELS)
@pytest.mark.parametrize("mode", ["add", "erase"])
def test_other_level_counts(nlevels, mode):
    sc = mc.nlevels_scene(nlevels, mode)
    assert len(sc["params"]["scale_factors"]) == nlevels and sc["kf"]["kp"]["octave"].max() == nlevels - 1
    assert "range_of_other_nlevels" in events_of(sc, mode)
