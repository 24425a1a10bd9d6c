"""CPU: matcher oracle against independent brute-force restatements in numpy."""
import numpy as np
import pytest

from oracle import pyoracle
from tests.matcher_cases import (GRID, UNDIST_BOUNDS, UNDIST_GRID, brute_candidates, grid_pos, half_cell_coords, make_bow_case,
                                 make_frame_pair, make_grid_edge_pair, make_projection_case, make_projection_edge_case)


def test_descriptor_distance_is_popcount():
    rng = np.random.default_rng(0)
    for _ in range(200):
        a = rng.integers(0, 256, 32, dtype=np.uint8); b = rng.integers(0, 256, 32, dtype=np.uint8)
        assert pyoracle.descriptor_distance(a, b) == int(np.unpackbits(a ^ b).sum())


def brute_match_by_window(kp1, d1, kp2, d2, prev, grid, win, ratio):
    """Brute-force greedy MatchByWindow with the reference's semantics, candidates from an explicit grid walk."""
    vdist = np.full(len(kp2), np.iinfo(np.int32).max, np.int64); m21 = -np.ones(len(kp2), int); m12 = -np.ones(len(kp1), int)
    hist = [[] for _ in range(30)]
    for i1 in range(len(kp1)):
        lvl = int(kp1["octave"][i1])
        cand = brute_candidates(kp2, prev[i1, 0], prev[i1, 1], win, max(lvl - 1, 0), lvl + 1, grid)
        best = best2 = 1 << 31; bi = -1
        for i2 in cand:
            dist = int(np.unpackbits(d1[i1] ^ d2[i2]).sum())
            if vdist[i2] <= dist:
                continue
            if dist < best:
                best2, best, bi = best, dist, i2
            elif dist < best2:
                best2 = dist
        if best <= 75 and best < np.float32(best2) * np.float32(ratio):
            if m21[bi] >= 0:
                m12[m21[bi]] = -1
            m12[i1] = bi; m21[bi] = i1; vdist[bi] = best
            rot = np.float32(kp1["angle"][i1]) - np.float32(kp2["angle"][bi])
            if rot < 0:
                rot = np.float32(rot + np.float32(360))
            b = int(np.floor(np.float32(rot * np.float32(30.0 / 360.0)) + 0.5))
            hist[0 if b == 30 else b].append(i1)
    sizes = [len(h) for h in hist]
    order = sorted(range(30), key=lambda i: (-sizes[i], i))
    top = [order[0]]
    if sizes[order[1]] >= 0.1 * sizes[order[0]]:
        top.append(order[1])
        if sizes[order[2]] >= 0.1 * sizes[order[0]]:
            top.append(order[2])
    for b in range(30):
        if b not in top:
            for i1 in hist[b]:
                m12[i1] = -1
    prev_out = prev.copy()
    for i1 in np.flatnonzero(m12 >= 0):
        prev_out[i1] = kp2["x"][m12[i1]], kp2["y"][m12[i1]]
    return int((m12 >= 0).sum()), m12, prev_out


def test_match_by_window_against_bruteforce():
    f1, f2, prev = make_frame_pair(seed=1)
    n, m, prev_out = pyoracle.match_by_window(f1["kp"], f1["desc"], f2["kp"], f2["desc"], prev, GRID, 20, 1, 0, 8, 0.9)
    n_b, m12, prev_b = brute_match_by_window(f1["kp"], f1["desc"], f2["kp"], f2["desc"], prev, GRID, 20.0, 0.9)
    assert n == n_b and n > 50
    np.testing.assert_array_equal(m, m12)
    np.testing.assert_array_equal(prev_out, prev_b)


def _popcount(a, b):
    return int(np.unpackbits(a ^ b).sum())


def _keep_top3_bins(hist):
    """ComputeThreeMaxima (ORBmatcher.cpp:64-105): three fullest bins, earlier bin wins ties, 10 % rule."""
    sizes = [len(h) for h in hist]
    order = sorted(range(len(hist)), key=lambda i: (-sizes[i], i))
    top = [order[0]] if sizes[order[0]] > 0 else []
    if top and sizes[order[1]] > 0 and not (sizes[order[1]] < np.float32(0.1) * np.float32(sizes[order[0]])):
        top.append(order[1])
        if sizes[order[2]] > 0 and not (sizes[order[2]] < np.float32(0.1) * np.float32(sizes[order[0]])):
            top.append(order[2])
    return top


def brute_match_by_projection(a):
    """Independent numpy restatement of ORBmatcher::MatchByProjection (ORBmatcher.cpp:383-454): explicit grid walk for
    GetFeaturesInArea, window = mMainOctave * winSize (0 px for octave 0), same-level ratio rule, TH_HIGH, steal."""
    kp, desc = a["kfkp"], a["kfdesc"]
    ratio = np.float32(a["nnratio"])
    INT_MAX = np.iinfo(np.int32).max
    vdist = np.full(len(kp), INT_MAX, np.int64)
    out = -np.ones(len(kp), int)
    nm = 0
    for i in range(len(a["mp_valid"])):
        if not a["mp_valid"][i]:
            continue
        pl = int(a["mp_octave"][i])
        lo = a["level_offset"]
        cand = brute_candidates(kp, a["mp_uv"][i, 0], a["mp_uv"][i, 1], float(pl * a["win_size"]), pl - lo if pl > lo else 0, pl + lo,
                                a["grid"])
        if not cand:
            continue
        best = best2 = INT_MAX
        lvl = lvl2 = bi = -1
        for idx in cand:
            if a["kf_observed"][idx]:
                continue
            dist = _popcount(a["mp_desc"][i], desc[idx])
            if vdist[idx] <= dist:
                continue
            if dist < best:
                best2, lvl2 = best, lvl
                best, lvl, bi = dist, int(kp["octave"][idx]), idx
            elif dist < best2:
                best2, lvl2 = dist, int(kp["octave"][idx])
        if best <= 100:
            if lvl == lvl2 and np.float32(best) > ratio * np.float32(best2):
                continue
            if out[bi] >= 0:
                out[bi] = -1; nm -= 1
            out[bi] = i; vdist[bi] = best; nm += 1
    return nm, out


@pytest.mark.parametrize("seed", [2, 7, 11])
def test_match_by_projection_against_bruteforce(seed):
    a = make_projection_case(seed=seed)["args"]
    n, m = pyoracle.match_by_projection(**a)
    nm, out = brute_match_by_projection(a)
    assert n == nm and n > 20
    np.testing.assert_array_equal(m, out)
    assert not np.any(a["kf_observed"].astype(bool) & (m >= 0))


def test_grid_pos_rounds_half_away_from_zero():
    """PosInGrid uses C++ round() of the float32 product: -0.5 cells -> -1 (outside), 1.5 -> 2, 2.5 -> 3 (round-half-even would
    give 2), 63.5 -> 64 and 47.5 -> 48 (outside)."""
    minX, minY, invW, invH = UNDIST_GRID
    hx = half_cell_coords(minX, invW, [-0.5, 1.5, 2.5, 63.5])
    hy = half_cell_coords(minY, invH, [-0.5, 2.5, 47.5])
    kp = np.zeros(len(hx) + len(hy), pyoracle.KP_DTYPE)
    kp["x"][:len(hx)], kp["y"][:len(hx)] = list(hx.values()), minY + 100
    kp["x"][len(hx):], kp["y"][len(hx):] = minX + 100, list(hy.values())
    px, py, inside = grid_pos(kp, UNDIST_GRID)
    np.testing.assert_array_equal(px[:len(hx)], [int(np.floor(h)) + 1 if h > 0 else -1 for h in hx])
    np.testing.assert_array_equal(py[len(hx):], [int(np.floor(h)) + 1 if h > 0 else -1 for h in hy])
    assert list(inside) == [h not in (-0.5, 63.5) for h in hx] + [h not in (-0.5, 47.5) for h in hy]
    assert set(hx) == {-0.5, 1.5, 2.5, 63.5} and set(hy) == {-0.5, 2.5, 47.5}


@pytest.mark.parametrize("seed", [21, 23])
def test_match_by_window_against_bruteforce_on_grid_edges(seed):
    """Non-zero origin, non-round cells (undistorted bounds), keypoints outside the grid and on half cells, windows outside."""
    f1, f2, prev, q = make_grid_edge_pair(seed=seed)
    kp2 = f2["kp"]
    _, _, inside = grid_pos(kp2, UNDIST_GRID)
    assert (kp2["x"] < 0).any() and (kp2["x"] >= UNDIST_BOUNDS[2]).any() and (kp2["y"] >= UNDIST_BOUNDS[3]).any() and (~inside).sum() > 50
    for i in q["empty"]:
        assert brute_candidates(kp2, prev[i, 0], prev[i, 1], 20.0, -1, -1, UNDIST_GRID) == []
    n, m, prev_out = pyoracle.match_by_window(f1["kp"], f1["desc"], kp2, f2["desc"], prev, UNDIST_GRID, 20, 1, 0, 8, 0.9)
    n_b, m12, prev_b = brute_match_by_window(f1["kp"], f1["desc"], kp2, f2["desc"], prev, UNDIST_GRID, 20.0, 0.9)
    assert n == n_b and n > 300
    np.testing.assert_array_equal(m, m12)
    np.testing.assert_array_equal(prev_out, prev_b)
    assert inside[m[m >= 0]].all()            # nothing outside the grid is ever matched
    assert (m[q["empty"]] == -1).all()


@pytest.mark.parametrize("seed", [22, 24])
def test_match_by_projection_against_bruteforce_on_grid_edges(seed):
    c = make_projection_edge_case(seed=seed)
    a = c["args"]
    n, m = pyoracle.match_by_projection(**a)
    nm, out = brute_match_by_projection(a)
    assert n == nm and n > 150
    np.testing.assert_array_equal(m, out)
    _, _, inside = grid_pos(a["kfkp"], a["grid"])
    assert inside[m >= 0].all()
    # the grid walk's order decides every tie: the lower index B, visited first, takes the map point
    for (b, a_), mp in zip(c["ties"], c["tie_mps"]):
        assert m[b] == mp and m[a_] == -1, (b, a_, mp)


@pytest.mark.parametrize("seed,mp_only,ori", [(3, True, True), (8, False, True), (9, True, False), (12, False, False)])
def test_search_by_bow_against_bruteforce(seed, mp_only, ori):
    """Independent numpy restatement of ORBmatcher::SearchByBoW (ORBmatcher.cpp:128-276) over dict feature vectors."""
    k1, k2 = make_bow_case(seed=seed)
    n, m = pyoracle.search_by_bow(k1, k2, mp_only, 0.6, ori)
    fv1 = {int(nd): k1["feat"][k1["ptr"][i]:k1["ptr"][i + 1]].tolist() for i, nd in enumerate(k1["node"])}
    fv2 = {int(nd): k2["feat"][k2["ptr"][i]:k2["ptr"][i + 1]].tolist() for i, nd in enumerate(k2["node"])}
    matched2 = np.zeros(len(k2["desc"]), bool)
    mm = {}
    hist = [[] for _ in range(30)]
    ratio = np.float32(0.6)
    INT_MAX = np.iinfo(np.int32).max
    nm = 0
    for nd in sorted(set(fv1) & set(fv2)):          # the two-iterator walk visits exactly the common node ids, ascending
        for idx1 in fv1[nd]:
            if mp_only and not k1["has_mp"][idx1]:
                continue
            best = best2 = INT_MAX
            bi = -1
            for idx2 in fv2[nd]:
                if mp_only and not k2["has_mp"][idx2]:
                    continue
                if matched2[idx2]:
                    continue
                dist = _popcount(k1["desc"][idx1], k2["desc"][idx2])
                if dist < best:
                    best2, best, bi = best, dist, idx2
                elif dist < best2:
                    best2 = dist
            if best < 75 and np.float32(best) < ratio * np.float32(best2):
                mm[idx1] = bi; matched2[bi] = True
                if ori:
                    rot = np.float32(k1["angle"][idx1]) - np.float32(k2["angle"][bi])
                    if rot < 0:
                        rot = np.float32(rot + np.float32(360))
                    b = int(np.floor(np.float32(rot * np.float32(30.0 / 360.0)) + 0.5))
                    hist[0 if b == 30 else b].append(idx1)
                nm += 1
    if ori:
        top = _keep_top3_bins(hist)
        for b in range(30):
            if b not in top:
                for idx1 in hist[b]:
                    mm.pop(idx1, None); nm -= 1
    ref = -np.ones(len(k1["desc"]), int)
    for i1, i2 in mm.items():
        ref[i1] = i2
    assert n == nm and n > 20
    np.testing.assert_array_equal(m, ref)
    got = m[m >= 0]
    assert len(np.unique(got)) == len(got)        # vbMatched2: one-to-one
