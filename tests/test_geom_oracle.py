"""CPU checks of the two-view geometry oracle: the cv2 fixture, ground-truth recovery on noise-free scenes, and the
depth / parallax / acceptNewObserve decisions against an independent numpy restatement away from their thresholds."""
import os

import numpy as np
import pytest

from oracle import pygeom
from tools import geom_scenes as gs

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "geom_golden.npz")


@pytest.fixture(scope="module")
def golden():
    return np.load(GOLDEN)


def test_svd_equals_cv2_fixture(golden):
    w, vt = pygeom.svd4(golden["svd_A"])
    assert w.tobytes() == golden["svd_w"].tobytes()
    assert vt.tobytes() == golden["svd_vt"].tobytes()


def test_degenerate_families_present(golden):
    assert set(np.unique(golden["svd_kind"])) == {0, 1, 2, 3, 4, 5}


def test_primitives_equal_cv2_fixture(golden):
    P = np.zeros((len(golden["row_x"]), 3, 4), np.float32)
    P[:, 0] = golden["row_P"][:, 0]; P[:, 2] = golden["row_P"][:, 1]
    rows = np.stack([pygeom.build_a(np.array([x, 0], np.float32), np.zeros(2, np.float32), p, p)[0]
                     for x, p in zip(golden["row_x"], P)])
    assert rows.tobytes() == golden["row_out"].tobytes()
    A, B = golden["gemm_A"], golden["gemm_B"]
    assert np.stack([pygeom.gemm3(a, b) for a, b in zip(A, B)]).tobytes() == golden["gemm_34"].tobytes()
    assert np.stack([pygeom.gemm3(a, b[:, 3:4], -1.0) for a, b in zip(A, B)]).tobytes() == golden["gemm_31"].tobytes()
    assert np.stack([pygeom.gemm3_at_b(a, d) for a, d in zip(A, golden["gemm_D"])]).tobytes() == golden["gemm_1T"].tobytes()
    assert np.stack([pygeom.rodrigues(v) for v in golden["rod_v"]]).tobytes() == golden["rod_R"].tobytes()


def test_inv_is_the_rigid_inverse():
    T = gs.pose_table(4, seed=3)[2]
    Ti = pygeom.inv(T)
    np.testing.assert_allclose(Ti.astype(np.float64) @ T.astype(np.float64), np.eye(4), atol=1e-5)


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_noise_free_triangulation_recovers_truth(seed):
    sc = gs.track_scene(300, seed=seed, noise=0.0, frac_matched=1.0, frac_observed=0.0, degenerate=False)
    m, lm, good, (n_old, n_good) = pygeom.track_triangulate(sc["kp_kf"], sc["kp_frame"], sc["matches12"], sc["kf_observed"],
                                                            sc["kf_view_mp"], sc["Tcr"], sc["K"], sc["lower"], sc["upper"], 2,
                                                            sc["local_mps"])
    assert n_old == 0 and (m >= 0).all()
    rel = np.linalg.norm(lm - sc["truth"], axis=1) / np.linalg.norm(sc["truth"], axis=1)
    assert np.median(rel) < 1e-4 and rel.max() < 2e-2


def test_triangulate_entry_recovers_world_points():
    sc = gs.triangulate_scene(200, seed=4, noise=0.0)
    keep = sc["idx1"] != sc["idx2"]
    xyz = pygeom.triangulate(sc["pt1"], sc["pt2"], sc["P"], sc["idx1"], sc["idx2"])
    rel = np.linalg.norm(xyz[keep] - sc["Xw"][keep], axis=1) / np.linalg.norm(sc["Xw"][keep], axis=1)
    assert np.median(rel) < 1e-4


def _np_cos_parallax(o1, o2, p):
    a = p.astype(np.float64) - o1; b = p.astype(np.float64) - o2
    return abs(a @ b) / (np.linalg.norm(a) * np.linalg.norm(b))


def test_parallax_decisions_match_numpy_away_from_threshold():
    rng = np.random.default_rng(5)
    checked = 0
    for _ in range(2000):
        o2 = rng.normal(0, 0.3, 3).astype(np.float32); p = (rng.normal(0, 3, 3) + [0, 0, 5]).astype(np.float32)
        c = _np_cos_parallax(np.zeros(3), o2.astype(np.float64), p)
        for deg, th in ((1, 0.9998), (2, 0.9994), (4, 0.9976)):
            if abs(c - th) < 1e-5:
                continue
            assert pygeom.check_parallax(np.zeros(3, np.float32), o2, p, deg) == (c < th)
            checked += 1
    assert checked > 5000


def test_depth_decisions_match_numpy():
    sc = gs.track_scene(1000, seed=6)
    m, lm, good, _ = pygeom.track_triangulate(sc["kp_kf"], sc["kp_frame"], sc["matches12"], sc["kf_observed"], sc["kf_view_mp"],
                                              sc["Tcr"], sc["K"], sc["lower"], sc["upper"], 2, sc["local_mps"])
    tri = (sc["matches12"] >= 0) & (sc["kf_observed"] == 0)
    # an independent float64 triangulation (numpy SVD) decides the same away from the depth window's edges
    P0 = sc["K"].astype(np.float64) @ np.eye(3, 4); P1 = sc["K"].astype(np.float64) @ sc["Tcr"][:3].astype(np.float64)
    agree = total = 0
    for i in np.flatnonzero(tri):
        a = sc["kp_kf"][i]; b = sc["kp_frame"][sc["matches12"][i]]
        A = np.stack([a["x"] * P0[2] - P0[0], a["y"] * P0[2] - P0[1], b["x"] * P1[2] - P1[0], b["y"] * P1[2] - P1[1]])
        X = np.linalg.svd(A)[2][3]
        z = X[2] / X[3]
        if not np.isfinite(z) or min(abs(z - sc["lower"]), abs(z - sc["upper"])) < 1e-2 * max(1.0, abs(z)):
            continue
        total += 1
        agree += (m[i] >= 0) == (sc["lower"] <= z <= sc["upper"])
    assert total > 500 and agree == total
    # untouched: unmatched entries, and depth failures keep their previous local_mps
    keep = (sc["matches12"] < 0) | (tri & (m < 0))
    assert lm[keep].tobytes() == sc["local_mps"][keep].tobytes()
    obs = (sc["matches12"] >= 0) & (sc["kf_observed"] == 1)
    assert lm[obs].tobytes() == sc["kf_view_mp"][obs].tobytes()
    assert not good[~tri].any()


def test_accept_new_observe_matches_numpy_away_from_thresholds():
    rng = np.random.default_rng(8)
    checked = 0
    for _ in range(3000):
        pos = (rng.normal(0, 2, 3) + [0, 0, 4]).astype(np.float32)
        nv = rng.normal(0, 1, 3); nv = (nv / np.linalg.norm(nv) * 0.3 + pos / np.linalg.norm(pos)).astype(np.float32)
        mo, o = int(rng.integers(0, 8)), int(rng.integers(0, 8))
        d = np.linalg.norm(pos.astype(np.float64))
        lo, hi = np.float32(d * rng.uniform(0.5, 1.2)), np.float32(d * rng.uniform(0.9, 2.0))
        cosang = abs(pos.astype(np.float64) @ nv.astype(np.float64)) / (d * np.linalg.norm(nv.astype(np.float64)))
        if abs(cosang - 0.866) < 1e-5 or min(abs(d - lo), abs(d - hi)) < 1e-4 * d:
            continue
        want = abs(mo - o) <= 2 and cosang >= 0.866 and lo <= d <= hi
        assert pygeom.accept_new_observe(pos, nv, mo, o, lo, hi) == want
        checked += 1
    assert checked > 2500


def test_xyz_info_is_symmetric_positive_definite():
    sc = gs.xyz_info_scene(200, seed=2)
    i1, i2 = pygeom.xyz_info(sc["xyz1"], sc["pose1"], sc["pose2"], sc["Tcw"], sc["fx"])
    ok = np.isfinite(i1).all(axis=(1, 2)) & np.isfinite(i2).all(axis=(1, 2))
    assert ok.sum() > 150
    for M in np.concatenate([i1[ok], i2[ok]]):
        np.testing.assert_allclose(M, M.T, rtol=1e-4, atol=1e-6 * np.abs(M).max())
        assert np.linalg.eigvalsh(0.5 * (M + M.T)).min() > -1e-4 * np.abs(M).max()


def test_projection_observations_accept_some_and_reject_some():
    sc = gs.projection_scene(500, seed=3)
    acc, pos, info = pygeom.projection_observations(sc["kf_kp"], sc["matches_idx_mp"], sc["Tcw_new"], sc["mp"], sc["Tcw_table"],
                                                    sc["K"], sc["lower"], sc["upper"], sc["fx"])
    assert 50 < acc.sum() < (sc["matches_idx_mp"] >= 0).sum()
    assert not acc[sc["matches_idx_mp"] < 0].any()
    assert (pos[acc == 1][:, 2] >= sc["lower"]).all() and (pos[acc == 0] == 0).all()
