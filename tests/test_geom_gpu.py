"""Two-view geometry entry points on the GPU against the oracle, bit for bit (NaN payloads aside: x86 and the GPU produce
different quiet-NaN bit patterns, so every NaN is compared as one canonical NaN; infinities and zero signs compare exactly)."""
import ctypes as C
import os

import numpy as np
import pytest

from oracle import pygeom
from tools import geom_scenes as gs

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")
if not torch.cuda.is_available():
    pytest.skip("no CUDA device", allow_module_level=True)

from se2lam_b200 import _capi, geometry  # noqa: E402
from se2lam_b200._capi import ptr  # noqa: E402

SIZES = [1, 37, 1000, 64 * 1000]
ERR_INVALID = -3


def canon(a):
    a = np.array(a, copy=True)
    if a.dtype == np.float32:
        a[np.isnan(a)] = np.float32("nan")
    elif a.dtype == np.float64:
        a[np.isnan(a)] = np.nan
    v = a.view(np.uint32 if a.dtype == np.float32 else np.uint64)
    if a.dtype.kind == "f":
        v[np.isnan(a)] = np.array(np.nan, a.dtype).view(v.dtype)
    return a.tobytes()


def same(a, b):
    return np.asarray(a).shape == np.asarray(b).shape and canon(np.asarray(a)) == canon(np.asarray(b))


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a).view(np.uint8).reshape(-1).copy()).cuda()


def host(t, dtype, shape):
    return t.cpu().numpy().view(dtype).reshape(shape)


# ------------------------------------------------------------------------------------------ triangulate
@pytest.mark.parametrize("n", SIZES)
def test_triangulate(n):
    sc = gs.triangulate_scene(n, seed=n)
    want = pygeom.triangulate(sc["pt1"], sc["pt2"], sc["P"], sc["idx1"], sc["idx2"])
    got = geometry.triangulate(sc["pt1"], sc["pt2"], sc["P"], sc["idx1"], sc["idx2"])
    assert same(got, want)


def test_triangulate_device_form_on_a_stream():
    sc = gs.triangulate_scene(1000, seed=11)
    want = pygeom.triangulate(sc["pt1"], sc["pt2"], sc["P"], sc["idx1"], sc["idx2"])
    d = [dev(sc[k]) for k in ("pt1", "pt2", "P", "idx1", "idx2")]
    out = torch.zeros(1000 * 3 * 4, dtype=torch.uint8, device="cuda")
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        rc = _capi.lib().se2gpu_triangulate_device(1000, *[ptr(t) for t in d], ptr(out), C.c_void_p(s.cuda_stream))
    assert rc == 0
    s.synchronize()
    assert same(host(out, np.float32, (1000, 3)), want)


def test_svd_hook_on_golden_degenerate_matrices():
    g = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "geom_golden.npz"))
    w, vt = geometry.debug_svd4(g["svd_A"])
    assert w.tobytes() == g["svd_w"].tobytes()
    assert vt.tobytes() == g["svd_vt"].tobytes()


# ------------------------------------------------------------------------------------------ doTriangulate
def _track_oracle(sc):
    return pygeom.track_triangulate(sc["kp_kf"], sc["kp_frame"], sc["matches12"], sc["kf_observed"], sc["kf_view_mp"], sc["Tcr"],
                                    sc["K"], sc["lower"], sc["upper"], 2, sc["local_mps"])


def _track_gpu(sc):
    return geometry.doTriangulate(sc["kp_kf"], sc["kp_frame"], sc["matches12"], sc["kf_observed"], sc["kf_view_mp"], sc["Tcr"],
                                  sc["K"], sc["lower"], sc["upper"], sc["local_mps"])


@pytest.mark.parametrize("n", SIZES)
def test_track_triangulate(n):
    sc = gs.track_scene(n, seed=n + 1)
    m, lm, good, (n_old, n_good) = _track_oracle(sc)
    g_old, g_m, g_lm, g_good, g_ngood = _track_gpu(sc)
    assert (g_old, g_ngood) == (n_old, n_good)
    assert np.array_equal(g_m, m) and same(g_lm, lm) and np.array_equal(g_good, good.astype(bool))
    if n >= 1000:
        assert 0 < n_good and (m < 0).sum() > (sc["matches12"] < 0).sum()


def _parallel_rays(sc, rows):
    """Make keyframe keypoints `rows` and their matches exactly parallel rays: Tcr a pure sideways translation and both
    keypoints at the principal point. Column 2 of A is then exactly zero, the Jacobi sweeps never rotate it, and it sorts
    last: vt.row(3) = (0, 0, 1, 0), w = 0, the point at infinity."""
    K = sc["K"]
    Tcr = np.eye(4, dtype=np.float32); Tcr[0, 3] = 0.3
    sc["Tcr"] = Tcr
    kp_kf = sc["kp_kf"].copy(); kp_fr = sc["kp_frame"].copy()
    for r in rows:
        kp_kf[r]["x"], kp_kf[r]["y"] = K[0, 2], K[1, 2]
        kp_fr[sc["matches12"][r]]["x"], kp_fr[sc["matches12"][r]]["y"] = K[0, 2], K[1, 2]
    sc["kp_kf"], sc["kp_frame"] = kp_kf, kp_fr
    P0 = pygeom.gemm3(K, np.eye(3, 4, dtype=np.float32)); P1 = pygeom.gemm3(K, Tcr[:3])
    pp = np.array([K[0, 2], K[1, 2]], np.float32)
    return pygeom.build_a(pp, pp, P0, P1), P0, P1, pp


def test_points_at_infinity_are_rejected_and_left_untouched():
    sc = gs.track_scene(64, seed=5, frac_matched=1.0, frac_observed=0.0)
    rows = [5, 17, 40]
    A, P0, P1, pp = _parallel_rays(sc, rows)
    # the w = 0 path is really taken, on both sides
    _, vt_o = pygeom.svd4(A)
    _, vt_g = geometry.debug_svd4(A[None])
    assert vt_o[3, 3] == 0 and vt_g[0, 3, 3] == 0 and vt_g.tobytes() == vt_o[None].tobytes()
    xyz = geometry.triangulate(pp[None], pp[None], np.stack([P0, P1]), [0], [1])
    assert np.isinf(xyz[0, 2]) and same(xyz, pygeom.triangulate(pp[None], pp[None], np.stack([P0, P1]), [0], [1]))
    m, lm, good, counts = _track_oracle(sc)
    g_old, g_m, g_lm, g_good, g_ngood = _track_gpu(sc)
    assert np.array_equal(g_m, m) and same(g_lm, lm) and (g_old, g_ngood) == counts and np.array_equal(g_good, good.astype(bool))
    assert (g_m[rows] == -1).all()                                                       # rejected by the depth test
    assert g_lm[rows].tobytes() == sc["local_mps"][rows].tobytes()                       # left untouched


def test_points_behind_the_camera_are_rejected_and_left_untouched():
    sc = gs.track_scene(64, seed=6, frac_matched=1.0, frac_observed=0.0)
    m, lm, _, _ = _track_oracle(sc)
    _, g_m, g_lm, _, _ = _track_gpu(sc)
    assert g_m[2] == -1 and m[2] == -1 and lm[2].tobytes() == sc["local_mps"][2].tobytes()    # row 2 is behind the camera
    assert g_lm[2].tobytes() == sc["local_mps"][2].tobytes()
    assert np.array_equal(g_m, m) and same(g_lm, lm)


def test_track_triangulate_zero_matches_and_all_observed():
    sc = gs.track_scene(100, seed=9, frac_matched=0.0)
    g_old, g_m, g_lm, g_good, g_ngood = _track_gpu(sc)
    assert (g_old, g_ngood) == (0, 0) and (g_m == -1).all() and g_lm.tobytes() == sc["local_mps"].tobytes() and not g_good.any()
    sc = gs.track_scene(100, seed=10, frac_matched=1.0, frac_observed=1.0)
    g_old, g_m, g_lm, g_good, g_ngood = _track_gpu(sc)
    assert g_old == 100 and g_ngood == 0 and g_lm.tobytes() == sc["kf_view_mp"].tobytes()
    assert geometry.doTriangulate(sc["kp_kf"][:0], sc["kp_frame"], sc["matches12"][:0], sc["kf_observed"][:0], sc["kf_view_mp"][:0],
                                  sc["Tcr"], sc["K"], 0.1, 10, sc["local_mps"][:0])[0] == 0


def test_track_triangulate_device_count_below_capacity():
    n, cnt = 1000, 613
    sc = gs.track_scene(n, seed=12)
    sub = dict(sc, kp_kf=sc["kp_kf"][:cnt], matches12=sc["matches12"][:cnt], kf_observed=sc["kf_observed"][:cnt],
               kf_view_mp=sc["kf_view_mp"][:cnt], local_mps=sc["local_mps"][:cnt])
    m, lm, good, counts = _track_oracle(sub)
    d_kf, d_fr, d_m, d_obs, d_vm, d_T, d_K, d_lm = [dev(sc[k]) for k in ("kp_kf", "kp_frame", "matches12", "kf_observed", "kf_view_mp",
                                                                          "Tcr", "K", "local_mps")]
    d_good = torch.full((n,), 7, dtype=torch.uint8, device="cuda")
    d_cnt = torch.zeros(8, dtype=torch.uint8, device="cuda")
    d_n = torch.tensor([cnt], dtype=torch.int32, device="cuda")
    rc = _capi.lib().se2gpu_track_triangulate_device(ptr(d_kf), n, ptr(d_n), ptr(d_fr), ptr(d_m), ptr(d_obs), ptr(d_vm), ptr(d_T),
                                                     ptr(d_K), 0.1, 10.0, 2, ptr(d_lm), ptr(d_good), ptr(d_cnt), None)
    assert rc == 0
    torch.cuda.synchronize()
    g_m = host(d_m, np.int32, (n,)); g_lm = host(d_lm, np.float32, (n, 3)); g_good = d_good.cpu().numpy()
    assert tuple(host(d_cnt, np.int32, (2,))) == counts
    assert np.array_equal(g_m[:cnt], m) and same(g_lm[:cnt], lm) and np.array_equal(g_good[:cnt], good)
    assert np.array_equal(g_m[cnt:], sc["matches12"][cnt:]) and g_lm[cnt:].tobytes() == sc["local_mps"][cnt:].tobytes()
    assert (g_good[cnt:] == 7).all()


# ------------------------------------------------------------------------------------------ calcSE3toXYZInfo
@pytest.mark.parametrize("n", SIZES)
def test_xyz_info(n):
    sc = gs.xyz_info_scene(n, seed=n + 2)
    w1, w2 = pygeom.xyz_info(sc["xyz1"], sc["pose1"], sc["pose2"], sc["Tcw"], sc["fx"])
    g1, g2 = geometry.calcSE3toXYZInfo(sc["xyz1"], sc["pose1"], sc["pose2"], sc["Tcw"], sc["fx"])
    assert same(g1, w1) and same(g2, w2)


# ------------------------------------------------------------------------------------------ findCorrespd projection branch
@pytest.mark.parametrize("n", SIZES)
def test_projection_observations(n):
    sc = gs.projection_scene(n, n_mp=min(n, 4000), seed=n + 3)
    acc, pos, info = pygeom.projection_observations(sc["kf_kp"], sc["matches_idx_mp"], sc["Tcw_new"], sc["mp"], sc["Tcw_table"], sc["K"],
                                                    sc["lower"], sc["upper"], sc["fx"])
    g_acc, g_pos, g_info = geometry.findCorrespdProjection(sc["kf_kp"], sc["matches_idx_mp"], sc["Tcw_new"], sc["mp"], sc["Tcw_table"],
                                                           sc["K"], sc["lower"], sc["upper"], sc["fx"])
    assert np.array_equal(g_acc, acc.astype(bool)) and same(g_pos, pos) and same(g_info, info)
    if n >= 1000:
        assert 0 < acc.sum() < (sc["matches_idx_mp"] >= 0).sum()


# ------------------------------------------------------------------------------------------ device-resident chains
def test_device_resident_extract_then_match_then_triangulate():
    from oracle import pyoracle
    from se2lam_b200.matcher import ORBmatcher
    from se2lam_b200.orb import ORBextractor
    from tools import synth
    W, H, NF = 320, 240, 500
    img1 = synth.orb_frame(1000, W, H)
    img2 = np.roll(img1, (2, 3), axis=(0, 1))
    ext = ORBextractor(NF, 1.2, 6, fastTh=20, max_width=W, max_height=H, max_batch=2, device=0)
    lib = _capi.lib()
    frames = torch.from_numpy(np.stack([img1, img2])).cuda()
    d_kps = torch.zeros(2 * NF * 28, dtype=torch.uint8, device="cuda")
    d_desc = torch.zeros(2 * NF * 32, dtype=torch.uint8, device="cuda")
    d_cnt = torch.zeros(2, dtype=torch.int32, device="cuda")
    assert lib.se2gpu_orb_extract_device(ext.h, ptr(frames), 2, W, H, W, W * H, ptr(d_kps), ptr(d_desc), ptr(d_cnt), None) == 0
    m = ORBmatcher(0.9, max_queries=NF, max_db=NF)
    kp1, kp2 = d_kps.data_ptr(), d_kps.data_ptr() + NF * 28
    de1, de2 = d_desc.data_ptr(), d_desc.data_ptr() + NF * 32
    cnt1, cnt2 = d_cnt.data_ptr(), d_cnt.data_ptr() + 4
    d_prev = torch.zeros(NF * 2, dtype=torch.float32, device="cuda")
    assert lib.se2gpu_keypoints_to_points_device(C.c_void_p(kp1), NF, C.c_void_p(cnt1), ptr(d_prev), None) == 0
    f32 = np.float32
    grid = _capi.GridParams(f32(0), f32(0), f32(f32(64) / f32(W)), f32(f32(48) / f32(H)))
    d_m12 = torch.full((NF,), -1, dtype=torch.int32, device="cuda")
    d_nm = torch.zeros(1, dtype=torch.int32, device="cuda")
    assert lib.se2gpu_match_by_window_device(m.h, C.c_void_p(kp1), C.c_void_p(de1), NF, C.c_void_p(cnt1), C.c_void_p(kp2),
                                             C.c_void_p(de2), NF, C.c_void_p(cnt2), ptr(d_prev), grid, 20, 1, 0, 8, 0.9,
                                             ptr(d_m12), ptr(d_nm), None) == 0
    sc = gs.track_scene(NF, seed=21)
    Kc = np.array([[200, 0, W / 2], [0, 200, H / 2], [0, 0, 1]], np.float32)
    d_obs, d_vm, d_T, d_K, d_lm = [dev(a) for a in (sc["kf_observed"], sc["kf_view_mp"], sc["Tcr"], Kc, sc["local_mps"])]
    d_good = torch.zeros(NF, dtype=torch.uint8, device="cuda")
    d_counts = torch.zeros(2, dtype=torch.int32, device="cuda")
    assert lib.se2gpu_track_triangulate_device(C.c_void_p(kp1), NF, C.c_void_p(cnt1), C.c_void_p(kp2), ptr(d_m12), ptr(d_obs), ptr(d_vm),
                                               ptr(d_T), ptr(d_K), 0.1, 10.0, 2, ptr(d_lm), ptr(d_good), ptr(d_counts), None) == 0
    torch.cuda.synchronize()
    # the same chain on the oracle
    k1, dd1 = pyoracle.OrbOracle(NF, 1.2, 6, 20).extract(img1)
    k2, dd2 = pyoracle.OrbOracle(NF, 1.2, 6, 20).extract(img2)
    prev = np.stack([k1["x"], k1["y"]], 1).astype(f32)
    _, m_o, _ = pyoracle.match_by_window(k1, dd1, k2, dd2, prev, (f32(0), f32(0), grid.inv_w, grid.inv_h), 20, 1, 0, 8, 0.9)
    n1 = len(k1)
    assert (m_o >= 0).sum() > 50
    mo, lmo, goodo, counts = pygeom.track_triangulate(k1, k2, m_o, sc["kf_observed"][:n1], sc["kf_view_mp"][:n1], sc["Tcr"], Kc,
                                                      0.1, 10.0, 2, sc["local_mps"][:n1])
    assert tuple(d_counts.cpu().numpy()) == counts
    assert np.array_equal(d_m12.cpu().numpy()[:n1], mo)
    assert same(host(d_lm, np.float32, (-1, 3))[:n1], lmo)
    assert np.array_equal(d_good.cpu().numpy()[:n1], goodo)
    m.close()


def test_projection_branch_fed_by_match_by_projection_device():
    from oracle import pyoracle
    from se2lam_b200.matcher import ORBmatcher
    from tests.matcher_cases import make_projection_case
    a = make_projection_case(seed=2)["args"]
    n_kf, n_mp = len(a["kfkp"]), len(a["mp_valid"])
    geo = gs.projection_scene(n_kf, n_mp=n_mp, seed=17)
    m = ORBmatcher(a["nnratio"], max_queries=n_mp, max_db=n_kf)
    d = {k: dev(a[k]) for k in ("kfkp", "kfdesc", "kf_observed", "mp_valid", "mp_uv", "mp_octave", "mp_desc")}
    d_mi = torch.full((n_kf,), -1, dtype=torch.int32, device="cuda")
    grid = _capi.GridParams(*a["grid"])
    m.MatchByProjectionDevice(d["kfkp"], d["kfdesc"], n_kf, d["kf_observed"], d["mp_valid"], d["mp_uv"], n_mp, d["mp_octave"],
                              d["mp_desc"], grid, a["win_size"], a["level_offset"], d_mi)
    mp = geo["mp"]
    g = [dev(x) for x in (geo["Tcw_new"], mp["main_measure"], mp["main_pose"], mp["main_octave"], mp["normal"], mp["min_dist"],
                          mp["max_dist"], geo["Tcw_table"], geo["K"])]
    d_acc = torch.zeros(n_kf, dtype=torch.uint8, device="cuda")
    d_pos = torch.zeros(n_kf * 3, dtype=torch.float32, device="cuda")
    d_info = torch.zeros(n_kf * 9, dtype=torch.float64, device="cuda")
    assert _capi.lib().se2gpu_projection_observations_device(ptr(d["kfkp"]), n_kf, None, ptr(d_mi), *[ptr(t) for t in g],
                                                             float(geo["lower"]), float(geo["upper"]), float(geo["fx"]), ptr(d_acc),
                                                             ptr(d_pos), ptr(d_info), None) == 0
    torch.cuda.synchronize()
    n_o, m_o = pyoracle.match_by_projection(**a)
    assert np.array_equal(d_mi.cpu().numpy(), m_o) and n_o > 50
    acc, pos, info = pygeom.projection_observations(a["kfkp"], m_o, geo["Tcw_new"], mp, geo["Tcw_table"], geo["K"], geo["lower"],
                                                    geo["upper"], geo["fx"])
    assert np.array_equal(d_acc.cpu().numpy(), acc)
    assert same(d_pos.cpu().numpy().reshape(-1, 3), pos) and same(d_info.cpu().numpy().reshape(-1, 3, 3), info)
    m.close()


# ------------------------------------------------------------------------------------------ invalid arguments
def test_invalid_arguments():
    lib = _capi.lib()
    f = np.zeros(16, np.float32); i = np.zeros(4, np.int32); kp = np.zeros(4, _capi.KP_DTYPE); u8 = np.zeros(4, np.uint8)
    d = np.zeros(36, np.float64); bad_idx = np.array([0, 5, 0, 0], np.int32)
    assert lib.se2gpu_triangulate(-1, ptr(f), ptr(f), ptr(f), 1, ptr(i), ptr(i), ptr(f), 0) == ERR_INVALID
    assert lib.se2gpu_triangulate(4, ptr(f), ptr(f), ptr(f), 1, ptr(bad_idx), ptr(i), ptr(f), 0) == ERR_INVALID
    assert lib.se2gpu_triangulate(4, None, ptr(f), ptr(f), 1, ptr(i), ptr(i), ptr(f), 0) == ERR_INVALID
    assert lib.se2gpu_triangulate_device(4, None, None, None, None, None, None, None) == ERR_INVALID
    assert lib.se2gpu_track_triangulate(ptr(kp), 4, ptr(kp), 4, ptr(i), ptr(u8), ptr(f), ptr(f), ptr(f), 0.1, 10, 0, ptr(f), ptr(u8),
                                        ptr(i), 0) == ERR_INVALID                 # parallax degree 0
    assert lib.se2gpu_track_triangulate(ptr(kp), 4, ptr(kp), 4, ptr(bad_idx), ptr(u8), ptr(f), ptr(f), ptr(f), 0.1, 10, 2, ptr(f),
                                        ptr(u8), ptr(i), 0) == ERR_INVALID        # match past the frame's keypoints
    assert lib.se2gpu_track_triangulate_device(None, 4, None, None, None, None, None, None, None, 0.1, 10, 2, None, None, None,
                                               None) == ERR_INVALID
    assert lib.se2gpu_xyz_info(4, ptr(f), ptr(bad_idx), ptr(i), ptr(f), 1, 200.0, ptr(d), ptr(d), 0) == ERR_INVALID
    assert lib.se2gpu_xyz_info_device(-2, None, None, None, None, 200.0, None, None, None) == ERR_INVALID
    assert lib.se2gpu_projection_observations(ptr(kp), 4, ptr(bad_idx), ptr(f), ptr(f), ptr(i), ptr(i), ptr(f), ptr(f), ptr(f), 1,
                                              ptr(f), 1, ptr(f), 0.1, 10, 200.0, ptr(u8), ptr(f), ptr(d), 0) == ERR_INVALID
    assert lib.se2gpu_projection_observations_device(None, 4, None, None, None, None, None, None, None, None, None, None, None,
                                                     0.1, 10, 200.0, None, None, None, None) == ERR_INVALID
    assert lib.se2gpu_debug_svd4(-1, None, None, None, 0) == ERR_INVALID
