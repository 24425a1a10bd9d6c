"""Two-view geometry and map-point updates on the GPU where the seeded scenes of tests/test_geom_gpu.py and
tests/test_mappoint_gpu.py do not reach: every boundary pair of tests/geom_boundaries.py through the host and the _device
entries, the map-point scenes of long update runs, main-keyframe erasure, long lists and other pyramid level counts, and
the batched doTriangulate over many streams. Bit for bit against the oracle, NaNs compared as one canonical NaN."""
import ctypes as C

import numpy as np
import pytest

from oracle import pymappoint as pm
from tests import geom_boundaries as gb
from tests import mappoint_cases as mc
from tests.test_geom_gpu import dev as dev_bytes, host as host_bytes, same
from tests.test_mappoint_gpu import MP_KEYS, canon, diff, run, run_device
from tests.test_mappoint_gpu import dev as table_dev
from tools import geom_scenes as gs
from tools import mappoint_scenes as ms

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")
if not torch.cuda.is_available():
    pytest.skip("no CUDA device", allow_module_level=True)

from se2lam_b200 import _capi, geometry, mappoint  # noqa: E402
from se2lam_b200._capi import ptr  # noqa: E402

ERR_INVALID, ERR_CAPACITY = -3, -4
PAIRS = gb.all_pairs()


def lib():
    return _capi.lib()


# ------------------------------------------------------------------------------------------ boundary pairs
def track_device(c):
    d = {k: dev_bytes(c[k]) for k in ("kp_kf", "kp_frame", "matches12", "kf_observed", "kf_view_mp", "Tcr", "K", "local_mps")}
    d_good = torch.full((1,), 9, dtype=torch.uint8, device="cuda")
    d_cnt = torch.full((2,), 5, dtype=torch.int32, device="cuda")
    assert lib().se2gpu_track_triangulate_device(ptr(d["kp_kf"]), 1, None, ptr(d["kp_frame"]), ptr(d["matches12"]),
                                                 ptr(d["kf_observed"]), ptr(d["kf_view_mp"]), ptr(d["Tcr"]), ptr(d["K"]),
                                                 float(c["lower"]), float(c["upper"]), c["deg"], ptr(d["local_mps"]),
                                                 ptr(d_good), ptr(d_cnt), None) == 0
    torch.cuda.synchronize()
    return (host_bytes(d["matches12"], np.int32, (1,)), host_bytes(d["local_mps"], np.float32, (1, 3)), d_good.cpu().numpy(),
            tuple(int(v) for v in d_cnt.cpu().numpy()))


def projection_device(c):
    mp = c["mp"]
    g = [dev_bytes(x) for x in (c["kf_kp"], c["matches_idx_mp"], c["Tcw_new"], mp["main_measure"], mp["main_pose"],
                                mp["main_octave"], mp["normal"], mp["min_dist"], mp["max_dist"], c["Tcw_table"], c["K"])]
    d_acc = torch.full((1,), 9, dtype=torch.uint8, device="cuda")
    d_pos = torch.zeros(3, dtype=torch.float32, device="cuda"); d_info = torch.zeros(9, dtype=torch.float64, device="cuda")
    assert lib().se2gpu_projection_observations_device(ptr(g[0]), 1, None, *[ptr(t) for t in g[1:]], float(c["lower"]),
                                                       float(c["upper"]), float(c["fx"]), ptr(d_acc), ptr(d_pos), ptr(d_info),
                                                       None) == 0
    torch.cuda.synchronize()
    return d_acc.cpu().numpy(), d_pos.cpu().numpy().reshape(1, 3), d_info.cpu().numpy().reshape(1, 3, 3)


@pytest.mark.parametrize("i", range(len(PAIRS)), ids=[f"{p.kind}-{p.what}" for p in PAIRS])
def test_boundary_pair(i):
    p = PAIRS[i]
    decided = []
    for c in (p.a, p.b):
        if p.kind == "track":
            m, lm, good, counts = gb.track_oracle(c)
            g_old, g_m, g_lm, g_good, g_ngood = geometry.doTriangulate(c["kp_kf"], c["kp_frame"], c["matches12"], c["kf_observed"],
                                                                       c["kf_view_mp"], c["Tcr"], c["K"], c["lower"], c["upper"],
                                                                       c["local_mps"], min_parallax_deg=c["deg"])
            assert np.array_equal(g_m, m) and same(g_lm, lm) and np.array_equal(g_good, good.astype(bool))
            assert (g_old, g_ngood) == counts
            d_m, d_lm, d_good, d_cnt = track_device(c)
            assert np.array_equal(d_m, m) and same(d_lm, lm) and np.array_equal(d_good, good) and d_cnt == counts
            decided.append((int(m[0]), int(good[0])))
        elif p.kind == "projection":
            acc, pos, info = gb.projection_oracle(c)
            g_acc, g_pos, g_info = geometry.findCorrespdProjection(c["kf_kp"], c["matches_idx_mp"], c["Tcw_new"], c["mp"],
                                                                   c["Tcw_table"], c["K"], c["lower"], c["upper"], c["fx"])
            assert np.array_equal(g_acc, acc.astype(bool)) and same(g_pos, pos) and same(g_info, info)
            d_acc, d_pos, d_info = projection_device(c)
            assert np.array_equal(d_acc, acc) and same(d_pos, pos) and same(d_info, info)
            decided.append(int(acc[0]))
        else:
            kf_o, mp_o, ab_o = gb.mp_oracle(c)
            kf_g, mp_g, ab_g = run(c, "add", "gpu")
            assert not diff(kf_g, kf_o, ["view_mp", "view_info"]) and not diff(mp_g, mp_o, MP_KEYS) and np.array_equal(ab_g, ab_o)
            kf_d, mp_d, ab_d, st = run_device(c, "add")
            assert st == 0 and not diff(kf_d, kf_o, ["view_mp", "view_info"]) and not diff(mp_d, mp_o, MP_KEYS)
            assert np.array_equal(ab_d, ab_o)
            decided.append((int(mp_o["good_prl"][0]), bool(ab_o[0]), canon(kf_o["view_info"])))   # pKF0 shows in view_info
    assert decided[0] != decided[1]                 # the pair really straddles the decision


# ------------------------------------------------------------------------------------------ map-point scenes
def assert_same(sc, mode):
    kf_g, mp_g, ab_g = run(sc, mode, "gpu")
    kf_o, mp_o, ab_o = run(sc, mode, "oracle")
    assert not diff(kf_g, kf_o, ["view_mp", "view_info"]) and not diff(mp_g, mp_o, MP_KEYS)
    assert np.array_equal(ab_g, ab_o)
    kf_d, mp_d, ab_d, st = run_device(sc, mode)
    assert st == 0 and not diff(kf_d, kf_o, ["view_mp", "view_info"]) and not diff(mp_d, mp_o, MP_KEYS)
    assert np.array_equal(ab_d, ab_o)
    return ab_o


def test_many_updates_per_point():
    ab = assert_same(mc.many_updates_scene(), "add")
    assert ab.sum() > 10


def test_erase_the_main_keyframe_down_to_an_empty_list():
    ab = assert_same(mc.erase_main_scene(), "erase")
    assert ab.sum() > 50


@pytest.mark.parametrize("mode", ["add", "erase"])
def test_list_lengths(mode):
    sc = mc.list_length_scene(mode)
    assert sorted(set(np.diff(sc["mp"]["obs_ptr"]))) == list(mc.LIST_LENGTHS)
    assert_same(sc, mode)


@pytest.mark.parametrize("nlevels", mc.NLEVELS)
@pytest.mark.parametrize("mode", ["add", "erase"])
def test_level_counts(nlevels, mode):
    assert_same(mc.nlevels_scene(nlevels, mode), mode)


@pytest.mark.parametrize("which", ["lengths", "nlevels"])
def test_update_measure_on_the_new_scenes(which):
    sc = mc.list_length_scene("add") if which == "lengths" else mc.nlevels_scene(5)
    M = len(sc["mp"]["obs_ptr"]) - 1
    pts = np.arange(0, M, 2, dtype=np.int32)
    kf_g, mp_g = ms.copy_tables(sc); kf_o, mp_o = ms.copy_tables(sc)
    mappoint.MapPoints(kf_g, mp_g, **sc["params"]).updateMeasureInKFs(pts)
    pm.update_measure(kf_o, mp_o, pts)
    assert canon(kf_g["view_mp"]) == canon(kf_o["view_mp"]) and canon(kf_o["view_mp"]) != canon(sc["kf"]["view_mp"])
    dkf = {k: table_dev(v) for k, v in sc["kf"].items()}
    dmp = {k: table_dev(v) for k, v in sc["mp"].items()}
    d_st = torch.full((1,), 5, dtype=torch.int32, device="cuda"); d_pts = table_dev(pts)
    assert lib().se2gpu_mp_update_measure_device(C.byref(mappoint.keyframes(dkf)), C.byref(mappoint.points(dmp)), len(pts),
                                                 ptr(d_pts), ptr(d_st), None) == 0
    torch.cuda.synchronize()
    assert int(d_st.item()) == 0 and canon(dkf["view_mp"].cpu().numpy()) == canon(kf_o["view_mp"])


def _params_with_nlevels(sc, n):
    prm = mappoint.params(**sc["params"])
    prm.nlevels = n
    return prm


@pytest.mark.parametrize("mode", ["add", "erase"])
def test_octave_at_nlevels_is_refused_and_changes_nothing(mode):
    sc0 = mc.nlevels_scene(5, mode)
    kp = sc0["kf"]["kp"].copy()
    s = int(sc0["kf"]["kp_base"][sc0["mp"]["obs_kf"][7]] + sc0["mp"]["obs_idx"][7])   # an observed slot
    kp["octave"][s] = 5
    sc = dict(sc0, kf=dict(sc0["kf"], kp=kp))
    kf, mp = ms.copy_tables(sc)
    pts = mappoint.MapPoints(kf, mp, **sc["params"])
    with pytest.raises(_capi.Se2GpuError, match=str(ERR_INVALID)):
        (pts.addObservation if mode == "add" else pts.eraseObservation)(sc["upd_ptr"], sc["upd_pos"])
    assert not diff(kf, sc["kf"], list(kf)) and not diff(mp, sc["mp"], list(mp))
    kf_d, mp_d, ab_d, st = run_device(sc, mode)
    assert st == ERR_INVALID and (ab_d == 1).all()
    assert not diff(kf_d, sc["kf"], list(kf)) and not diff(mp_d, sc["mp"], list(mp))
    kp["octave"][s] = 4                                                              # the top level is accepted
    assert_same(sc, mode)


@pytest.mark.parametrize("nlevels", [0, 33])
@pytest.mark.parametrize("mode", ["add", "erase"])
def test_level_count_out_of_range_is_refused_and_changes_nothing(nlevels, mode):
    sc = mc.nlevels_scene(32, mode)
    prm = _params_with_nlevels(sc, nlevels)
    kf, mp = ms.copy_tables(sc)
    ab = np.full(len(mp["obs_ptr"]) - 1, 7, np.uint8)
    fn = lib().se2gpu_mp_add_observations if mode == "add" else lib().se2gpu_mp_erase_observations
    assert fn(C.byref(mappoint.keyframes(kf)), C.byref(mappoint.points(mp)), ptr(sc["upd_ptr"]), ptr(sc["upd_pos"]), C.byref(prm),
              ptr(ab), 0) == ERR_INVALID
    assert not diff(kf, sc["kf"], list(kf)) and not diff(mp, sc["mp"], list(mp)) and (ab == 7).all()
    dkf = {k: table_dev(v) for k, v in sc["kf"].items()}
    dmp = {k: table_dev(v) for k, v in sc["mp"].items()}
    d_ab = torch.full((len(ab),), 7, dtype=torch.uint8, device="cuda"); d_st = torch.full((1,), 5, dtype=torch.int32, device="cuda")
    d_up, d_pos = table_dev(sc["upd_ptr"]), table_dev(sc["upd_pos"])
    fn = lib().se2gpu_mp_add_observations_device if mode == "add" else lib().se2gpu_mp_erase_observations_device
    assert fn(C.byref(mappoint.keyframes(dkf)), C.byref(mappoint.points(dmp)), ptr(d_up), ptr(d_pos), C.byref(prm), ptr(d_ab),
              ptr(d_st), None) == ERR_INVALID
    torch.cuda.synchronize()
    assert int(d_st.item()) == 5 and (d_ab.cpu().numpy() == 7).all()
    assert canon(dkf["view_mp"].cpu().numpy()) == canon(sc["kf"]["view_mp"]) and canon(dkf["view_info"].cpu().numpy()) == canon(sc["kf"]["view_info"])
    for k in MP_KEYS:
        assert canon(dmp[k].cpu().numpy()) == canon(sc["mp"][k]), k


# ------------------------------------------------------------------------------------------ batched doTriangulate
def batch_inputs(B, cap, cap_fr, seed):
    """B streams drawn from one pool of matched keypoints, each with its own Tcr (the pool's with a perturbed translation),
    its keyframe rows at b * cap and its frame rows at b * cap_fr (matches inside the stream's frame rows)"""
    rng = np.random.default_rng(seed)
    pool = gs.track_scene(4096, seed=seed)
    N = len(pool["kp_kf"])
    rows = (rng.integers(0, N, B)[:, None] + np.arange(cap)[None, :]) % N
    kp_kf = pool["kp_kf"][rows]
    kp_fr = np.zeros((B, cap_fr), gs.KP_DTYPE)
    kp_fr["x"] = rng.uniform(0, gs.W, (B, cap_fr)); kp_fr["y"] = rng.uniform(0, gs.H, (B, cap_fr)); kp_fr["size"] = 31
    slots = np.argsort(rng.random((B, max(cap, cap_fr))), axis=1)[:, :cap]          # a distinct frame row per keyframe row
    pm_ = pool["matches12"][rows]
    matched = (pm_ >= 0) & (slots < cap_fr)
    matches = np.where(matched, slots, -1).astype(np.int32)
    b_idx, i_idx = np.nonzero(matched)
    kp_fr[b_idx, slots[b_idx, i_idx]] = pool["kp_frame"][pm_[b_idx, i_idx]]
    Tcr = np.repeat(pool["Tcr"][None], B, 0).copy()
    Tcr[:, :3, 3] *= rng.uniform(0.7, 1.3, (B, 3)).astype(np.float32)
    return dict(kp_kf=kp_kf, kp_fr=kp_fr, matches=matches, observed=pool["kf_observed"][rows], view_mp=pool["kf_view_mp"][rows],
                local_mps=pool["local_mps"][rows], Tcr=Tcr, K=pool["K"])


BATCHES = [  # B, cap, cap_frame, degree, d_n ("null" or "short"), gate (None, "mixed")
    (1, 200, 257, 1, "short", None),
    (3, 300, 200, 2, "null", "mixed"),
    (64, 128, 160, 3, "short", "mixed"),
    (64, 129, 129, 4, "null", None),
    (65535, 1, 2, 4, "short", "mixed"),
    (65535, 1, 1, 1, "null", "mixed"),
]


@pytest.mark.parametrize("B,cap,cap_fr,deg,n_mode,gate_mode", BATCHES)
def test_batched_do_triangulate(B, cap, cap_fr, deg, n_mode, gate_mode):
    x = batch_inputs(B, cap, cap_fr, seed=B + cap + deg)
    rng = np.random.default_rng(B * 7 + deg)
    n = rng.integers(0, cap + 1, B).astype(np.int32) if n_mode == "short" else np.full(B, cap, np.int32)
    if n_mode == "short" and B > 1:
        n[0], n[-1] = cap, 0
    gate = None if gate_mode is None else (rng.random(B) < 0.75).astype(np.int32)
    if gate is not None:
        gate[0], gate[-1] = 1, 0
    good0 = np.full((B, cap), 9, np.uint8)
    d = {k: dev_bytes(x[k]) for k in ("kp_kf", "kp_fr", "matches", "observed", "view_mp", "local_mps", "Tcr", "K")}
    d_good = dev_bytes(good0)
    d_cnt = torch.full((2 * B,), 5, dtype=torch.int32, device="cuda")
    d_n = dev_bytes(n) if n_mode == "short" else None
    d_gate = dev_bytes(gate) if gate is not None else None
    lower, upper = gs.LOWER_DEPTH, gs.UPPER_DEPTH
    assert lib().se2gpu_track_triangulate_batch_device(B, ptr(d["kp_kf"]), cap, ptr(d_n) if d_n is not None else None, ptr(d["kp_fr"]),
                                                       cap_fr, ptr(d["matches"]), ptr(d["observed"]), ptr(d["view_mp"]), ptr(d["Tcr"]),
                                                       ptr(d_gate) if d_gate is not None else None, ptr(d["K"]), lower, upper, deg,
                                                       ptr(d["local_mps"]), ptr(d_good), ptr(d_cnt), None) == 0
    torch.cuda.synchronize()
    g_m = host_bytes(d["matches"], np.int32, (B, cap)); g_lm = host_bytes(d["local_mps"], np.float32, (B, cap, 3))
    g_good = host_bytes(d_good, np.uint8, (B, cap)); g_cnt = d_cnt.cpu().numpy().reshape(B, 2)
    on = np.ones(B, bool) if gate is None else gate.astype(bool)
    assert on.any() and (B == 1 or gate is None or not on.all())
    # gated streams: every byte as it was, counts 0
    assert np.array_equal(g_m[~on], x["matches"][~on]) and g_lm[~on].tobytes() == x["local_mps"][~on].tobytes()
    assert (g_good[~on] == 9).all() and (g_cnt[~on] == 0).all()
    for b in np.flatnonzero(on):
        k = int(n[b])
        m, lm, good, counts = gb.pygeom.track_triangulate(x["kp_kf"][b, :k], x["kp_fr"][b], x["matches"][b, :k], x["observed"][b, :k],
                                                           x["view_mp"][b, :k], x["Tcr"][b], x["K"], lower, upper, deg, x["local_mps"][b, :k])
        assert np.array_equal(g_m[b, :k], m) and same(g_lm[b, :k], lm) and np.array_equal(g_good[b, :k], good), b
        assert tuple(g_cnt[b]) == counts, b
        # past d_n[b]: as it was
        assert np.array_equal(g_m[b, k:], x["matches"][b, k:]) and g_lm[b, k:].tobytes() == x["local_mps"][b, k:].tobytes()
        assert (g_good[b, k:] == 9).all()
    if B >= 64 and cap > 1:
        assert g_cnt[on, 1].sum() > 0 and (g_m[on] == -1).sum() > (x["matches"][on] == -1).sum()
    # the single-stream call on a stream's slices gives the same bytes (a sample of the streams when B is large)
    sample = np.flatnonzero(on) if B <= 64 else np.flatnonzero(on)[np.linspace(0, on.sum() - 1, 24).astype(int)]
    for b in sample:
        s = {k: dev_bytes(x[k][b]) for k in ("kp_kf", "kp_fr", "matches", "observed", "view_mp", "local_mps", "Tcr")}
        s_good = dev_bytes(good0[b]); s_cnt = torch.full((2,), 5, dtype=torch.int32, device="cuda")
        s_n = dev_bytes(n[b:b + 1]) if n_mode == "short" else None
        assert lib().se2gpu_track_triangulate_device(ptr(s["kp_kf"]), cap, ptr(s_n) if s_n is not None else None, ptr(s["kp_fr"]),
                                                     ptr(s["matches"]), ptr(s["observed"]), ptr(s["view_mp"]), ptr(s["Tcr"]), ptr(d["K"]),
                                                     lower, upper, deg, ptr(s["local_mps"]), ptr(s_good), ptr(s_cnt), None) == 0
        torch.cuda.synchronize()
        assert host_bytes(s["matches"], np.int32, (cap,)).tobytes() == g_m[b].tobytes(), b
        assert host_bytes(s["local_mps"], np.float32, (cap, 3)).tobytes() == g_lm[b].tobytes(), b
        assert s_good.cpu().numpy().tobytes() == g_good[b].tobytes() and tuple(s_cnt.cpu().numpy()) == tuple(g_cnt[b]), b


def test_batched_do_triangulate_refuses_more_than_65535_streams():
    x = batch_inputs(2, 1, 1, seed=3)
    d = {k: dev_bytes(x[k]) for k in ("kp_kf", "kp_fr", "matches", "observed", "view_mp", "local_mps", "Tcr", "K")}
    d_good = torch.full((2,), 9, dtype=torch.uint8, device="cuda"); d_cnt = torch.full((4,), 5, dtype=torch.int32, device="cuda")
    before = {k: v.clone() for k, v in d.items()}
    assert lib().se2gpu_track_triangulate_batch_device(65536, ptr(d["kp_kf"]), 1, None, ptr(d["kp_fr"]), 1, ptr(d["matches"]),
                                                       ptr(d["observed"]), ptr(d["view_mp"]), ptr(d["Tcr"]), None, ptr(d["K"]),
                                                       gs.LOWER_DEPTH, gs.UPPER_DEPTH, 2, ptr(d["local_mps"]), ptr(d_good),
                                                       ptr(d_cnt), None) == ERR_CAPACITY
    torch.cuda.synchronize()
    assert all(torch.equal(before[k], d[k]) for k in d)
    assert (d_good.cpu() == 9).all() and (d_cnt.cpu() == 5).all()
