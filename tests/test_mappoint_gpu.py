"""Map-point updates on the GPU (se2gpu_mp_*) against the oracle, byte for byte on every output: the point table, view_mp,
view_info and the abandoned flags (NaN payloads aside, as in tests/test_geom_gpu.py)."""
import ctypes as C

import numpy as np
import pytest

from oracle import pygeom, pymappoint as pm, pyoracle
from tests import mappoint_cases as mc
from tools import mappoint_scenes as ms

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")
if not torch.cuda.is_available():
    pytest.skip("no CUDA device", allow_module_level=True)

from se2lam_b200 import _capi, mappoint  # noqa: E402
from se2lam_b200._capi import KP_DTYPE, ptr  # noqa: E402

SIZES = [1, 37, 1000, 64 * 1000]
ERR_INVALID = -3
MP_KEYS = [k for k in mappoint.MP_FIELDS if k not in ("obs_ptr", "obs_kf", "obs_idx")]


def canon(a):
    a = np.array(a, copy=True)
    if a.dtype.kind == "f":
        a[np.isnan(a)] = np.nan
    return a.tobytes()


def diff(a, b, keys):
    return [k for k in keys if canon(a[k]) != canon(b[k])]


def run(sc, mode, where):
    kf, mp = ms.copy_tables(sc)
    if where == "oracle":
        fn = pm.add_observations if mode == "add" else pm.erase_observations
        ab = fn(kf, mp, sc["upd_ptr"], sc["upd_pos"], sc["params"])
    else:
        pts = mappoint.MapPoints(kf, mp, **sc["params"])
        ab = (pts.addObservation if mode == "add" else pts.eraseObservation)(sc["upd_ptr"], sc["upd_pos"])
    return kf, mp, ab


def assert_same(sc, mode):
    kf_g, mp_g, ab_g = run(sc, mode, "gpu")
    kf_o, mp_o, ab_o = run(sc, mode, "oracle")
    assert not diff(kf_g, kf_o, ["view_mp", "view_info"]) and not diff(mp_g, mp_o, MP_KEYS)
    assert np.array_equal(ab_g, ab_o)
    return kf_g, mp_g, ab_g


@pytest.mark.parametrize("n", SIZES)
def test_add(n):
    assert_same(ms.scene(n, seed=n), "add")


@pytest.mark.parametrize("n", SIZES)
def test_erase(n):
    assert_same(ms.scene(n, seed=n + 1, mode="erase"), "erase")


@pytest.mark.parametrize("n", SIZES)
def test_update_measure(n):
    sc = ms.scene(n, seed=n + 2)
    pts = np.arange(0, n, 2, dtype=np.int32)
    kf_g, mp_g = ms.copy_tables(sc); kf_o, mp_o = ms.copy_tables(sc)
    mappoint.MapPoints(kf_g, mp_g, **sc["params"]).updateMeasureInKFs(pts)
    pm.update_measure(kf_o, mp_o, pts)
    assert canon(kf_g["view_mp"]) == canon(kf_o["view_mp"])


@pytest.mark.parametrize("family,i", [("add", i) for i in range(len(mc.add_scenes()))] + [("erase", i) for i in range(len(mc.erase_scenes()))])
def test_branch_scenes(family, i):
    sc = (mc.add_scenes() if family == "add" else mc.erase_scenes())[i][1]
    assert_same(sc, family)


@pytest.mark.parametrize("mode", ["add", "erase"])
def test_lists_past_the_shared_memory_list(mode):
    sc = mc.long_scene(mode)
    kf, mp, ab = assert_same(sc, mode)
    assert (np.diff(sc["mp"]["obs_ptr"]) > 32).sum() >= 20


# ------------------------------------------------------------------------------------------ device entries
def dev(a):
    a = np.ascontiguousarray(a)
    return torch.from_numpy(a.view(np.uint8).reshape(len(a), -1) if a.dtype == KP_DTYPE else a).cuda()


def host(t, like):
    a = t.cpu().numpy()
    return a.view(KP_DTYPE).reshape(like.shape) if like.dtype == KP_DTYPE else a.reshape(like.shape)


def run_device(sc, mode, stream=None):
    dkf = {k: dev(v) for k, v in sc["kf"].items()}
    dmp = {k: dev(v) for k, v in sc["mp"].items()}
    M = len(sc["mp"]["obs_ptr"]) - 1
    d_ab = torch.full((M,), 7, dtype=torch.uint8, device="cuda"); d_st = torch.full((1,), 5, dtype=torch.int32, device="cuda")
    prm = mappoint.params(**sc["params"])
    d_up, d_pos = dev(sc["upd_ptr"]), dev(sc["upd_pos"])       # held: the call only takes their addresses
    fn = _capi.lib().se2gpu_mp_add_observations_device if mode == "add" else _capi.lib().se2gpu_mp_erase_observations_device
    rc = fn(C.byref(mappoint.keyframes(dkf)), C.byref(mappoint.points(dmp)), ptr(d_up), ptr(d_pos),
            C.byref(prm), ptr(d_ab), ptr(d_st), C.c_void_p(stream.cuda_stream if stream else 0))
    assert rc == 0
    torch.cuda.synchronize()
    return ({k: host(v, sc["kf"][k]) for k, v in dkf.items()}, {k: host(v, sc["mp"][k]) for k, v in dmp.items()},
            d_ab.cpu().numpy().astype(bool), int(d_st.item()))


@pytest.mark.parametrize("mode", ["add", "erase"])
def test_device_entries_equal_host_entries(mode):
    sc = ms.scene(1000, seed=601, mode=mode)
    kf_h, mp_h, ab_h = run(sc, mode, "gpu")
    kf_d, mp_d, ab_d, st = run_device(sc, mode, torch.cuda.Stream())
    assert st == 0
    assert not diff(kf_h, kf_d, ["view_mp", "view_info"]) and not diff(mp_h, mp_d, MP_KEYS) and np.array_equal(ab_h, ab_d)


def test_update_measure_device_equals_host():
    sc = ms.scene(1000, seed=602)
    pts = np.arange(1, 1000, 3, dtype=np.int32)
    kf_h, mp_h = ms.copy_tables(sc)
    mappoint.MapPoints(kf_h, mp_h, **sc["params"]).updateMeasureInKFs(pts)
    dkf = {k: dev(v) for k, v in sc["kf"].items()}; dmp = {k: dev(v) for k, v in sc["mp"].items()}
    d_st = torch.full((1,), 5, dtype=torch.int32, device="cuda"); d_pts = dev(pts)
    assert _capi.lib().se2gpu_mp_update_measure_device(C.byref(mappoint.keyframes(dkf)), C.byref(mappoint.points(dmp)), len(pts),
                                                       ptr(d_pts), ptr(d_st), None) == 0
    torch.cuda.synchronize()
    assert int(d_st.item()) == 0 and canon(host(dkf["view_mp"], kf_h["view_mp"])) == canon(kf_h["view_mp"])


# ------------------------------------------------------------------------------------------ invalid input
def _bad_cases(sc):
    kf, mp = sc["kf"], sc["mp"]
    m = int(np.nonzero(np.diff(sc["upd_ptr"]) == 2)[0][0])
    yield "obs_kf", dict(mp=dict(mp, obs_kf=np.where(np.arange(len(mp["obs_kf"])) == 3, len(kf["kf_id"]), mp["obs_kf"]).astype(np.int32)))
    yield "obs_idx", dict(mp=dict(mp, obs_idx=np.where(np.arange(len(mp["obs_idx"])) == 5, 10 ** 6, mp["obs_idx"]).astype(np.int32)))
    yield "main_kf", dict(mp=dict(mp, main_kf=np.where(np.arange(len(mp["main_kf"])) == 2, -2, mp["main_kf"]).astype(np.int32)))
    pos = sc["upd_pos"].copy(); pos[sc["upd_ptr"][m] + 1] = pos[sc["upd_ptr"][m]]
    yield "repeated", dict(upd_pos=pos)
    pos = sc["upd_pos"].copy(); pos[0] = 10 ** 6
    yield "position", dict(upd_pos=pos)
    kb = kf["kp_base"].copy(); kb[1] = -1
    yield "kp_base", dict(kf=dict(kf, kp_base=kb))


@pytest.mark.parametrize("mode", ["add", "erase"])
def test_invalid_input_changes_nothing(mode):
    sc0 = ms.scene(200, seed=603, mode=mode)
    for name, change in _bad_cases(sc0):
        sc = dict(sc0, **change)
        kf, mp = ms.copy_tables(sc)
        pts = mappoint.MapPoints(kf, mp, **sc["params"])
        fn = pts.addObservation if mode == "add" else pts.eraseObservation
        with pytest.raises(_capi.Se2GpuError, match=str(ERR_INVALID)):
            fn(sc["upd_ptr"], sc["upd_pos"])
        assert not diff(kf, sc["kf"], list(kf)) and not diff(mp, sc["mp"], list(mp)), name
        kf_d, mp_d, ab_d, st = run_device(sc, mode)
        assert st == ERR_INVALID, name
        assert not diff(kf_d, sc["kf"], list(kf)) and not diff(mp_d, sc["mp"], list(mp)) and (ab_d == 1).all(), name


def test_update_measure_rejects_a_point_outside_the_table():
    sc = ms.scene(50, seed=604)
    kf, mp = ms.copy_tables(sc)
    with pytest.raises(_capi.Se2GpuError, match=str(ERR_INVALID)):
        mappoint.MapPoints(kf, mp, **sc["params"]).updateMeasureInKFs([0, 50])
    assert canon(kf["view_mp"]) == canon(sc["kf"]["view_mp"])


# ------------------------------------------------------------------------------------------ findCorrespd on the device
def append_entries(obs_ptr, obs_kf, obs_idx, pts, kf, idx):
    """each point of `pts` (ascending, distinct) gains the entry (kf, idx[i]) at the end of its list; returns the new lists
    and the updates that insert them. Works on torch tensors of either device."""
    M = obs_ptr.numel() - 1
    lens = obs_ptr[1:] - obs_ptr[:-1]
    add = torch.zeros(M, dtype=torch.int32, device=obs_ptr.device); add[pts] = 1
    new_ptr = torch.zeros(M + 1, dtype=torch.int32, device=obs_ptr.device); new_ptr[1:] = torch.cumsum(lens + add, 0)
    owner = torch.repeat_interleave(torch.arange(M, device=obs_ptr.device), lens)
    dst = new_ptr[owner] + (torch.arange(owner.numel(), device=obs_ptr.device) - obs_ptr[owner])
    n = int(new_ptr[-1])
    nk = torch.empty(n, dtype=torch.int32, device=obs_ptr.device); ni = torch.empty_like(nk)
    nk[dst] = obs_kf; ni[dst] = obs_idx
    nk[new_ptr[pts] + lens[pts]] = kf; ni[new_ptr[pts] + lens[pts]] = idx
    upd_ptr = torch.zeros(M + 1, dtype=torch.int32, device=obs_ptr.device); upd_ptr[1:] = torch.cumsum(add, 0)
    return new_ptr, nk, ni, upd_ptr, lens[pts].to(torch.int32)


def test_find_correspd_sequence_stays_on_the_device():
    """loop 1 adds for the tracked points, se2gpu_match_by_projection_device and se2gpu_projection_observations_device on
    the updated point table, loop 2 adds from the accepted rows, loop 3 adds (two per point) for new points; against the
    oracle running the same sequence"""
    from se2lam_b200.matcher import FrameView, ORBmatcher
    sc = ms.scene(3000, seed=605, good_frac=0.7)
    kf0, mp0 = ms.copy_tables(sc)
    M, K = len(mp0["obs_ptr"]) - 1, len(kf0["kf_id"])
    new, pref = K // 2, K // 2 - 1
    # half of the points that observe the new keyframe lose that entry: their keypoint is left for MatchByProjection to
    # find, with a normal, octave and distance range it accepts
    owner = np.repeat(np.arange(M), np.diff(mp0["obs_ptr"]))
    drop = (mp0["obs_kf"] == new) & (owner % 2 == 1) & (np.diff(mp0["obs_ptr"])[owner] > 1)
    s_drop = kf0["kp_base"][new] + mp0["obs_idx"][drop]
    m_drop = owner[drop]
    mp0["normal"][m_drop] = kf0["view_mp"][s_drop] / np.linalg.norm(kf0["view_mp"][s_drop], axis=1, keepdims=True)
    kf0["kp"]["octave"][s_drop] = mp0["main_octave"][m_drop]
    mp0["min_dist"][m_drop] = 0; mp0["max_dist"][m_drop] = 1e3
    mp0["obs_kf"], mp0["obs_idx"] = mp0["obs_kf"][~drop].copy(), mp0["obs_idx"][~drop].copy()
    mp0["obs_ptr"][1:] = np.cumsum(np.diff(mp0["obs_ptr"]) - np.bincount(m_drop, minlength=M)).astype(np.int32)
    owner = np.repeat(np.arange(M), np.diff(mp0["obs_ptr"]))
    at_new = mp0["obs_kf"] == new
    # loop 1: every point that observes the new keyframe inserts that entry
    u1_ptr = np.zeros(M + 1, np.int32); u1_ptr[1:] = np.cumsum(np.bincount(owner[at_new], minlength=M))
    u1_pos = (np.nonzero(at_new)[0] - mp0["obs_ptr"][owner[at_new]]).astype(np.int32)
    n_kf = int(np.bincount(kf0["kp_base"].searchsorted(np.arange(len(kf0["kp"])), "right") - 1, minlength=K)[new])
    base = int(kf0["kp_base"][new])
    observed = np.zeros(n_kf, np.uint8); observed[mp0["obs_idx"][at_new]] = 1
    observes_new = np.zeros(M, np.uint8); observes_new[owner[at_new]] = 1
    prm_args = sc["params"]
    Kc = np.asarray(prm_args["K"], np.float32)
    grid = FrameView(None, None).grid()
    mt = ORBmatcher(0.6, max_queries=M, max_db=n_kf)

    def sequence(kf, mp, on_gpu):
        t = (lambda a: dev(a)) if on_gpu else (lambda a: torch.from_numpy(np.ascontiguousarray(a).view(np.uint8).reshape(len(a), -1)
                                                                           if np.asarray(a).dtype == KP_DTYPE else np.ascontiguousarray(a).copy()))
        T = {k: t(v) for k, v in kf.items()}; P = {k: t(v) for k, v in mp.items()}
        st = torch.zeros(1, dtype=torch.int32, device=T["kf_id"].device)
        ab = torch.zeros(M, dtype=torch.uint8, device=T["kf_id"].device)

        def add(upd_ptr, upd_pos, n_points):
            if on_gpu:
                a = torch.zeros(n_points, dtype=torch.uint8, device="cuda")
                assert _capi.lib().se2gpu_mp_add_observations_device(
                    C.byref(mappoint.keyframes(T)), C.byref(mappoint.points(P)), ptr(upd_ptr), ptr(upd_pos),
                    C.byref(mappoint.params(**prm_args)), ptr(a), ptr(st), None) == 0
                return a
            k = {n: (v.numpy().view(KP_DTYPE).reshape(-1) if n == "kp" else v.numpy()) for n, v in T.items()}
            p = {n: v.numpy() for n, v in P.items()}
            return torch.from_numpy(pm.add_observations(k, p, upd_ptr.numpy(), upd_pos.numpy(), prm_args).astype(np.uint8))

        add(t(u1_ptr), t(u1_pos), M)
        # MatchByProjection's inputs from the updated table: mp_valid and the predicted uv of every point
        # elementwise, one rounding per operation, so that both devices predict the same uv
        Tn = T["Tcw"][new].to(torch.float64)
        x = P["pos"].to(torch.float64)
        pc = [x[:, 0] * Tn[i, 0] + x[:, 1] * Tn[i, 1] + x[:, 2] * Tn[i, 2] + Tn[i, 3] for i in range(3)]
        u = (pc[0] * float(Kc[0, 0]) + pc[2] * float(Kc[0, 2])) / pc[2]
        w = (pc[1] * float(Kc[1, 1]) + pc[2] * float(Kc[1, 2])) / pc[2]
        uv = torch.stack([u, w], 1).to(torch.float32).contiguous()
        inb = (pc[2] > 0) & (uv[:, 0] >= 0) & (uv[:, 0] < 640) & (uv[:, 1] >= 0) & (uv[:, 1] < 480)
        # a point with good parallax always has a main keyframe in the reference; the scene's -1 entries are left out
        valid = ((P["good_prl"] == 1) & (P["null"] == 0) & (P["main_kf"] >= 0) & (t(observes_new) == 0) & inb).to(torch.uint8)
        kp_new = T["kp"][base:base + n_kf].contiguous(); desc_new = T["desc"][base:base + n_kf].contiguous()
        if on_gpu:
            match = torch.full((n_kf,), -1, dtype=torch.int32, device="cuda")
            mt.MatchByProjectionDevice(kp_new, desc_new, n_kf, t(observed), valid, uv, M, P["main_octave"], P["main_desc"],
                                       grid, 15, 2, match)
            acc = torch.zeros(n_kf, dtype=torch.uint8, device="cuda")
            pos = torch.zeros((n_kf, 3), dtype=torch.float32, device="cuda"); info = torch.zeros((n_kf, 9), dtype=torch.float64, device="cuda")
            K_d = t(Kc.reshape(-1).copy())
            assert _capi.lib().se2gpu_projection_observations_device(
                ptr(kp_new), n_kf, None, ptr(match), ptr(T["Tcw"][new].contiguous()), ptr(P["main_measure"]), ptr(P["main_kf"]),
                ptr(P["main_octave"]), ptr(P["normal"]), ptr(P["min_dist"]), ptr(P["max_dist"]), ptr(T["Tcw"]), ptr(K_d),
                float(prm_args["lower_depth"]), float(prm_args["upper_depth"]), float(prm_args["fx"]), ptr(acc), ptr(pos),
                ptr(info), None) == 0
        else:
            kpn = kp_new.numpy().view(KP_DTYPE).reshape(-1)
            m_o = pyoracle.match_by_projection(kpn, desc_new.numpy(), observed, valid.numpy(), uv.numpy(), P["main_octave"].numpy(),
                                               P["main_desc"].numpy(), (grid.min_x, grid.min_y, grid.inv_w, grid.inv_h), 15, 2, 0.6)
            match = torch.from_numpy(m_o[1])
            mpd = dict(main_measure=P["main_measure"].numpy(), main_pose=P["main_kf"].numpy(), main_octave=P["main_octave"].numpy(),
                       normal=P["normal"].numpy(), min_dist=P["min_dist"].numpy(), max_dist=P["max_dist"].numpy())
            a_o, p_o, i_o = pygeom.projection_observations(kpn, match.numpy(), T["Tcw"][new].numpy(), mpd, T["Tcw"].numpy(), Kc,
                                                           prm_args["lower_depth"], prm_args["upper_depth"], prm_args["fx"])
            acc, pos, info = torch.from_numpy(a_o), torch.from_numpy(p_o), torch.from_numpy(i_o.reshape(-1, 9))
        # loop 2: setViewMP of the accepted rows, then the points' new entries (the first row of a point that several match)
        rows = torch.nonzero(acc == 1).flatten()
        pts_all = match[rows].long()
        order = torch.argsort(pts_all * n_kf + rows, stable=True)
        pts_sorted, rows_sorted = pts_all[order], rows[order]
        first = torch.ones_like(pts_sorted, dtype=torch.bool); first[1:] = pts_sorted[1:] != pts_sorted[:-1]
        pts, rows = pts_sorted[first], rows_sorted[first]
        T["view_mp"][base + rows] = pos[rows]
        T["view_info"][base + rows] = info[rows].reshape(-1, 3, 3)
        ptr2, k2, i2, u2p, u2 = append_entries(P["obs_ptr"], P["obs_kf"], P["obs_idx"], pts, new, rows.to(torch.int32))
        P["obs_ptr"], P["obs_kf"], P["obs_idx"] = ptr2, k2, i2
        ab2 = add(u2p, u2, M)
        # loop 3: two new points on the spare keypoints 0 of the previous and the new keyframe, and the last ones
        spare = [(pref, 0, new, 0), (pref, 1, new, n_kf - 1)]
        n3 = len(spare)
        P2 = {}
        for name, v in P.items():
            if name in ("obs_ptr", "obs_kf", "obs_idx"):
                continue
            z = torch.zeros((n3,) + tuple(v.shape[1:]), dtype=v.dtype, device=v.device)
            if name == "main_kf":
                z -= 1
            if name == "pos":
                z += torch.tensor([[0.3, 0.1, 2.5]], dtype=v.dtype, device=v.device)
            P2[name] = torch.cat([v, z])
        P2["obs_ptr"] = torch.cat([P["obs_ptr"], P["obs_ptr"][-1] + torch.tensor([2, 4], dtype=torch.int32, device=v.device)])
        P2["obs_kf"] = torch.cat([P["obs_kf"], torch.tensor([s[c] for s in spare for c in (0, 2)], dtype=torch.int32, device=v.device)])
        P2["obs_idx"] = torch.cat([P["obs_idx"], torch.tensor([s[c] for s in spare for c in (1, 3)], dtype=torch.int32, device=v.device)])
        P = P2
        u3p = torch.zeros(M + n3 + 1, dtype=torch.int32, device=v.device); u3p[M + 1:] = torch.tensor([2, 4], dtype=torch.int32, device=v.device)
        ab3 = add(u3p, torch.tensor([0, 1, 0, 1], dtype=torch.int32, device=v.device), M + n3)
        if on_gpu:
            torch.cuda.synchronize()
            assert int(st.item()) == 0
        out_kf = {k: v.cpu().numpy() for k, v in T.items()}
        out_mp = {k: v.cpu().numpy() for k, v in P.items()}
        return out_kf, out_mp, acc.cpu().numpy(), ab2.cpu().numpy(), ab3.cpu().numpy(), match.cpu().numpy(), uv.cpu().numpy()

    g = sequence(kf0, mp0, True)
    o = sequence(kf0, mp0, False)
    assert g[6].tobytes() == o[6].tobytes() and np.array_equal(g[5], o[5])
    assert g[2].sum() > 20                            # MatchByProjection's branch accepted a real share of rows
    assert np.array_equal(g[2], o[2])
    assert canon(g[0]["view_mp"]) == canon(o[0]["view_mp"]) and canon(g[0]["view_info"]) == canon(o[0]["view_info"])
    assert not diff(g[1], o[1], list(g[1])) and np.array_equal(g[3], o[3]) and np.array_equal(g[4], o[4])
