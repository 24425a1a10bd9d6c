"""GPU: the batched device matchers (se2gpu_match_by_window_batch_device, se2gpu_match_by_projection_batch_device) pair by pair
against the single-pair device calls and the CPU oracle, bit for bit.

Pair b reads and writes slot b of every array (the extractor's layout). Its outputs must be the bytes the single-pair call
makes for that pair alone at the same capacities and device counts - matches, vbPrevMatched, match count and the
rounds / fallback diagnostics - and one batched call must issue the kernel launches of one single-pair call, whatever B is.
"""
import ctypes as C

import numpy as np
import pytest

from oracle import pyoracle
from se2lam_b200._capi import KP_DTYPE, lib, ptr
from se2lam_b200.matcher import FrameView, ORBmatcher
from tests.matcher_cases import (make_big_window_case, make_frame_pair, make_grid_edge_pair, make_projection_case,
                                 make_projection_chain_case, make_projection_edge_case)
from tests.matcher_cases import UNDIST_BOUNDS
from tools import synth

pytestmark = pytest.mark.gpu

f32 = np.float32
RATIO, WIN = 0.9, 20
ERR_INVALID, ERR_CAPACITY = -3, -4
GRID = FrameView(None, None).grid()
UGRID = FrameView(None, None, UNDIST_BOUNDS[0], UNDIST_BOUNDS[2], UNDIST_BOUNDS[1], UNDIST_BOUNDS[3]).grid()


def oracle_grid(g):
    return (f32(g.min_x), f32(g.min_y), f32(g.inv_w), f32(g.inv_h))


def counted(call):
    l0 = lib().se2gpu_launch_count()
    call()
    return lib().se2gpu_launch_count() - l0


def stream():
    import torch
    return torch.cuda.current_stream().cuda_stream


def dev(a):
    import torch
    a = np.ascontiguousarray(a)
    if a.dtype == KP_DTYPE:
        a = a.view(np.uint8)
    return torch.from_numpy(a.copy()).to("cuda:0")


def host(t):
    return t.cpu().numpy()


def slot(a, count, cap):
    """`a` in a slot of `cap` entries: the first `count` kept, every entry past it a copy of a real entry, so that a read past
    the count creates or changes a match."""
    src = np.arange(cap)
    src[count:] = np.arange(count, cap) % count if count else np.arange(cap - count) % len(a)
    return a[src].copy()


# ---------------------------------------------------------------------------------------------- MatchByWindow
def window_batch(pairs, cap1, cap2):
    """pairs: (f1, f2, prev, n1, n2) -> stacked host slots [B, cap] and the counts."""
    s = dict(kp1=[], d1=[], kp2=[], d2=[], prev=[], n1=[], n2=[])
    for f1, f2, prev, n1, n2 in pairs:
        s["kp1"].append(slot(f1["kp"], n1, cap1)); s["d1"].append(slot(f1["desc"], n1, cap1)); s["prev"].append(slot(prev, n1, cap1))
        s["kp2"].append(slot(f2["kp"], n2, cap2)); s["d2"].append(slot(f2["desc"], n2, cap2))
        s["n1"].append(n1); s["n2"].append(n2)
    return {k: np.stack(v) if k not in ("n1", "n2") else np.asarray(v, np.int32) for k, v in s.items()}


def window_oracle(s, b, grid):
    n1, n2 = s["n1"][b], s["n2"][b]
    if n1 == 0:
        return 0, np.zeros(0, np.int32), np.zeros((0, 2), f32)
    return pyoracle.match_by_window(s["kp1"][b, :n1], s["d1"][b, :n1], s["kp2"][b, :n2], s["d2"][b, :n2], s["prev"][b, :n1],
                                    oracle_grid(grid), WIN, 1, 0, 8, RATIO)


def window_single(mt, s, b, grid):
    """One pair through se2gpu_match_by_window_device: (matches [cap1], prev [cap1, 2], nmatches, rounds, fallback, launches)."""
    import torch
    cap1, cap2 = s["kp1"].shape[1], s["kp2"].shape[1]
    d_prev, d_m, d_nm = dev(s["prev"][b]), dev(np.full(cap1, 7, np.int32)), dev(np.full(1, 7, np.int32))
    d_n = dev(np.array([s["n1"][b], s["n2"][b]], np.int32))
    args = (dev(s["kp1"][b]), dev(s["d1"][b]), cap1, dev(s["kp2"][b]), dev(s["d2"][b]), cap2, d_prev, grid, WIN, d_m, d_nm)
    launches = counted(lambda: mt.MatchByWindowDevice(*args, d_n1=d_n.data_ptr(), d_n2=d_n.data_ptr() + 4, stream=stream()))
    torch.cuda.synchronize()
    rounds, fallback = mt.last_rounds()
    return host(d_m), host(d_prev), int(d_nm.item()), rounds, fallback, launches


def window_batched(mt, s, grid, null_counts=False):
    """All pairs in one se2gpu_match_by_window_batch_device call: (matches [B, cap1], prev [B, cap1, 2], nmatches [B], rounds [B],
    fallback [B], launches)."""
    import torch
    B, cap1 = s["kp1"].shape[:2]
    cap2 = s["kp2"].shape[1]
    d_prev, d_m, d_nm = dev(s["prev"]), dev(np.full((B, cap1), 7, np.int32)), dev(np.full(B, 7, np.int32))
    d_n1, d_n2 = (None, None) if null_counts else (dev(s["n1"]), dev(s["n2"]))
    args = (B, dev(s["kp1"]), dev(s["d1"]), cap1, dev(s["kp2"]), dev(s["d2"]), cap2, d_prev, grid, WIN, d_m, d_nm)
    launches = counted(lambda: mt.MatchByWindowBatchDevice(*args, d_n1=d_n1, d_n2=d_n2, stream=stream()))
    torch.cuda.synchronize()
    rounds, fallback = mt.last_rounds_batch(B)
    return host(d_m), host(d_prev), host(d_nm), rounds, fallback, launches


def check_window(s, grid, batched, single_mt):
    """Every pair of `batched` equals the single-pair call (all bytes, diagnostics, launches) and the oracle."""
    m_b, prev_b, nm_b, rounds_b, fb_b, launches_b = batched
    for b in range(len(s["n1"])):
        m_s, prev_s, nm_s, rounds_s, fb_s, launches_s = window_single(single_mt, s, b, grid)
        assert m_b[b].tobytes() == m_s.tobytes(), b
        assert prev_b[b].tobytes() == prev_s.tobytes(), b
        assert (nm_b[b], rounds_b[b], fb_b[b]) == (nm_s, rounds_s, fb_s), b
        assert launches_b == launches_s, (launches_b, launches_s)
        n1 = s["n1"][b]
        n_o, m_o, prev_o = window_oracle(s, b, grid)
        assert nm_b[b] == n_o, b
        np.testing.assert_array_equal(m_b[b, :n1], m_o)
        assert (m_b[b, n1:] == -1).all(), b
        np.testing.assert_array_equal(prev_b[b, :n1], prev_o)
        np.testing.assert_array_equal(prev_b[b, n1:], s["prev"][b, n1:])


def steal_chain_pair(n=200):
    """40 queries that each beat the previous claim on keypoint 0 of frame 2: more claims than the claim table holds."""
    rng = np.random.default_rng(5)
    f1, f2, _ = make_frame_pair(seed=9, n=n)
    kp1, d1, kp2, d2 = f1["kp"], f1["desc"], f2["kp"], f2["desc"]
    kp2["x"][0], kp2["y"][0], kp2["octave"][0] = 300.0, 200.0, 0
    for q in range(40):
        kp1["x"][q], kp1["y"][q], kp1["octave"][q] = 300.0 + 0.1 * q, 200.0, 0
        kp1["angle"][q] = f32((float(kp2["angle"][0]) - 7.0) % 360.0)
        d1[q] = d2[0]
        for bit in rng.choice(256, 40 - q, replace=False):
            d1[q, bit // 8] ^= np.uint8(1 << (bit % 8))
    prev = np.stack([kp1["x"], kp1["y"]], axis=1).astype(f32)
    return f1, f2, prev


def test_window_batch_of_eight_cases():
    """Frame pairs, the grid-edge pair (non-zero origin, half cells, windows outside the grid), a steal chain that takes the
    sequential fallback in its pair only, a pair with *d_n1 = 0, and pairs with device counts below the capacity whose slots
    past the counts hold copies of real entries. One grid for the batch: the undistorted bounds."""
    cap1 = cap2 = 1000
    e1, e2, eprev, _ = make_grid_edge_pair(seed=21)
    c1, c2, cprev = steal_chain_pair()
    b1, b2, bprev = make_big_window_case(63, 1000, 1000)
    pairs = [make_frame_pair(seed=1) + (900, 900),
             (e1, e2, eprev, 700, 700),
             (c1, c2, cprev, 200, 200),
             make_frame_pair(seed=5, n=400) + (0, 400),
             (b1, b2, bprev, 600, 700),
             make_frame_pair(seed=6, n=1000) + (1000, 800),
             make_frame_pair(seed=7, n=500) + (500, 500),
             make_frame_pair(seed=4) + (900, 450)]
    s = window_batch(pairs, cap1, cap2)
    mt = ORBmatcher(RATIO, max_queries=cap1, max_db=cap2, max_batch=8)
    batched = window_batched(mt, s, UGRID)
    _, _, nm, rounds, fallback, launches = batched
    assert launches == 4
    assert fallback.tolist() == [False, False, True, False, False, False, False, False], fallback
    assert (rounds >= 1).all(), rounds
    assert nm[3] == 0 and (nm[[0, 1, 4, 5]] > 100).all(), nm
    check_window(s, UGRID, batched, ORBmatcher(RATIO, max_queries=cap1, max_db=cap2))
    # NULL count arrays: every pair at its capacity
    full = window_batch([make_frame_pair(seed=s_, n=1000) + (1000, 1000) for s_ in (11, 12, 13)], cap1, cap2)
    check_window(full, GRID, window_batched(mt, full, GRID, null_counts=True), ORBmatcher(RATIO, max_queries=cap1, max_db=cap2))


def test_window_batch_large_database():
    """Databases of 8193, 16384 and 10000 keypoints at a capacity of 16384 in one call: the global-memory grid for every pair
    and no claim table (K = 0), so the host raises every pair's flag and the sequential kernel runs each."""
    cap1, cap2 = 2000, 16384
    pairs = []
    for seed, ndb in ((61, 8193), (62, 16384), (64, 10000)):
        f1, f2, prev = make_big_window_case(seed, cap1, ndb)
        pairs.append((f1, f2, prev, cap1, ndb))
    s = window_batch(pairs, cap1, cap2)
    mt = ORBmatcher(RATIO, max_queries=cap1, max_db=cap2, max_batch=3)
    batched = window_batched(mt, s, GRID)
    _, _, nm, rounds, fallback, launches = batched
    assert launches == 4 and fallback.all() and (rounds == 0).all(), (launches, fallback, rounds)
    assert (nm > 500).all(), nm
    check_window(s, GRID, batched, ORBmatcher(RATIO, max_queries=cap1, max_db=cap2))


@pytest.mark.parametrize("cap1,cap2,want", [(1000, 1000, 4), (200, 8193, 5)])
def test_window_batch_launch_count(cap1, cap2, want):
    """A batched call issues the launches of one single-pair call for B = 1, 8 and 64: 4 with the shared-memory grid, 5 with
    the global-memory grid (k_grid_cell_big + k_grid_order_big) and the claim table."""
    if cap2 == cap1:
        base = [make_frame_pair(seed=100 + k, n=cap1) + (cap1 - 37 * k, cap2 - 41 * k) for k in range(8)]
    else:
        base = [make_big_window_case(100 + k, cap1, cap2) + (cap1, cap2 - 97 * k) for k in range(8)]
    single = ORBmatcher(RATIO, max_queries=cap1, max_db=cap2)
    s8 = window_batch(base, cap1, cap2)
    ref = [window_single(single, s8, b, GRID) for b in range(8)]
    assert {r[5] for r in ref} == {want}
    mt = ORBmatcher(RATIO, max_queries=cap1, max_db=cap2, max_batch=64)
    for B in (1, 8, 64):
        s = window_batch([base[b % 8] for b in range(B)], cap1, cap2)
        m, prev, nm, rounds, fallback, launches = window_batched(mt, s, GRID)
        assert launches == want, (B, launches)
        for b in range(B):
            r = ref[b % 8]
            assert m[b].tobytes() == r[0].tobytes() and prev[b].tobytes() == r[1].tobytes(), (B, b)
            assert (nm[b], rounds[b], fallback[b]) == r[2:5], (B, b)


# ---------------------------------------------------------------------------------------------- MatchByProjection
def projection_batch(cases, cap_kf, cap_mp):
    """cases: (args, n_kf) with args as make_projection_case's; map-point lists padded to cap_mp with mp_valid = 0 (and
    garbage behind it), keyframe slots past n_kf copies of real keypoints with kf_observed 0."""
    rng = np.random.default_rng(77)
    s = dict(kp=[], desc=[], obs=[], valid=[], uv=[], octv=[], mdesc=[], n_kf=[], n_mp=[])
    for a, n_kf in cases:
        nmp = len(a["mp_valid"])
        s["kp"].append(slot(a["kfkp"], n_kf, cap_kf)); s["desc"].append(slot(a["kfdesc"], n_kf, cap_kf))
        obs = slot(a["kf_observed"], n_kf, cap_kf)
        obs[n_kf:] = 0
        s["obs"].append(obs)
        pad = cap_mp - nmp
        s["valid"].append(np.concatenate([a["mp_valid"], np.zeros(pad, np.uint8)]))
        s["uv"].append(np.concatenate([a["mp_uv"], rng.uniform(0, 480, (pad, 2)).astype(f32)]))
        s["octv"].append(np.concatenate([a["mp_octave"], rng.integers(0, 8, pad).astype(np.int32)]))
        s["mdesc"].append(np.concatenate([a["mp_desc"], rng.integers(0, 256, (pad, 32), dtype=np.uint8)]))
        s["n_kf"].append(n_kf); s["n_mp"].append(nmp)
    return {k: np.stack(v) if k not in ("n_kf", "n_mp") else np.asarray(v, np.int32) for k, v in s.items()}


def projection_oracle(s, b, grid):
    n_kf, nmp = s["n_kf"][b], s["n_mp"][b]
    if n_kf == 0 or nmp == 0:
        return 0, np.full(n_kf, -1, np.int32)
    return pyoracle.match_by_projection(s["kp"][b, :n_kf], s["desc"][b, :n_kf], s["obs"][b, :n_kf], s["valid"][b, :nmp], s["uv"][b, :nmp],
                                        s["octv"][b, :nmp], s["mdesc"][b, :nmp], oracle_grid(grid), 15, 2, 0.6)


def projection_single(mt, s, b, grid, padded=True):
    """One pair through se2gpu_match_by_projection_device, with the padded map-point slot (padded) or the real list only."""
    import torch
    cap_kf = s["kp"].shape[1]
    nmp = s["valid"].shape[1] if padded else s["n_mp"][b]
    d_m, d_nm, d_n = dev(np.full(cap_kf, 7, np.int32)), dev(np.full(1, 7, np.int32)), dev(s["n_kf"][b:b + 1])
    args = (dev(s["kp"][b]), dev(s["desc"][b]), cap_kf, dev(s["obs"][b]), dev(s["valid"][b, :nmp]), dev(s["uv"][b, :nmp]), nmp,
            dev(s["octv"][b, :nmp]), dev(s["mdesc"][b, :nmp]), grid, 15, 2, d_m, d_nm)
    launches = counted(lambda: mt.MatchByProjectionDevice(*args, d_n_kf=d_n, stream=stream()))
    torch.cuda.synchronize()
    rounds, fallback = mt.last_rounds()
    return host(d_m), int(d_nm.item()), rounds, fallback, launches


def projection_batched(mt, s, grid):
    import torch
    B, cap_kf = s["kp"].shape[:2]
    cap_mp = s["valid"].shape[1]
    d_m, d_nm = dev(np.full((B, cap_kf), 7, np.int32)), dev(np.full(B, 7, np.int32))
    args = (B, dev(s["kp"]), dev(s["desc"]), cap_kf, dev(s["obs"]), dev(s["valid"]), dev(s["uv"]), cap_mp, dev(s["octv"]), dev(s["mdesc"]),
            grid, 15, 2, d_m, d_nm)
    d_n_kf = dev(s["n_kf"])
    launches = counted(lambda: mt.MatchByProjectionBatchDevice(*args, d_n_kf=d_n_kf, stream=stream()))
    torch.cuda.synchronize()
    rounds, fallback = mt.last_rounds_batch(B)
    return host(d_m), host(d_nm), rounds, fallback, launches


def test_projection_batch_of_eight_cases():
    """Map-point lists of different lengths padded with mp_valid = 0 (one of them empty), the grid-edge keyframe with its order
    ties, a steal chain that takes the fallback in its pair only, keyframe counts below the capacity with copies of real
    keypoints past them, and a keyframe count of 0. Each pair equals the single call on the padded slot, the single call on
    the unpadded list and the oracle."""
    cap_kf, cap_mp = 1000, 700
    edge = make_projection_edge_case(seed=22)
    cases = [(make_projection_case(seed=2, n=900, nmp=700)["args"], 900),
             (make_projection_case(seed=7, n=900, nmp=500)["args"], 900),
             (make_projection_chain_case(), 200),
             (edge["args"], 700),
             (make_projection_case(seed=33, n=1000, nmp=600)["args"], 650),
             (make_projection_case(seed=34, n=800, nmp=300)["args"], 0),
             (make_projection_case(seed=35, n=1000, nmp=250)["args"], 1000),
             (make_projection_case(seed=36, n=600, nmp=0)["args"], 600)]
    assert all((a["win_size"], a["level_offset"], a["nnratio"]) == (15, 2, 0.6) for a, _ in cases)
    s = projection_batch(cases, cap_kf, cap_mp)
    mt = ORBmatcher(0.6, max_queries=cap_mp, max_db=cap_kf, max_batch=8)
    m_b, nm_b, rounds_b, fb_b, launches_b = projection_batched(mt, s, UGRID)
    assert launches_b == 4
    assert fb_b.tolist() == [False, False, True, False, False, False, False, False], fb_b
    assert nm_b[5] == 0 and nm_b[7] == 0 and (nm_b[[0, 1, 3, 4]] > 100).all(), nm_b
    single = ORBmatcher(0.6, max_queries=cap_mp, max_db=cap_kf)
    for b in range(8):
        m_s, nm_s, rounds_s, fb_s, launches_s = projection_single(single, s, b, UGRID)
        assert m_b[b].tobytes() == m_s.tobytes(), b
        assert (nm_b[b], rounds_b[b], fb_b[b]) == (nm_s, rounds_s, fb_s), b
        assert launches_s == launches_b
        m_u, nm_u, _, _, _ = projection_single(single, s, b, UGRID, padded=False)
        assert m_b[b].tobytes() == m_u.tobytes() and nm_b[b] == nm_u, b
        n_o, m_o = projection_oracle(s, b, UGRID)
        n_kf = s["n_kf"][b]
        assert nm_b[b] == n_o, b
        np.testing.assert_array_equal(m_b[b, :n_kf], m_o)
        assert (m_b[b, n_kf:] == -1).all(), b
    ties = edge["ties"]
    assert all(m_b[3, bb] == mp for (bb, _), mp in zip(ties, edge["tie_mps"]))


# ---------------------------------------------------------------------------------------------- extractor -> matcher -> removeOutliers
def test_extract_window_batch_remove_outliers_on_device():
    """2B frames through se2gpu_orb_extract_device (first the B reference frames, then the B current frames), vbPrevMatched
    from the keypoints by a torch slice, the window batch, then se2gpu_remove_outliers_device on its output as it lies: the
    same bytes as the per-pair chain (keypoints_to_points, single-pair window, one-pair outlier rejection), with no
    host <-> device copy between the steps."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    from se2lam_b200.orb import ORBextractor
    B, nf, H, W = 8, 1000, 480, 640
    ref = [synth.orb_frame(3000 + b) for b in range(B)]
    cur = [np.roll(f, (2 + b % 3, -3 + b % 5), axis=(0, 1)) for b, f in enumerate(ref)]
    L = lib()
    e = ORBextractor(nf, 1.2, 8, max_batch=2 * B)
    KB, DB = nf * 28, nf * 32
    d_kps = torch.zeros(2 * B * KB, dtype=torch.uint8, device="cuda:0")
    d_desc = torch.zeros(2 * B * DB, dtype=torch.uint8, device="cuda:0")
    d_cnt = torch.zeros(2 * B, dtype=torch.int32, device="cuda:0")
    d_img = dev(np.stack(ref + cur))
    e.extract_device(d_img, 2 * B, H, W, d_kps, d_desc, d_cnt, stream=stream())
    kp, desc, cnt = d_kps.data_ptr(), d_desc.data_ptr(), d_cnt.data_ptr()
    st = C.c_void_p(stream())

    # per-pair chain
    mt1 = ORBmatcher(RATIO, max_queries=nf, max_db=nf)
    p_prev = torch.zeros((B, nf, 2), dtype=torch.float32, device="cuda:0")
    p_m = torch.full((B, nf), 7, dtype=torch.int32, device="cuda:0")
    p_nm, p_nin, p_it = (torch.full((B,), 7, dtype=torch.int32, device="cuda:0") for _ in range(3))
    p_F = torch.zeros((B, 9), dtype=torch.float64, device="cuda:0")
    for b in range(B):
        k1, k2, n1, n2 = kp + b * KB, kp + (B + b) * KB, cnt + 4 * b, cnt + 4 * (B + b)
        ORBmatcher.KeypointsToPointsDevice(k1, nf, p_prev[b], d_n=n1, stream=stream())
        mt1.MatchByWindowDevice(k1, desc + b * DB, nf, k2, desc + (B + b) * DB, nf, p_prev[b], GRID, WIN, p_m[b], p_nm[b:b + 1],
                                d_n1=n1, d_n2=n2, stream=stream())
    p_matched = p_m.clone()
    for b in range(B):
        assert L.se2gpu_remove_outliers_device(1, C.c_void_p(kp + b * KB), C.c_void_p(cnt + 4 * b), nf, C.c_void_p(kp + (B + b) * KB),
                                               C.c_void_p(cnt + 4 * (B + b)), nf, ptr(p_m[b]), ptr(p_nin[b:b + 1]), ptr(p_F[b]),
                                               ptr(p_it[b:b + 1]), st) == 0

    # batched chain
    mtB = ORBmatcher(RATIO, max_queries=nf, max_db=nf, max_batch=B)
    b_m = torch.full((B, nf), 7, dtype=torch.int32, device="cuda:0")
    b_nm, b_nin, b_it = (torch.full((B,), 7, dtype=torch.int32, device="cuda:0") for _ in range(3))
    b_F = torch.zeros((B, 9), dtype=torch.float64, device="cuda:0")
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        b_prev = d_kps.view(torch.float32).view(2 * B, nf, 7)[:B, :, :2].contiguous()
        prev0 = b_prev.clone()
        mtB.MatchByWindowBatchDevice(B, kp, desc, nf, kp + B * KB, desc + B * DB, nf, b_prev, GRID, WIN, b_m, b_nm,
                                     d_n1=cnt, d_n2=cnt + 4 * B, stream=stream())
        b_matched = b_m.clone()
        assert L.se2gpu_remove_outliers_device(B, C.c_void_p(kp), C.c_void_p(cnt), nf, C.c_void_p(kp + B * KB), C.c_void_p(cnt + 4 * B),
                                               nf, ptr(b_m), ptr(b_nin), ptr(b_F), ptr(b_it), st) == 0
        torch.cuda.synchronize()
    copies = [ev.name for ev in prof.events() if "Memcpy" in ev.name and ("HtoD" in ev.name or "DtoH" in ev.name)]
    assert not copies, copies

    c = host(d_cnt)
    kps = host(d_kps).view(KP_DTYPE).reshape(2 * B, nf)
    dsc = host(d_desc).reshape(2 * B, nf, 32)
    bp, pp, p0 = host(b_prev), host(p_prev), host(prev0)
    assert host(b_matched).tobytes() == host(p_matched).tobytes()
    for t_b, t_p in ((b_m, p_m), (b_nm, p_nm), (b_nin, p_nin), (b_it, p_it), (b_F, p_F)):
        assert host(t_b).tobytes() == host(t_p).tobytes()
    for b in range(B):
        n1 = c[b]
        assert bp[b, :n1].tobytes() == pp[b, :n1].tobytes(), b
        np.testing.assert_array_equal(bp[b, n1:], p0[b, n1:])
        k1 = kps[b, :n1]
        prev = np.stack([k1["x"], k1["y"]], axis=1).astype(f32)
        n_o, m_o, prev_o = pyoracle.match_by_window(k1, dsc[b, :n1], kps[B + b, :c[B + b]], dsc[B + b, :c[B + b]], prev,
                                                    oracle_grid(GRID), WIN, 1, 0, 8, RATIO)
        assert n_o > 300 and host(b_nm)[b] == n_o, b
        np.testing.assert_array_equal(host(b_matched)[b, :n1], m_o)
        np.testing.assert_array_equal(bp[b, :n1], prev_o)
    assert (host(b_nin) >= 10).all(), host(b_nin)


# ---------------------------------------------------------------------------------------------- errors
def test_batch_errors_leave_the_context_usable():
    """B above max_batch and capacities above the context's are SE2GPU_ERR_CAPACITY, B < 0 and NULL required pointers
    SE2GPU_ERR_INVALID, B = 0 does nothing; after each failed call the next call on the context is right."""
    import torch
    L = lib()
    cap = 300
    s = window_batch([make_frame_pair(seed=40 + k, n=cap) + (cap, cap) for k in range(4)], cap, cap)
    mt = ORBmatcher(RATIO, max_queries=cap, max_db=cap, max_batch=4)
    single = ORBmatcher(RATIO, max_queries=cap, max_db=cap)
    good = window_batched(mt, s, GRID)
    check_window(s, GRID, good, single)
    kp1, d1, kp2, d2, prev = dev(s["kp1"]), dev(s["d1"]), dev(s["kp2"]), dev(s["d2"]), dev(s["prev"])
    m, nm = dev(np.zeros((4, cap), np.int32)), dev(np.zeros(4, np.int32))
    h, sp = C.c_void_p(mt.h), C.c_void_p(stream())

    def window(B, c1=cap, c2=cap, p=(kp1, d1, kp2, d2, prev, m)):
        return L.se2gpu_match_by_window_batch_device(h, B, ptr(p[0]), ptr(p[1]), c1, None, ptr(p[2]), ptr(p[3]), c2, None, ptr(p[4]),
                                                     GRID, WIN, 1, 0, 8, RATIO, ptr(p[5]), ptr(nm), sp)

    def projection(B, c_kf=cap, c_mp=cap, kf=kp2):
        return L.se2gpu_match_by_projection_batch_device(h, B, ptr(kf), ptr(d2), c_kf, None, ptr(m), ptr(m), ptr(prev), c_mp, ptr(m),
                                                         ptr(d1), GRID, 15, 2, 0.6, ptr(m), ptr(nm), sp)
    failing = [(lambda: window(5), ERR_CAPACITY), (lambda: window(2, c1=cap + 1), ERR_CAPACITY), (lambda: window(2, c2=cap + 1), ERR_CAPACITY),
               (lambda: window(-1), ERR_INVALID), (lambda: window(2, p=(None, d1, kp2, d2, prev, m)), ERR_INVALID),
               (lambda: window(2, p=(kp1, d1, kp2, None, prev, m)), ERR_INVALID), (lambda: window(2, p=(kp1, d1, kp2, d2, None, m)), ERR_INVALID),
               (lambda: window(2, p=(kp1, d1, kp2, d2, prev, None)), ERR_INVALID),
               (lambda: projection(5), ERR_CAPACITY), (lambda: projection(2, c_kf=cap + 1), ERR_CAPACITY),
               (lambda: projection(2, c_mp=cap + 1), ERR_CAPACITY), (lambda: projection(-1), ERR_INVALID),
               (lambda: projection(2, kf=None), ERR_INVALID),
               (lambda: L.se2gpu_matcher_last_rounds_batch(h, 5, None, None), ERR_INVALID),
               (lambda: L.se2gpu_match_by_window_batch_device(None, 1, None, None, cap, None, None, None, cap, None, None, GRID, WIN, 1, 0, 8,
                                                              RATIO, None, None, None), ERR_INVALID)]
    for k, (call, code) in enumerate(failing):
        m.fill_(7); nm.fill_(7)
        assert counted(call) == 0
        assert call() == code, k
        torch.cuda.synchronize()
        assert (host(m) == 7).all() and (host(nm) == 7).all(), k      # nothing written
        check_window(s, GRID, window_batched(mt, s, GRID), single)
    assert counted(lambda: window(0, p=(None,) * 6)) == 0
    assert window(0, p=(None,) * 6) == 0 and projection(0, kf=None) == 0
    assert L.se2gpu_matcher_last_rounds_batch(h, 0, None, None) == 0
    assert not L.se2gpu_matcher_create_batch(cap, cap, 0, 0)
    assert not L.se2gpu_matcher_create_batch(8192, 8192, 9, 0)      # 9 x 512 MiB candidate tables: above 4 GiB
    assert not L.se2gpu_matcher_create_batch(1, 1, 65536, 0)        # more pairs than a launch grid's y dimension
