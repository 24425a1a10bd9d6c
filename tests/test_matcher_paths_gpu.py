"""GPU: every path of matcher.cu against the CPU oracle, bit for bit - the sequential fallbacks (claim-table overflow and
K = 0), the large-database grid (> 8192 keypoints), device-side counts below the capacity, more than 1024 queries, a grid
with a non-zero origin and the regrowth of the handle-less default context.

Each test also checks that it reached the path it was written for, from the number of kernel launches of the call
(se2gpu_launch_count) and ORBmatcher.last_rounds():

    path                                        launches  used_fallback
    small grid (<= 8192 keypoints), k_resolve   4         False
    small grid, claim table overflows           4         True, rounds >= 1
    big grid (k_grid_cell_big + _order_big)     5         either, rounds >= 1
    big grid, claim table too large (K = 0)     4         True, rounds == 0
    SearchByBoW                                 3         either (2 and True, rounds == 0 with K = 0)
"""
import numpy as np
import pytest

from oracle import pyoracle
from se2lam_b200._capi import KP_DTYPE, lib
from se2lam_b200.matcher import FrameView, ORBmatcher
from tests.matcher_cases import (GRID, UNDIST_BOUNDS, make_big_projection_case, make_big_window_case, make_bow_case, make_frame_pair,
                                 make_grid_edge_pair, make_projection_case, make_projection_chain_case, make_projection_edge_case)
from tools import synth

pytestmark = pytest.mark.gpu

PATHS = {"resolve": (4, False), "overflow": (4, True), "big": (5, None), "big_sequential": (4, True), "bow": (3, None),
         "bow_overflow": (3, True), "bow_sequential": (2, True)}


def counted(call):
    l0 = lib().se2gpu_launch_count()
    out = call()
    return out, lib().se2gpu_launch_count() - l0


def assert_path(mt, launches, path):
    import torch
    torch.cuda.synchronize()
    rounds, fallback = mt.last_rounds()
    want, want_fallback = PATHS[path]
    assert launches == want, f"{path}: {launches} launches (rounds {rounds}, fallback {fallback})"
    if want_fallback is not None:
        assert fallback == want_fallback, f"{path}: fallback {fallback} (rounds {rounds})"
    if path.endswith("sequential"):
        assert rounds == 0, rounds
    else:
        assert rounds >= 1, rounds


def frame_view(f, bounds=None):
    return FrameView(f["kp"], f["desc"]) if bounds is None else FrameView(f["kp"], f["desc"], bounds[0], bounds[2], bounds[1], bounds[3])


def window_host(mt, f1, f2, prev, grid, win=20, ratio=0.9, bounds=None):
    n_o, m_o, prev_o = pyoracle.match_by_window(f1["kp"], f1["desc"], f2["kp"], f2["desc"], prev, grid, win, 1, 0, 8, ratio)
    prev_g = prev.copy()
    (n_g, m_g), launches = counted(lambda: mt.MatchByWindow(frame_view(f1, bounds), frame_view(f2, bounds), prev_g, win))
    assert n_g == n_o
    np.testing.assert_array_equal(m_g, m_o)
    np.testing.assert_array_equal(prev_g, prev_o)
    return launches, m_o


def projection_host(mt, a, bounds=None):
    n_o, m_o = pyoracle.match_by_projection(**a)
    kf = FrameView(a["kfkp"], a["kfdesc"]) if bounds is None else FrameView(a["kfkp"], a["kfdesc"], bounds[0], bounds[2], bounds[1], bounds[3])
    (n_g, m_g), launches = counted(lambda: mt.MatchByProjection(kf, a["kf_observed"], a["mp_valid"], a["mp_uv"], a["mp_octave"],
                                                                a["mp_desc"], a["win_size"], a["level_offset"]))
    assert n_g == n_o
    np.testing.assert_array_equal(m_g, m_o)
    return launches, m_o


def bow_host(mt, k1, k2, mp_only, ori):
    n_o, m_o = pyoracle.search_by_bow(k1, k2, mp_only, 0.6, ori)
    (n_g, m_g), launches = counted(lambda: mt.SearchByBoW(k1, k2, mp_only))
    assert n_g == n_o
    np.testing.assert_array_equal(m_g, m_o)
    return launches, m_o


def dev(a):
    import torch
    a = np.ascontiguousarray(a)
    if a.dtype == KP_DTYPE:
        a = a.view(np.uint8)
    return torch.from_numpy(a.copy()).to("cuda:0")


# ---------------------------------------------------------------------------------------------- sequential fallbacks
def test_projection_steal_chain_takes_the_fallback():
    """48 map points predicted at one keyframe keypoint, each closer than the one before: more simultaneous claims than the
    claim table holds. The same-level ratio rule rejects some of them, bestLevel2 of another octave lets others through,
    and the last one finds the keypoint already matched at the same distance."""
    a = make_projection_chain_case()
    mt = ORBmatcher(a["nnratio"], max_queries=256, max_db=256)
    launches, m_o = projection_host(mt, a)
    assert m_o[0] == 46 and m_o[2] == 47, m_o[:4]
    assert_path(mt, launches, "overflow")


@pytest.mark.parametrize("mp_only", [True, False])
@pytest.mark.parametrize("ori", [True, False])
def test_bow_chain_takes_the_fallback(mp_only, ori):
    """48 KF1 features of one vocabulary node whose nearest KF2 feature is the same: sequentially the first takes it and
    the others fall through vbMatched2 to the next ones."""
    k1, k2 = make_bow_case(seed=13, chain=48)
    mt = ORBmatcher(0.6, ori, max_queries=1024, max_db=1024)
    launches, m_o = bow_host(mt, k1, k2, mp_only, ori)
    chain = m_o[-48:]
    assert (chain >= 0).sum() >= 2 and len(set(chain[chain >= 0])) == (chain >= 0).sum()
    assert_path(mt, launches, "bow_overflow")


# ---------------------------------------------------------------------------------------------- large databases
@pytest.mark.parametrize("ndb,path", [(8192, "resolve"), (8193, "big"), (10000, "big"), (16384, "big_sequential")])
def test_window_large_database(ndb, path):
    """2000 queries against 8192 keypoints (the largest shared-memory grid), 8193 (the first global-memory grid), 10000
    (claim table of 2 slots per keypoint) and 16384 (no claim table: the sequential kernel alone)."""
    f1, f2, prev = make_big_window_case(61, 2000, ndb)
    mt = ORBmatcher(0.9, max_queries=2000, max_db=ndb)
    launches, m_o = window_host(mt, f1, f2, prev, GRID)
    assert (m_o >= 0).sum() > 500
    if path == "resolve":
        assert launches == 4 and mt.last_rounds()[0] >= 1
    else:
        assert_path(mt, launches, path)


@pytest.mark.parametrize("n_kf,path", [(10000, "big"), (16384, "big_sequential")])
def test_projection_large_database(n_kf, path):
    """2000 map points against a large keyframe, with order ties in one grid cell that the grid walk's order decides."""
    a, ties = make_big_projection_case(62, n_kf, 2000)
    mt = ORBmatcher(a["nnratio"], max_queries=2000, max_db=n_kf)
    launches, m_o = projection_host(mt, a)
    assert sum(m_o[b] >= 0 and m_o[a_] < 0 for b, a_ in ties) >= len(ties) // 2
    assert_path(mt, launches, path)


@pytest.mark.parametrize("mp_only,ori", [(True, True), (False, False)])
def test_bow_large_database(mp_only, ori):
    """2000 KF1 features against 16384 KF2 features: no claim table fits, the sequential kernel runs alone."""
    k1, k2 = make_bow_case(seed=14, n=2000, n2_extra=14384)
    mt = ORBmatcher(0.6, ori, max_queries=2048, max_db=16384)
    launches, m_o = bow_host(mt, k1, k2, mp_only, ori)
    assert (m_o >= 0).sum() > 200
    assert_path(mt, launches, "bow_sequential")


# ---------------------------------------------------------------------------------------------- device counts
def _poison_tail(a, count):
    """Entries past `count` become copies of real entries: a read past the count creates or changes a match."""
    a = a.copy()
    a[count:] = a[np.arange(count, len(a)) % count]
    return a


@pytest.mark.parametrize("n2_cap,n2,chain", [(1000, 700, False), (1000, 700, True), (9000, 6000, False)])
def test_window_device_counts_below_capacity(n2_cap, n2, chain):
    """se2gpu_match_by_window_device with *d_n1 / *d_n2 well below the capacities; keypoints, descriptors and vbPrevMatched
    past the counts are copies of real entries. chain: a steal chain inside the counted range (sequential fallback).
    n2_cap 9000: the global-memory grid."""
    import torch
    n1_cap, n1 = 1000, 600
    f1, f2, prev = make_big_window_case(63, n1_cap, n2_cap)
    kp1, d1, kp2, d2 = f1["kp"], f1["desc"], f2["kp"], f2["desc"]
    if chain:
        rng = np.random.default_rng(5)
        kp2["x"][0], kp2["y"][0], kp2["octave"][0] = 300.0, 200.0, 0
        for q in range(40):
            kp1["x"][q], kp1["y"][q], kp1["octave"][q] = 300.0 + 0.1 * q, 200.0, 0
            kp1["angle"][q] = np.float32((float(kp2["angle"][0]) - 7.0) % 360.0)
            d1[q] = d2[0]
            for b in rng.choice(256, 40 - q, replace=False):
                d1[q, b // 8] ^= np.uint8(1 << (b % 8))
        prev = np.stack([kp1["x"], kp1["y"]], axis=1).astype(np.float32)
    kp1, d1, prev = _poison_tail(kp1, n1), _poison_tail(d1, n1), _poison_tail(prev, n1)
    kp2, d2 = _poison_tail(kp2, n2), _poison_tail(d2, n2)
    n_o, m_o, prev_o = pyoracle.match_by_window(kp1[:n1], d1[:n1], kp2[:n2], d2[:n2], prev[:n1], GRID, 20, 1, 0, 8, 0.9)
    mt = ORBmatcher(0.9, max_queries=n1_cap, max_db=n2_cap)
    d_prev, d_m, d_nm = dev(prev), dev(np.full(n1_cap, 7, np.int32)), dev(np.zeros(1, np.int32))
    d_n = dev(np.array([n1, n2], np.int32))
    args = (dev(kp1), dev(d1), n1_cap, dev(kp2), dev(d2), n2_cap, d_prev, FrameView(None, None).grid(), 20, d_m, d_nm)
    _, launches = counted(lambda: mt.MatchByWindowDevice(*args, d_n1=d_n.data_ptr(), d_n2=d_n.data_ptr() + 4,
                                                         stream=torch.cuda.current_stream().cuda_stream))
    torch.cuda.synchronize()
    m_g, prev_g = d_m.cpu().numpy(), d_prev.cpu().numpy()
    assert int(d_nm.item()) == n_o and n_o > 200
    np.testing.assert_array_equal(m_g[:n1], m_o)
    assert (m_g[n1:] == -1).all()
    np.testing.assert_array_equal(prev_g[:n1], prev_o)
    np.testing.assert_array_equal(prev_g[n1:], prev[n1:])
    assert_path(mt, launches, "overflow" if chain else ("big" if n2_cap > 8192 else "resolve"))


@pytest.mark.parametrize("chain", [False, True])
def test_projection_device_counts_below_capacity(chain):
    """se2gpu_match_by_projection_device with *d_n_kf well below the capacity; keypoints and descriptors past it are copies
    of real entries, and matchesIdxMP past it must be -1."""
    import torch
    n_cap, n = 1000, 650
    a = make_projection_chain_case(seed=32, n=n_cap, nmp=600) if chain else make_projection_case(seed=33, n=n_cap, nmp=600)["args"]
    kp, desc = _poison_tail(a["kfkp"], n), _poison_tail(a["kfdesc"], n)
    obs = a["kf_observed"].copy()
    obs[n:] = 0
    ref = dict(a, kfkp=kp[:n], kfdesc=desc[:n], kf_observed=obs[:n])
    n_o, m_o = pyoracle.match_by_projection(**ref)
    mt = ORBmatcher(a["nnratio"], max_queries=600, max_db=n_cap)
    d_m, d_nm, d_n = dev(np.full(n_cap, 7, np.int32)), dev(np.zeros(1, np.int32)), dev(np.array([n], np.int32))
    args = (dev(kp), dev(desc), n_cap, dev(obs), dev(a["mp_valid"]), dev(a["mp_uv"]), len(a["mp_valid"]), dev(a["mp_octave"]),
            dev(a["mp_desc"]), FrameView(None, None).grid(), a["win_size"], a["level_offset"], d_m, d_nm)
    _, launches = counted(lambda: mt.MatchByProjectionDevice(*args, d_n_kf=d_n, stream=torch.cuda.current_stream().cuda_stream))
    torch.cuda.synchronize()
    m_g = d_m.cpu().numpy()
    assert int(d_nm.item()) == n_o and n_o > 100
    np.testing.assert_array_equal(m_g[:n], m_o)
    assert (m_g[n:] == -1).all()
    assert_path(mt, launches, "overflow" if chain else "resolve")


def _extract_then_match(nf, scale, nlevels, img1, img2, poison):
    """Extractor -> matcher in device memory, with device-side counts; the oracle runs on the keypoints the extractor wrote."""
    import torch
    from se2lam_b200.orb import ORBextractor
    e = ORBextractor(nf, scale, nlevels, max_batch=2)
    d_kps = torch.zeros(2 * nf * 28, dtype=torch.uint8, device="cuda:0")
    d_desc = torch.zeros(2 * nf * 32, dtype=torch.uint8, device="cuda:0")
    if poison:         # every slot past a frame's count holds a real keypoint of that frame
        for f, img in enumerate((img1, img2)):
            k, d = e(img)
            i = np.arange(nf) % len(k)
            d_kps[f * nf * 28:(f + 1) * nf * 28] = dev(k[i])
            d_desc[f * nf * 32:(f + 1) * nf * 32] = dev(d[i]).reshape(-1)
    d_counts = torch.zeros(2, dtype=torch.int32, device="cuda:0")
    s = torch.cuda.current_stream().cuda_stream
    e.extract_device(dev(np.stack([img1, img2])), 2, img1.shape[0], img1.shape[1], d_kps, d_desc, d_counts, stream=s)
    mt = ORBmatcher(0.9, max_queries=nf, max_db=nf)
    d_prev = torch.zeros(2 * nf, dtype=torch.float32, device="cuda:0")
    d_m = torch.full((nf,), 7, dtype=torch.int32, device="cuda:0")
    d_nm = torch.zeros(1, dtype=torch.int32, device="cuda:0")
    kp1, kp2 = d_kps.data_ptr(), d_kps.data_ptr() + nf * 28
    de1, de2 = d_desc.data_ptr(), d_desc.data_ptr() + nf * 32
    ORBmatcher.KeypointsToPointsDevice(kp1, nf, d_prev, d_n=d_counts.data_ptr(), stream=s)
    _, launches = counted(lambda: mt.MatchByWindowDevice(kp1, de1, nf, kp2, de2, nf, d_prev, FrameView(None, None).grid(), 20, d_m, d_nm,
                                                         d_n1=d_counts.data_ptr(), d_n2=d_counts.data_ptr() + 4, stream=s))
    torch.cuda.synchronize()
    c = d_counts.cpu().numpy()
    kps = d_kps.cpu().numpy().view(KP_DTYPE).reshape(2, nf)
    desc = d_desc.cpu().numpy().reshape(2, nf, 32)
    prev = np.stack([kps[0, :c[0]]["x"], kps[0, :c[0]]["y"]], axis=1).astype(np.float32)
    n_o, m_o, prev_o = pyoracle.match_by_window(kps[0, :c[0]], desc[0, :c[0]], kps[1, :c[1]], desc[1, :c[1]], prev, GRID, 20, 1, 0, 8, 0.9)
    m_g = d_m.cpu().numpy()
    assert int(d_nm.item()) == n_o
    np.testing.assert_array_equal(m_g[:c[0]], m_o)
    assert (m_g[c[0]:] == -1).all()
    np.testing.assert_array_equal(d_prev.cpu().numpy().reshape(-1, 2)[:c[0]], prev_o)
    return c, n_o, launches, mt


def test_extract_then_match_short_frames():
    """Frames that are constant but for a 160 x 160 textured patch give fewer keypoints than nfeatures; the extractor's
    buffers past the counts hold real keypoints beforehand."""
    img1 = np.full((480, 640), 128, np.uint8)
    img1[120:280, 200:360] = synth.orb_frame(1004)[120:280, 200:360]
    img2 = np.roll(img1, (3, -2), axis=(0, 1))
    c, n_o, launches, mt = _extract_then_match(1000, 1.2, 8, img1, img2, poison=True)
    assert c.max() < 1000, c
    assert n_o > 300
    assert_path(mt, launches, "resolve")


def test_extract_then_match_2000_queries():
    """ORBextractor(2000, 1.15, 6) on a frame and its shifted copy, 2000 x 2000 through the device buffers: k_resolve strides
    over more queries than its 1024 threads."""
    img1 = synth.orb_frame(1005)
    img2 = np.roll(img1, (-3, 4), axis=(0, 1))
    c, n_o, launches, mt = _extract_then_match(2000, 1.15, 6, img1, img2, poison=False)
    assert c.min() > 1500, c
    assert n_o > 600
    assert_path(mt, launches, "resolve")


# ---------------------------------------------------------------------------------------------- grid with a non-zero origin
@pytest.mark.parametrize("seed", [21, 23])
def test_window_on_undistorted_grid(seed):
    """Non-zero origin and non-round cells: keypoints outside the grid and exactly on half cells, windows outside the grid;
    through the host and the device entry points."""
    import torch
    f1, f2, prev, _ = make_grid_edge_pair(seed=seed)
    grid = FrameView(None, None, UNDIST_BOUNDS[0], UNDIST_BOUNDS[2], UNDIST_BOUNDS[1], UNDIST_BOUNDS[3]).grid()
    g = (np.float32(grid.min_x), np.float32(grid.min_y), np.float32(grid.inv_w), np.float32(grid.inv_h))
    mt = ORBmatcher(0.9, max_queries=1024, max_db=1024)
    launches, m_o = window_host(mt, f1, f2, prev, g, bounds=UNDIST_BOUNDS)
    assert (m_o >= 0).sum() > 300
    assert_path(mt, launches, "resolve")
    n = len(prev)
    _, _, prev_o = pyoracle.match_by_window(f1["kp"], f1["desc"], f2["kp"], f2["desc"], prev, g, 20, 1, 0, 8, 0.9)
    d_prev, d_m, d_nm = dev(prev), dev(np.full(n, 7, np.int32)), dev(np.zeros(1, np.int32))
    _, launches = counted(lambda: mt.MatchByWindowDevice(dev(f1["kp"]), dev(f1["desc"]), n, dev(f2["kp"]), dev(f2["desc"]), n, d_prev, grid,
                                                         20, d_m, d_nm, stream=torch.cuda.current_stream().cuda_stream))
    torch.cuda.synchronize()
    np.testing.assert_array_equal(d_m.cpu().numpy(), m_o)
    np.testing.assert_array_equal(d_prev.cpu().numpy().reshape(-1, 2), prev_o)
    assert int(d_nm.item()) == (m_o >= 0).sum()
    assert_path(mt, launches, "resolve")


@pytest.mark.parametrize("seed", [22, 24])
def test_projection_on_undistorted_grid(seed):
    """The same for MatchByProjection, with order ties that an even half cell decides (round() keeps A in B's cell)."""
    import torch
    c = make_projection_edge_case(seed=seed)
    a = c["args"]
    grid = FrameView(None, None, UNDIST_BOUNDS[0], UNDIST_BOUNDS[2], UNDIST_BOUNDS[1], UNDIST_BOUNDS[3]).grid()
    assert (np.float32(grid.min_x), np.float32(grid.min_y), np.float32(grid.inv_w), np.float32(grid.inv_h)) == a["grid"]
    mt = ORBmatcher(a["nnratio"], max_queries=1024, max_db=1024)
    launches, m_o = projection_host(mt, a, bounds=UNDIST_BOUNDS)
    assert all(m_o[b] == mp for (b, _), mp in zip(c["ties"], c["tie_mps"]))
    assert_path(mt, launches, "resolve")
    n, nmp = len(a["kfkp"]), len(a["mp_valid"])
    d_m, d_nm = dev(np.full(n, 7, np.int32)), dev(np.zeros(1, np.int32))
    _, launches = counted(lambda: mt.MatchByProjectionDevice(dev(a["kfkp"]), dev(a["kfdesc"]), n, dev(a["kf_observed"]), dev(a["mp_valid"]),
                                                             dev(a["mp_uv"]), nmp, dev(a["mp_octave"]), dev(a["mp_desc"]), grid,
                                                             a["win_size"], a["level_offset"], d_m, d_nm,
                                                             stream=torch.cuda.current_stream().cuda_stream))
    torch.cuda.synchronize()
    np.testing.assert_array_equal(d_m.cpu().numpy(), m_o)
    assert int(d_nm.item()) == (m_o >= 0).sum()
    assert_path(mt, launches, "resolve")


# ---------------------------------------------------------------------------------------------- default context
def test_default_context_regrowth():
    """Handle-less calls share one context per device, created at 2048 x 2048 and replaced by a larger one when a call
    needs it: 900 queries, then 3000, then 900 again."""
    for n in (900, 3000, 900):
        f1, f2, prev = make_frame_pair(seed=71 + n, n=n)
        n_o, m_o, prev_o = pyoracle.match_by_window(f1["kp"], f1["desc"], f2["kp"], f2["desc"], prev, GRID, 20, 1, 0, 8, 0.9)
        prev_g = prev.copy()
        (n_g, m_g), launches = counted(lambda: ORBmatcher(0.9).MatchByWindow(frame_view(f1), frame_view(f2), prev_g, 20))
        assert n_g == n_o and n_o > 100
        np.testing.assert_array_equal(m_g, m_o)
        np.testing.assert_array_equal(prev_g, prev_o)
        assert launches == 4, launches
