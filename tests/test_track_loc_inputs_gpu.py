"""The tracker (se2lam_b200.track) and the localization handle (se2lam_b200.loc) on the inputs their ABI promises beyond
one 320x240 packed batch: lens distortion of every supported length, padded and per-frame frame layouts from the host and
the device, calls over a prefix of the streams, frame sizes that re-prepare the extractor, and feature counts past the
matcher's full claim table and past a 1 024-thread keypoint round. Every comparison is the one of tests/test_tracker_gpu.py
(byte for byte against oracle/pytrack.py) or tests/test_loc_gpu.py (teacher-forced against oracle/pyloc.py)."""
import numpy as np
import pytest

from oracle import pyoracle
from tests.test_loc_gpu import Harness as LocHarness
from tests.test_loc_gpu import check_relocalize, check_step as loc_check, scene
from tests.test_loc_gpu import run as loc_run
from tests.test_tracker_gpu import Harness as TrackHarness
from tests.test_tracker_gpu import _params as track_params
from tests.test_tracker_gpu import check_step as track_check
from tests.test_tracker_gpu import mixed, run_against_oracle
from tools import loc_scenes as ls
from tools import track_scenes as ts

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")

BRANCHES = ("first_low", "gated", "new_kf", "abort", "cleared", "c1c2", "empty")


def _same_state(a, b, where):
    for key in a:
        assert np.asarray(a[key]).tobytes() == np.asarray(b[key]).tobytes(), f"{where}: {key}"


# ------------------------------------------------------------------------------------------------------- distortion
@pytest.mark.parametrize("n", sorted(ts.DISTORTION))
def test_tracker_distortion_matches_oracle(n):
    cfg = ts.config(dist=ts.DISTORTION[n])
    _, seen = run_against_oracle(mixed(8, 20, cfg), cfg, 20)
    for key in BRANCHES:
        assert seen.get(key, 0) > 0, f"no step reached branch {key}: {seen}"


def _loc_distorted_scene(n, **kw):
    cfg = ls.config(dist=ts.DISTORTION[n], **kw)
    orb = pyoracle.OrbOracle(cfg["nfeatures"], cfg["scale_factor"], cfg["nlevels"], cfg["fast_th"])
    m = ls.build_map(3, cfg, extract=lambda img: orb.extract(pyoracle.frame_image(img, cfg["K"], cfg["dist"])))
    return cfg, m


@pytest.mark.parametrize("n", sorted(ts.DISTORTION))
def test_localizer_distortion_matches_oracle(n):
    cfg, m = _loc_distorted_scene(n)
    _, seen = loc_run(4, 20, cfg=cfg, m=m)
    assert {"first", "relocalized", "tracked"} <= seen, seen


def test_distortion_graph_equals_eager_across_sizes():
    """the undistortion map is rebuilt for each frame size before the capture: replay and eager launches agree across
    320x240 -> 280x200 -> 320x240, and the replayed run matches the oracle"""
    cfg = ts.config(dist=ts.DISTORTION[12])
    full = mixed(4, 18, cfg)
    hg, he = TrackHarness(full, cfg), TrackHarness(full, cfg, oracle=False, eager=True)
    seen = {}
    for k in range(18):
        if k in (6, 12):
            for h in (hg, he):
                h.streams = [(s[0][:, :200, :280].copy() if k == 6 else s[0], s[1], s[2]) for s in full]
        rg, ref = hg.step(); re_, _ = he.step()
        track_check(hg, rg, ref, k, seen)
        assert rg.tobytes() == re_.tobytes(), f"frame {k}"
        for b in range(4):
            _same_state(hg.t.state(b), he.t.state(b), f"frame {k} stream {b}")


# ---------------------------------------------------------------------------------------------------- frame layouts
def _strided(frames, stride, fstride, device, size=None):
    """frames [B,h,w] copied into a buffer with the given row and frame strides and returned as a view of it"""
    B, h, w = frames.shape
    size = size or fstride * (B - 1) + stride * (h - 1) + w
    buf = np.full(size + 64, 0xA5, np.uint8)                # poison around and between the frames
    view = np.lib.stride_tricks.as_strided(buf, (B, h, w), (fstride, stride, 1))
    for b in range(B):
        for y in range(h):
            buf[b * fstride + y * stride:b * fstride + y * stride + w] = frames[b, y]
    if not device:
        return view
    d = torch.from_numpy(buf).cuda()
    return torch.as_strided(d, (B, h, w), (fstride, stride, 1))


def _crop_view(frames):
    """a CUDA view big[:, 1:h+1, 3:w+3] of a larger padded batch"""
    B, h, w = frames.shape
    big = torch.full((B, h + 5, w + 11), 0x5A, dtype=torch.uint8, device="cuda")
    big[:, 1:h + 1, 3:w + 3] = torch.from_numpy(frames).cuda()
    return big[:, 1:h + 1, 3:w + 3]


def _layouts():
    """name -> layout(frames); each passes its own row and frame strides through the binding"""
    out = {}
    for dev in (False, True):
        tag = "device" if dev else "host"
        out[f"padded_{tag}"] = lambda f, d=dev: _strided(f, f.shape[2] + 13, (f.shape[2] + 13) * f.shape[1], d)
        out[f"per_frame_{tag}"] = lambda f, d=dev: _strided(f, f.shape[2] + 13, (f.shape[2] + 13) * f.shape[1] + 4099, d)
        out[f"tightest_{tag}"] = lambda f, d=dev: _strided(f, f.shape[2] + 13, (f.shape[2] + 13) * (f.shape[1] - 1) + f.shape[2], d)
    out["cuda_view"] = _crop_view
    return out


def test_tracker_frame_layouts_equal_packed():
    cfg = ts.config()
    streams = mixed(4, 12, cfg)
    packed = TrackHarness(streams, cfg)
    lay = _layouts()
    hs = {name: TrackHarness(streams, cfg, oracle=False) for name in lay}
    one = TrackHarness(streams[:1], cfg, oracle=False)      # B = 1: any frame stride
    seen = {}
    for k in range(12):
        rec, ref = packed.step()
        track_check(packed, rec, ref, k, seen)
        for name, h in hs.items():
            r, _ = h.step(layout=lay[name])
            assert r.tobytes() == rec.tobytes(), f"{name} frame {k}"
            for b in range(4):
                _same_state(h.t.state(b), packed.t.state(b), f"{name} frame {k} stream {b}")
        r, _ = one.step(layout=lambda f: _strided(f, f.shape[2] + 3, 7, False, size=(f.shape[2] + 3) * f.shape[1]))
        assert r.tobytes() == rec[:1].tobytes(), f"B = 1 frame {k}"
        _same_state(one.t.state(0), packed.t.state(0), f"B = 1 frame {k}")


def _frame_args(cfg, B, k, streams, fstride_delta):
    w, h = cfg["w"], cfg["h"]
    stride = w + 13
    frames = np.stack([s[0][k] for s in streams[:B]])
    tight = stride * (h - 1) + w
    v = _strided(frames, stride, tight + fstride_delta, False, size=tight * B + stride * h)
    return v, stride, tight + fstride_delta, np.ascontiguousarray(np.stack([s[1][k] for s in streams[:B]]))


def test_overlapping_frames_are_refused_and_change_nothing():
    """a frame stride one byte below the tightest layout: SE2GPU_ERR_INVALID, records and state untouched"""
    from se2lam_b200._capi import LocResult, TrackKF, TrackResult, lib, ptr
    L = lib()
    cfg = ts.config()
    streams = mixed(2, 6, cfg)
    h = TrackHarness(streams, cfg, oracle=False)
    for _ in range(3):
        h.step()
    before = [h.t.state(b) for b in range(2)]
    v, stride, fs, odom = _frame_args(cfg, 2, 3, streams, -1)
    out = (TrackResult * 2)()
    for b in range(2):
        out[b].frame_id = 77
    kk = (TrackKF * 2)()
    for b, x in enumerate(h.kf(b) for b in range(2)):
        if x is not None:
            kk[b].d_observed, kk[b].d_view_mp = ptr(x["observed"]), ptr(x["view_mp"])
    base = v.ctypes.data
    assert L.se2gpu_tracker_step(h.t.h, 2, base, 0, cfg["w"], cfg["h"], stride, fs, ptr(odom), kk, out) == -3
    assert L.se2gpu_tracker_first(h.t.h, 2, base, 0, cfg["w"], cfg["h"], stride, fs, ptr(odom), out) == -3
    assert [out[b].frame_id for b in range(2)] == [77, 77]
    for b in range(2):
        _same_state(before[b], h.t.state(b), f"tracker stream {b}")
    lcfg, m = scene()
    lstreams = [ls.stream(600 + b, m, lcfg, 4, "along") for b in range(2)]
    lh = LocHarness(lstreams, lcfg, m, oracle=False)
    lh.step(); lh.step()
    lbefore = [lh.h.state(b) for b in range(2)]
    v, stride, fs, odom = _frame_args(lcfg, 2, 2, lstreams, -1)
    lout = (LocResult * 2)()
    lout[0].n_keypoints = lout[1].n_keypoints = 77
    assert L.se2gpu_loc_step(lh.h.h, 2, v.ctypes.data, 0, lcfg["w"], lcfg["h"], stride, fs, ptr(odom), lout) == -3
    assert lout[0].n_keypoints == lout[1].n_keypoints == 77
    for b in range(2):
        _same_state(lbefore[b], lh.h.state(b), f"localizer stream {b}")


def test_localizer_frame_layouts_equal_packed():
    cfg, m = scene()
    streams = [ls.stream(700 + b, m, cfg, 8, ls.KINDS[b % len(ls.KINDS)]) for b in range(4)]
    packed = LocHarness(streams, cfg, m)
    lay = _layouts()
    hs = {name: LocHarness(streams, cfg, m, oracle=False) for name in lay}
    one = LocHarness(streams[:1], cfg, m, oracle=False)      # B = 1: any frame stride
    for k in range(8):
        rec, ref = packed.step()
        loc_check(packed, rec, ref, k)
        for name, h in hs.items():
            assert h.step(layout=lay[name])[0].tobytes() == rec.tobytes(), f"{name} frame {k}"
        r1 = one.step(layout=lambda f: _strided(f, f.shape[2] + 3, 7, False, size=(f.shape[2] + 3) * f.shape[1]))[0]
        assert r1.tobytes() == rec[:1].tobytes(), f"B = 1 frame {k}"
        if k == 1:
            rr = check_relocalize(packed, list(range(4)))
            for name, h in hs.items():
                assert h.relocalize(list(range(4)))[0].tobytes() == rr.tobytes(), f"{name}: relocalize"
            assert one.relocalize([0])[0].tobytes() == rr[:1].tobytes(), "B = 1: relocalize"
        for name, h in list(hs.items()) + [("B = 1", one)]:
            for b in range(h.B):
                _same_state(h.h.state(b), packed.h.state(b), f"{name} frame {k} stream {b}")


# ------------------------------------------------------------------------------------------------------ sub-batches
SCHEDULE = [(8, False), (3, False), (8, False), (1, False), (5, False), (3, True), (8, False), (2, False), (8, False)]


def test_tracker_sub_batches():
    """calls over streams 0 .. B-1 of a tracker of 8: each stream's oracle advances only with the calls that cover it,
    the other streams' state keeps its bytes, first() on a prefix mid-sequence restarts exactly those streams, and
    eager launches equal the replayed graphs (recaptured at each change of B)"""
    cfg = ts.config()
    streams = mixed(8, 12, cfg)
    hg, he = TrackHarness(streams, cfg), TrackHarness(streams, cfg, oracle=False, eager=True)
    seen, untouched, restarted = {}, 0, 0
    for c, (B, first) in enumerate(SCHEDULE):
        before = [hg.t.state(b) for b in range(8)]
        rg, ref = hg.step(B=B, first=first or None)
        re_, _ = he.step(B=B, first=first or None)
        assert len(rg) == B and rg.tobytes() == re_.tobytes(), f"call {c}"
        track_check(hg, rg, ref, c, seen)
        if first:
            assert all(r["first"] for r in rg) and all(r["frame_id"] == 0 for r in rg)
            restarted += B
        for b in range(8):
            st = hg.t.state(b)
            _same_state(st, he.t.state(b), f"call {c} stream {b}: eager")
            if b >= B:
                _same_state(before[b], st, f"call {c} stream {b}: left out")
                untouched += 1
    assert untouched > 0 and restarted == 3


def test_localizer_sub_batches():
    cfg, m = scene()
    streams = [ls.stream(800 + b, m, cfg, 10, ls.KINDS[b % len(ls.KINDS)]) for b in range(8)]
    hg, he = LocHarness(streams, cfg, m), LocHarness(streams, cfg, m, oracle=False, eager=True)
    untouched = 0
    for c, (B, _) in enumerate(SCHEDULE):
        before = [hg.h.state(b) for b in range(8)]
        rg, ref = hg.step(B=B)
        re_, _ = he.step(B=B)
        assert len(rg) == B and rg.tobytes() == re_.tobytes(), f"call {c}"
        loc_check(hg, rg, ref, c)
        again = [b for b in range(B) if hg.ks[b] == 2]     # streams that just ran their frame 1
        if again:
            check_relocalize(hg, again)
            he.relocalize(again)
        for b in range(8):
            st = hg.h.state(b)
            _same_state(st, he.h.state(b), f"call {c} stream {b}: eager")
            if b >= B:
                _same_state(before[b], st, f"call {c} stream {b}: left out")
                untouched += 1
    assert untouched > 0
    seen = set().union(*(o.branches for o in hg.orc))
    assert {"first", "relocalized", "tracked"} <= seen, seen


# ------------------------------------------------------------------------------------------------------ frame sizes
SIZES = [(640, 480), (320, 240), (1280, 720), (637, 479), (640, 480)]


def test_tracker_frame_sizes():
    """a tracker made for 1280x720 driven at each size in turn, restarted with first() at each: the extractor's tables
    and level geometry are re-prepared before each capture"""
    cfg = ts.config(w=1280, h=720, fx=1200.0, min_frames=3)

    def streams(i):
        w, hh = SIZES[i]
        sc = dict(ts.config(w=w, h=hh, fx=1200.0 * w / 1280), nfeatures=cfg["nfeatures"])
        return [ts.stream(900 + 10 * i + b, 7, ts.KINDS[b], sc) for b in range(2)]

    h = TrackHarness(streams(0), cfg, max_w=1280, max_h=720)
    seen = {}
    for i in range(len(SIZES)):
        if i:
            h.streams = [(f, s[1], s[2]) for (f, _, _), s in zip(streams(i), h.streams)]
            h.ks = [0] * h.B
        for k in range(7):
            rec, ref = h.step()
            track_check(h, rec, ref, k, seen)
            assert rec[0]["n_keypoints"] > 0
    assert seen.get("gated", 0) > 0 and seen.get("new_kf", 0) > 0, seen


def test_localizer_640x480():
    cfg = ls.config(nfeatures=1000, w=640, h=480, fx=600.0, max_local_mps=4096)
    m = ls.build_map(5, cfg)
    _, seen = loc_run(2, 12, cfg=cfg, m=m, max_w=1280, max_h=720)
    assert {"first", "relocalized", "tracked"} <= seen, seen


# ---------------------------------------------------------------------------------------------- large feature counts
@pytest.mark.parametrize("nfeatures", [2000, 4000])
def test_tracker_large_feature_counts(nfeatures):
    """2 000 features keep the matcher's 16-wide claim table, 4 000 narrow it; more than 1 024 keypoints per frame"""
    cfg = ts.config(nfeatures=nfeatures, w=1280, h=720, fx=1200.0, fast_th=10, min_frames=4)
    h, seen = run_against_oracle(mixed(4, 12, cfg), cfg, 12)
    most = max(len(o.cur_kp) for o in h.orc)
    assert most > 1024, most
    assert seen.get("new_kf", 0) > 0 or seen.get("gated", 0) > 0, seen


def test_tracker_refuses_a_claim_table_below_two():
    """at 9 700 features even a claim table of width 2 overflows the matcher's shared memory (4 + K ints per keypoint
    against 227 KB less 2 KB on an H100): refused for that reason, not for a failed allocation, before the matcher
    allocates anything"""
    from se2lam_b200._capi import Se2GpuError
    from se2lam_b200.track import Tracker
    cfg = ts.config(nfeatures=9700)
    with pytest.raises(Se2GpuError, match="9700 features per frame are too many for the matcher's shared-memory resolve"):
        Tracker(1, cfg["w"], cfg["h"], track_params(cfg))


def test_localizer_dense_map_2000_features():
    """2 000 features on a dense map (tools/loc_bench.py's recipe: many keyframes close together, a small share of each
    one's keypoints made map points) with max_local_mps raised so no local map overflows: the edge scan walks two
    1 024-keypoint rounds per stream, and DoLocalBA has more than the 1 536 edges k_pose_ba stages in shared memory, so it
    reads them from each stream's global edge slot"""
    cfg = ls.config(nfeatures=2000, w=640, h=480, fx=600.0, fast_th=10, max_local_mps=8192)
    path = np.array([(0.012 * k - 0.3, 0.3 * np.sin(0.05 * k), 0.004 * k) for k in range(24)], np.float32)
    m = ls.build_map(11, cfg, share=0.15, path=path, min_shared=10)
    streams = [ls.stream(1000 + b, m, cfg, 6, "along") for b in range(2)]
    h = LocHarness(streams, cfg, m)
    most_edges = most_kp = 0
    for k in range(6):
        rec, ref = h.step()
        loc_check(h, rec, ref, k)
        for b, o in enumerate(h.orc):
            most_kp = max(most_kp, len(o.kp))
            if ref[b]["ba_status"] == 0:                    # DoLocalBA ran: one edge per observed usable map point
                obs = {int(j) for j in o.obs_mp if j >= 0}
                most_edges = max(most_edges, sum(1 for j in obs if not m["mp_null"][j] and m["mp_good_prl"][j]))
        if k == 1:
            check_relocalize(h, [0, 1])
    assert most_kp > 1024, most_kp
    assert most_edges > 1536, most_edges
    assert not any(h.h.state(b)["overflow"] for b in range(2))
