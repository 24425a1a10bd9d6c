"""The tracker (se2lam_b200.track, Track::mTrack over B camera streams with the state on the device) against the CPU
restatement of Track (oracle/pytrack.py) byte for byte: per-step records, decisions and the device state."""
import numpy as np
import pytest

from oracle import pytrack
from tools import track_scenes as ts

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")


def _params(cfg):
    from se2lam_b200 import track
    return track.params(cfg["nfeatures"], cfg["scale_factor"], cfg["nlevels"], cfg["K"], cfg["grid"], cfg["lower_depth"],
                        cfg["upper_depth"], cfg["cTb"], cfg["bTc"], cfg["odo_noise"], cfg["max_frames"], cfg["min_frames"],
                        cfg["fast_th"], cfg["dist"])


class Harness:
    """drives a tracker with one stream per stream given (frames up to max_w x max_h, default cfg's size) and one oracle
    per stream as Track::run and the caller's keyframe side would. Each stream keeps its own frame counter, so a call may
    cover streams 0 .. B-1 only."""

    def __init__(self, streams, cfg, oracle=True, eager=False, max_w=None, max_h=None):
        from se2lam_b200.track import Tracker
        self.cfg, self.streams, self.B = cfg, streams, len(streams)
        self.t = Tracker(self.B, max_w or cfg["w"], max_h or cfg["h"], _params(cfg))
        self.t.set_eager(eager)
        self.orc = [pytrack.TrackOracle(cfg) for _ in streams] if oracle else None
        self.dev = [dict(observed=torch.from_numpy(s[2]["observed"]).cuda(), view_mp=torch.from_numpy(s[2]["view_mp"]).cuda())
                    for s in streams]
        self.kf_odom = [None] * self.B
        self.ks = [0] * self.B

    def kf(self, b):
        s = self.streams[b][2]
        if self.kf_odom[b] is None:
            return None
        return dict(observed=self.dev[b]["observed"], view_mp=self.dev[b]["view_mp"], n_obs_mp=s["n_obs_mp"],
                    accept=bool(s["accept"][self.ks[b]]), odom=self.kf_odom[b])

    def step(self, device_frames=False, B=None, first=None, layout=None):
        """one call over streams 0 .. B-1 (default all), each at its own next frame; first: se2gpu_tracker_first (default:
        when every stream in the call is at its frame 0); layout(frames [B,h,w]) -> the array handed to the binding"""
        n = B or self.B
        ks = self.ks[:n]
        first = all(k == 0 for k in ks) if first is None else first
        frames = np.stack([self.streams[b][0][ks[b]] for b in range(n)])
        odom = np.stack([self.streams[b][1][ks[b]] for b in range(n)])
        if first:
            self.kf_odom[:n] = [None] * n
        kfs = [self.kf(b) for b in range(n)]
        fr = layout(frames) if layout else torch.from_numpy(frames).cuda() if device_frames else frames
        rec = self.t.first(fr, odom) if first else self.t.step(fr, odom, kfs if any(x is not None for x in kfs) else None)
        ref = None
        if self.orc:
            ref = []
            for b, o in enumerate(self.orc[:n]):
                kfo = None
                if kfs[b] is not None:
                    s = self.streams[b][2]
                    kfo = dict(observed=s["observed"], view_mp=s["view_mp"], n_obs_mp=s["n_obs_mp"], accept=kfs[b]["accept"],
                               odom=self.kf_odom[b])
                ref.append(o.first(frames[b], odom[b]) if first else o.step(frames[b], odom[b], kfo))
        new = [b for b in range(n) if rec[b]["new_kf"]]
        if new:
            self.t.reset(new, [self.dev[b]["view_mp"] for b in new])
            for b in new:
                self.kf_odom[b] = odom[b].copy()
                if self.orc:
                    self.orc[b].reset(self.streams[b][2]["view_mp"])
        for b in range(n):
            self.ks[b] += 1
        return rec, ref


def compare_state(h, b, where):
    st = h.t.state(b)
    o = h.orc[b]
    n = len(o.ref_kp)
    assert st["cur_kp"].tobytes() == o.cur_kp.tobytes(), f"{where}: current keypoints"
    assert st["cur_desc"].tobytes() == o.cur_desc.tobytes(), f"{where}: current descriptors"
    assert st["has_ref"] == o.has_ref and st["frame_id"] == o.frame_id, where
    assert st["local_mps"].tobytes() == o.local.tobytes(), f"{where}: mLocalMPs"
    assert st["good_prl"].tobytes() == o.good.tobytes(), f"{where}: mvbGoodPrl"
    if not o.has_ref:
        return
    assert st["ref_kp"].tobytes() == o.ref_kp.tobytes() and st["ref_desc"].tobytes() == o.ref_desc.tobytes(), f"{where}: reference"
    assert st["matches"].tobytes() == o.matches[:n].tobytes(), f"{where}: mMatchIdx"
    assert st["prev"][:n].tobytes() == o.prev[:n].tobytes(), f"{where}: mPrevMatched"
    assert st["Tcr"].tobytes() == o.Tcr.tobytes(), f"{where}: Tcr"
    assert st["pre_meas"].tobytes() == o.meas.tobytes() and st["pre_cov"].ravel(order="F").tobytes() == o.cov.tobytes(), f"{where}: preSE2"


def check_step(h, rec, ref, k, seen):
    """records and the state of the streams a call covered against their oracles; counts the branches reached in seen"""
    for b in range(len(rec)):
        got = {n: int(rec[b][n]) for n in rec.dtype.names}
        assert got == ref[b], f"frame {k} stream {b}: {got} != {ref[b]}"
        compare_state(h, b, f"frame {k} stream {b}")
        for key, hit in (("first_low", got["first"] and not got["new_kf"]), ("gated", not got["first"] and not got["triangulated"]),
                         ("new_kf", got["new_kf"] and not got["first"]), ("abort", got["abort_ba"]),
                         ("cleared", not got["first"] and got["n_matched"] > 0 and got["n_inlier"] == 0),
                         ("c1c2", got["new_kf"] and got["n_good_prl"] > 40), ("empty", got["n_keypoints"] == 0)):
            seen[key] = seen.get(key, 0) + bool(hit)


def run_against_oracle(streams, cfg, frames, device_frames=False, eager=False, layout=None, h=None):
    h = h or Harness(streams, cfg, eager=eager)
    seen = {}
    for k in range(frames):
        rec, ref = h.step(device_frames, layout=layout)
        check_step(h, rec, ref, k, seen)
    return h, seen


def mixed(B, frames, cfg):
    return [ts.stream(100 + b, frames, ts.KINDS[b % len(ts.KINDS)], cfg) for b in range(B)]


@pytest.mark.parametrize("B", [1, 8, 64])
def test_sequences_match_oracle(B):
    cfg = ts.config()
    _, seen = run_against_oracle(mixed(B, 30, cfg), cfg, 30)
    if B >= 8:
        for key in ("first_low", "gated", "new_kf", "abort", "cleared", "empty"):
            assert seen.get(key, 0) > 0, f"no step reached branch {key}: {seen}"


def test_every_branch_and_device_frames():
    cfg = ts.config()
    _, seen = run_against_oracle(mixed(len(ts.KINDS), 30, cfg), cfg, 30, device_frames=True)
    for key in ("first_low", "gated", "new_kf", "abort", "cleared", "c1c2", "empty"):
        assert seen.get(key, 0) > 0, f"no step reached branch {key}: {seen}"


def test_batch_equals_single_streams():
    cfg = ts.config()
    streams = mixed(8, 20, cfg)
    hb = Harness(streams, cfg, oracle=False)
    hs = [Harness([s], cfg, oracle=False) for s in streams]
    for k in range(20):
        rb, _ = hb.step()
        for b, h in enumerate(hs):
            r1, _ = h.step()
            assert rb[b].tobytes() == r1[0].tobytes(), f"frame {k} stream {b}"
            sb, s1 = hb.t.state(b), h.t.state(0)
            for key in ("cur_kp", "cur_desc", "ref_kp", "matches", "local_mps", "good_prl", "Tcr"):
                assert sb[key].tobytes() == s1[key].tobytes(), f"frame {k} stream {b}: {key}"


def test_graph_replay_equals_eager_and_recaptures_on_new_size():
    cfg = ts.config()
    streams = mixed(4, 16, cfg)
    hg, he = Harness(streams, cfg, oracle=False), Harness(streams, cfg, oracle=False, eager=True)
    for k in range(16):
        if k == 10:   # a smaller frame size from here on: a new capture
            for h in (hg, he):
                h.streams = [(s[0][:, :200, :280].copy(), s[1], s[2]) for s in h.streams]
        rg, _ = hg.step(); re_, _ = he.step()
        assert rg.tobytes() == re_.tobytes(), f"frame {k}"
        for b in range(4):
            sg, se = hg.t.state(b), he.t.state(b)
            for key in ("cur_kp", "cur_desc", "matches", "local_mps", "good_prl", "prev"):
                assert sg[key].tobytes() == se[key].tobytes(), f"frame {k} stream {b}: {key}"
    kernels, nodes = hg.t.graph_nodes()
    assert kernels > 5 and nodes >= kernels


def test_triangulation_batch_equals_single_calls():
    from se2lam_b200._capi import KP_DTYPE, lib, ptr
    rng = np.random.default_rng(5)
    B, cap = 6, 300
    K = np.array([[300, 0, 160], [0, 300, 120], [0, 0, 1]], np.float32)
    kp1 = np.zeros((B, cap), KP_DTYPE); kp2 = np.zeros((B, cap), KP_DTYPE)
    for a in (kp1, kp2):
        a["x"] = rng.uniform(0, 320, a.shape); a["y"] = rng.uniform(0, 240, a.shape)
    n = rng.integers(0, cap + 1, B).astype(np.int32)
    m = np.where(rng.random((B, cap)) < 0.7, rng.integers(0, cap, (B, cap)), -1).astype(np.int32)
    obs = (rng.random((B, cap)) < 0.2).astype(np.uint8)
    vm = rng.standard_normal((B, cap, 3)).astype(np.float32)
    T = np.tile(np.eye(4, dtype=np.float32), (B, 1, 1)); T[:, 0, 3] = rng.uniform(-0.3, 0.3, B)
    gate = np.array([1, 0, 1, 1, 0, 1], np.int32)
    lm0 = rng.standard_normal((B, cap, 3)).astype(np.float32)
    g = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()
    d = dict(kp1=g(kp1.view(np.uint8)), kp2=g(kp2.view(np.uint8)), n=g(n), m=g(m), obs=g(obs), vm=g(vm), T=g(T), gate=g(gate),
             K=g(K), lm=g(lm0), good=g(np.full((B, cap), 7, np.uint8)), c=g(np.zeros(2 * B, np.int32)))
    assert lib().se2gpu_track_triangulate_batch_device(B, ptr(d["kp1"]), cap, ptr(d["n"]), ptr(d["kp2"]), cap, ptr(d["m"]), ptr(d["obs"]),
                                                      ptr(d["vm"]), ptr(d["T"]), ptr(d["gate"]), ptr(d["K"]), 0.2, 10.0, 2,
                                                      ptr(d["lm"]), ptr(d["good"]), ptr(d["c"]), None) == 0
    torch.cuda.synchronize()
    for b in range(B):
        s = dict(kp1=g(kp1[b].view(np.uint8)), kp2=g(kp2[b].view(np.uint8)), n=g(n[b:b + 1]), m=g(m[b]), obs=g(obs[b]), vm=g(vm[b]),
                 T=g(T[b]), lm=g(lm0[b]), good=g(np.full(cap, 7, np.uint8)), c=g(np.zeros(2, np.int32)))
        if gate[b]:
            assert lib().se2gpu_track_triangulate_device(ptr(s["kp1"]), cap, ptr(s["n"]), ptr(s["kp2"]), ptr(s["m"]), ptr(s["obs"]),
                                                         ptr(s["vm"]), ptr(s["T"]), ptr(d["K"]), 0.2, 10.0, 2, ptr(s["lm"]),
                                                         ptr(s["good"]), ptr(s["c"]), None) == 0
        torch.cuda.synchronize()
        for key, k1 in (("m", "m"), ("lm", "lm"), ("good", "good")):
            assert d[key][b].cpu().numpy().tobytes() == s[k1].cpu().numpy().tobytes(), f"stream {b}: {key}"
        assert d["c"][2 * b:2 * b + 2].cpu().numpy().tolist() == (s["c"].cpu().numpy().tolist() if gate[b] else [0, 0])


def test_bad_input_changes_nothing():
    from se2lam_b200._capi import Se2GpuError, TrackKF, TrackResult, lib, ptr
    cfg = ts.config()
    streams = mixed(2, 12, cfg)
    h = Harness(streams, cfg, oracle=False)
    for _ in range(3):
        h.step()
    before = [h.t.state(b) for b in range(2)]
    frames = np.stack([s[0][3] for s in streams]); odom = np.stack([s[1][3] for s in streams])
    out = (TrackResult * 4)()
    L = lib()
    assert L.se2gpu_tracker_step(h.t.h, 3, ptr(frames), 0, ts.W, ts.H, ts.W, ts.W * ts.H, ptr(odom), None, out) == -4
    assert L.se2gpu_tracker_step(h.t.h, 2, None, 0, ts.W, ts.H, ts.W, ts.W * ts.H, ptr(odom), None, out) == -3
    assert L.se2gpu_tracker_step(h.t.h, 2, ptr(frames), 0, ts.W * 4, ts.H, ts.W * 4, ts.W * ts.H * 4, ptr(odom), None, out) == -4
    if any(h.kf_odom[b] is not None for b in range(2)):   # a tracking stream without its keyframe arrays
        assert L.se2gpu_tracker_step(h.t.h, 2, ptr(frames), 0, ts.W, ts.H, ts.W, ts.W * ts.H, ptr(odom), (TrackKF * 2)(), out) == -3
    with pytest.raises(Se2GpuError):
        h.t.reset([5], [h.dev[0]["view_mp"]])
    with pytest.raises(Se2GpuError):
        h.t.reset([0, 0], [h.dev[0]["view_mp"]] * 2)
    from se2lam_b200.track import Tracker
    fresh = Tracker(2, ts.W, ts.H, _params(cfg))
    with pytest.raises(Se2GpuError):   # no frame yet to become the reference
        fresh.reset([0], [h.dev[0]["view_mp"]])
    after = [h.t.state(b) for b in range(2)]
    for a, b in zip(before, after):
        for key in a:
            assert np.asarray(a[key]).tobytes() == np.asarray(b[key]).tobytes(), key
