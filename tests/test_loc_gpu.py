"""The localization handle (se2lam_b200.loc, Localizer::run over B streams against a static device map) against the CPU
restatement (oracle/pyloc.py), teacher-forced: the oracle runs step t from the handle's pose after step t-1, so every
discrete output must be byte-identical and the pose agree to 1e-5."""
import numpy as np
import pytest

from oracle import pyloc
from tools import loc_scenes as ls

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")

_SCENE = {}


def scene():
    if not _SCENE:
        cfg = ls.config()
        m = ls.build_map(3, cfg)
        _SCENE.update(cfg=cfg, m=m)
    return _SCENE["cfg"], _SCENE["m"]


def _params(cfg, **kw):
    from se2lam_b200 import loc
    c = dict(cfg, **kw)
    return loc.params(c["nfeatures"], c["scale_factor"], c["nlevels"], c["K"], c["grid"], c["bounds"], c["cTb"], c["bTc"], c["huber"],
                      c["max_local_mps"], c["fast_th"], c["dist"])


def _map_arrays(m):
    from se2lam_b200.loc import MAP_FIELDS
    return {k: m[k] for k in MAP_FIELDS}


class Harness:
    """streams through a handle with one stream per stream given (frames up to max_w x max_h, default cfg's size) and one
    oracle per stream; stream b relocalizes at its frame 1 against its start keyframe. Each stream keeps its own frame
    counter, so a call may cover streams 0 .. B-1 only."""

    def __init__(self, streams, cfg, m, oracle=True, eager=False, max_w=None, max_h=None, **kw):
        from se2lam_b200.loc import Localizer, inv_level_sigma2
        self.cfg, self.m, self.streams, self.B = dict(cfg, **kw), m, streams, len(streams)
        self.h = Localizer(self.B, max_w or cfg["w"], max_h or cfg["h"], _params(cfg, **kw), _map_arrays(m))
        self.h.set_eager(eager)
        isig = inv_level_sigma2(cfg["scale_factor"], cfg["nlevels"])
        logic = pyloc.CppLogic(m)
        self.orc = [pyloc.LocOracle(self.cfg, m, isig, logic) for _ in streams] if oracle else None
        self.ks = [0] * self.B

    def step(self, B=None, layout=None):
        """one call over streams 0 .. B-1 (default all), each at its own next frame; layout(frames [B,h,w]) -> the array
        handed to the binding"""
        n = B or self.B
        ks = self.ks[:n]
        frames = np.stack([self.streams[b][0][ks[b]] for b in range(n)])
        odom = np.stack([self.streams[b][1][ks[b]] for b in range(n)])
        prev = [self.h.state(b)["Tcw"] for b in range(n)]
        rec = self.h.step(layout(frames) if layout else frames, odom)
        ref = None
        if self.orc:
            ref = [o.step(frames[b], odom[b], prev[b] if ks[b] else None) for b, o in enumerate(self.orc[:n])]
        for b in range(n):
            self.ks[b] += 1
        return rec, ref

    def relocalize(self, streams):
        kf = [self.streams[b][3] for b in streams]
        pairs = []
        for b, k in zip(streams, kf):
            st = self.h.state(b)
            pairs.append(ls.loop_matches(st["kp"], st["desc"], self.m, k))
        rec, first = self.h.relocalize(streams, kf, pairs)
        ref = None
        if self.orc:
            ref = [self.orc[b].relocalize(k, p, first[j]) for j, (b, k, p) in enumerate(zip(streams, kf, pairs))]
        return rec, first, ref


def close(a, b):
    return np.abs(np.asarray(a, np.float64) - b).max() <= 1e-5 * max(1.0, np.abs(b).max())


def compare(h, b, rec, ref, where):
    # the LM iteration count follows the BA's sums, which agree with the oracle to 1e-5 only (DESIGN.md section 9)
    got = {n: int(rec[n]) for n in rec.dtype.names if n not in ("Tcw", "ba_iterations")}
    want = {n: int(v) for n, v in ref.items() if n != "ba_iterations"}
    assert got == want, f"{where}: {got} != {want}"
    o = h.orc[b]
    assert close(rec["Tcw"], o.Tcw), f"{where}: Tcw {rec['Tcw']} vs {o.Tcw}"
    st = h.h.state(b)
    assert st["kp"].tobytes() == o.kp.tobytes() and st["desc"].tobytes() == o.desc.tobytes(), f"{where}: keypoints"
    assert st["obs_mp"].tobytes() == o.obs_mp.tobytes(), f"{where}: obs_mp"
    assert st["tracked"] == o.tracked, where
    if o.tracked:
        assert set(np.flatnonzero(st["local_kfs"]).tolist()) == o.local_kfs, f"{where}: local keyframes"
        assert st["local_mps"].tolist() == o.local_mps[:h.cfg["max_local_mps"]], f"{where}: local map points"


def check_step(h, rec, ref, k):
    """the records and state of the streams a call covered against their oracles; a stream lost during this step refuses
    a relocalization"""
    for b in range(len(rec)):
        compare(h, b, rec[b], ref[b], f"frame {k} stream {b}")
        if h.orc[b].branches[-1] == "lost_now":   # lost during this step: no loop search before the next frame
            with pytest.raises(Exception):
                h.h.relocalize([b], [0], [[]])


def check_relocalize(h, streams):
    rr, first, rref = h.relocalize(streams)
    for j, b in enumerate(streams):
        want, ofirst = rref[j]
        assert close(first[j], ofirst), f"stream {b}: pose after the first BA"
        compare(h, b, rr[j], want, f"relocalize stream {b}")
    return rr


def run(B, frames=30, eager=False, cfg=None, m=None, streams=None, layout=None, **kw):
    if cfg is None:
        cfg, m = scene()
    streams = streams or [ls.stream(200 + b, m, cfg, frames, ls.KINDS[b % len(ls.KINDS)]) for b in range(B)]
    h = Harness(streams, cfg, m, eager=eager, **kw)
    seen = set()
    for k in range(frames):
        rec, ref = h.step(layout=layout)
        check_step(h, rec, ref, k)
        if k == 1:
            check_relocalize(h, list(range(B)))
    for o in h.orc:
        seen |= set(o.branches)
    return h, seen


@pytest.mark.parametrize("B", [1, 8, 64])
def test_sequences_match_oracle(B):
    _, seen = run(B)
    assert {"first", "relocalized", "tracked"} <= seen, seen
    assert {"loop_null", "loop_badprl", "loop_repeat"} <= seen, seen
    if B >= 8:
        assert {"gated", "lost_now", "lost"} <= seen, seen


def test_batch_equals_single_streams():
    cfg, m = scene()
    streams = [ls.stream(300 + b, m, cfg, 12, ls.KINDS[b % len(ls.KINDS)]) for b in range(4)]
    hb = Harness(streams, cfg, m, oracle=False)
    hs = [Harness([s], cfg, m, oracle=False) for s in streams]
    for k in range(12):
        rb, _ = hb.step()
        r1 = [h.step()[0] for h in hs]
        if k == 1:
            rb, _, _ = hb.relocalize(list(range(4)))
            r1 = [h.relocalize([0])[0] for h in hs]
        for b in range(4):
            assert rb[b].tobytes() == r1[b][0].tobytes(), f"frame {k} stream {b}"
            sb, s1 = hb.h.state(b), hs[b].h.state(0)
            for key in ("kp", "obs_mp", "local_mps", "local_kfs", "Tcw"):
                assert np.asarray(sb[key]).tobytes() == np.asarray(s1[key]).tobytes(), f"frame {k} stream {b}: {key}"


def test_graph_replay_equals_eager_and_recaptures_on_new_size():
    cfg, m = scene()
    streams = [ls.stream(400 + b, m, cfg, 12, "along") for b in range(3)]
    hg, he = Harness(streams, cfg, m, oracle=False), Harness(streams, cfg, m, oracle=False, eager=True)
    for k in range(12):
        if k == 8:
            for h in (hg, he):
                h.streams = [(s[0][:, :200, :280].copy(),) + tuple(s[1:]) for s in h.streams]
        rg, _ = hg.step(); re_, _ = he.step()
        if k == 1:
            rg, _, _ = hg.relocalize([0, 1, 2]); re_, _, _ = he.relocalize([0, 1, 2])
        assert rg.tobytes() == re_.tobytes(), f"frame {k}"
        for b in range(3):
            sg, se = hg.h.state(b), he.h.state(b)
            for key in ("kp", "obs_mp", "local_mps", "local_kfs", "Tcw"):
                assert np.asarray(sg[key]).tobytes() == np.asarray(se[key]).tobytes(), f"frame {k} stream {b}: {key}"
    kernels, nodes = hg.h.graph_nodes()
    assert kernels > 5 and nodes >= kernels


def test_capacity_overflow_and_bad_input_change_nothing():
    from se2lam_b200._capi import Se2GpuError, LocResult, lib, ptr
    cfg, m = scene()
    streams = [ls.stream(500 + b, m, cfg, 6, "along") for b in range(2)]
    h = Harness(streams, cfg, m, max_local_mps=64)
    h.step(); h.step()
    before = [h.h.state(b) for b in range(2)]
    frames = np.stack([s[0][2] for s in streams]); odom = np.stack([s[1][2] for s in streams])
    out = (LocResult * 4)()
    L = lib()
    W, H = cfg["w"], cfg["h"]
    assert L.se2gpu_loc_step(h.h.h, 3, ptr(frames), 0, W, H, W, W * H, ptr(odom), out) == -4
    assert L.se2gpu_loc_step(h.h.h, 2, None, 0, W, H, W, W * H, ptr(odom), out) == -3
    with pytest.raises(Se2GpuError):
        h.h.relocalize([0, 0], [0, 0], [[], []])
    with pytest.raises(Se2GpuError):
        h.h.relocalize([0], [len(m["kf_kp_ptr"])], [[]])
    with pytest.raises(Se2GpuError):
        h.h.relocalize([0], [0], [[(5, 0), (3, 0)]])
    after = [h.h.state(b) for b in range(2)]
    for a, b in zip(before, after):
        for key in a:
            assert np.asarray(a[key]).tobytes() == np.asarray(b[key]).tobytes(), key
    # a local map past max_local_mps: the relocalization reports it, then every step over the stream is refused
    with pytest.raises(Se2GpuError):
        h.relocalize([0])
    st = h.h.state(0)
    assert st["overflow"]
    assert L.se2gpu_loc_step(h.h.h, 2, ptr(frames), 0, W, H, W, W * H, ptr(odom), out) == -4
    assert h.h.state(0)["Tcw"].tobytes() == st["Tcw"].tobytes()
