"""GPU: KeyFrame::ComputeBoW and SearchByBoW over batches on the device (se2gpu_voc_compute_bow_device,
se2gpu_search_by_bow_batch_device) against the CPU oracles and the host entry points, bit for bit.

Keyframe b of a batch lies in slot b of every array (the extractor's layout); every slot past a keyframe's count holds
real data, so that a read past the count changes a result.
"""
import ctypes as C

import numpy as np
import pytest

from oracle import pybow, pyoracle
from se2lam_b200._capi import KP_DTYPE, lib
from se2lam_b200.bow import Vocabulary
from se2lam_b200.matcher import ORBmatcher
from tests.bow_cases import make_features, make_voc
from tests.matcher_cases import make_bow_case
from tools import synth

pytestmark = pytest.mark.gpu

ERR_INVALID, ERR_CAPACITY = -3, -4
RATIO = 0.6


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


def voc_handle(voc):
    return Vocabulary(voc["desc"], voc["child_ptr"], voc["children"], voc["word_id"], voc["weight"], voc["levels"])


# ---------------------------------------------------------------------------------------------- compute_bow
class BowOut:
    """The device outputs of compute_bow_device for B keyframes of cap slots, filled with a sentinel."""

    def __init__(self, B, cap, bow=True):
        import torch
        z = lambda *s, t=torch.int32: torch.full(s, 7, dtype=t, device="cuda:0")
        self.B, self.cap = B, cap
        self.word, self.value, self.nw = (z(B, cap), z(B, cap, t=torch.float64), z(B)) if bow else (None, None, None)
        self.node, self.ptr, self.feat, self.nn = z(B, cap), z(B, cap + 1), z(B, cap), z(B)

    def run(self, v, d_desc, d_n, levelsup):
        v.compute_bow_device(self.B, d_desc, self.cap, self.node, self.ptr, self.feat, self.nn, self.word, self.value, self.nw,
                             d_n=d_n, levelsup=levelsup, stream=stream())

    def keyframe(self, b):
        """keyframe b as the oracle's dict (the arrays up to their counts)"""
        k = int(host(self.nn)[b])
        ptr = host(self.ptr)[b, :k + 1]
        out = dict(node=host(self.node)[b, :k], ptr=ptr, feat=host(self.feat)[b, :ptr[-1]])
        if self.word is not None:
            w = int(host(self.nw)[b])
            out.update(word=host(self.word)[b, :w], value=host(self.value)[b, :w])
        return out

    def arrays(self):
        return [host(t) for t in (self.word, self.value, self.nw, self.node, self.ptr, self.feat, self.nn) if t is not None]


def assert_keyframe(got, want, bow=True):
    keys = ("word", "value", "node", "ptr", "feat") if bow else ("node", "ptr", "feat")
    for k in keys:
        assert got[k].tobytes() == np.ascontiguousarray(want[k]).astype(got[k].dtype).tobytes(), k


def host_transform(v, desc, levelsup):
    """Vocabulary.transform's host assembly as arrays"""
    bv, fv = v.transform(desc, levelsup)
    nodes = list(fv)
    return dict(word=np.asarray(list(bv), np.int32), value=np.asarray(list(bv.values()), np.float64), node=np.asarray(nodes, np.int32),
                ptr=np.cumsum([0] + [len(fv[n]) for n in nodes]).astype(np.int32), feat=np.asarray([i for n in nodes for i in fv[n]], np.int32))


@pytest.mark.parametrize("k,levels,ragged,levelsup,cap", [(10, 4, False, 2, 1000), (10, 6, False, 4, 2000), (7, 5, True, 3, 700),
                                                          (40, 2, False, 1, 300), (7, 5, True, 2, 700)])
def test_compute_bow_matches_the_oracle(k, levels, ragged, levelsup, cap):
    """The vocabulary shapes of test_voc_transform, and its ragged tree at a level some leaves are above (node -1); keyframes with 0, 1, cap, cap - 37
    and cap / 2 features, and a copy of the first with a third of its descriptors repeated (duplicate words). The BowVector
    bytes and the FeatureVector equal the oracle's and Vocabulary.transform's; the FeatureVector-only call writes the same
    FeatureVector; a NULL count array runs every keyframe at cap."""
    import torch
    voc = make_voc(k, levels, seed=levels, ragged=ragged)
    v = voc_handle(voc)
    counts = np.array([cap, 0, 1, cap, cap - 37, cap // 2, cap], np.int32)
    B = len(counts)
    desc = np.stack([make_features(voc, cap, seed=100 + b) for b in range(B)])
    desc[3] = desc[0]
    desc[3, 1::3] = desc[0, 0::3][: len(desc[3, 1::3])]
    d_desc, d_n = dev(desc), dev(counts)
    out = BowOut(B, cap)
    assert counted(lambda: out.run(v, d_desc, d_n, levelsup)) == 2
    fv_only = BowOut(B, cap, bow=False)
    assert counted(lambda: fv_only.run(v, d_desc, d_n, levelsup)) == 2
    full = BowOut(B, cap)
    full.run(v, d_desc, None, levelsup)
    torch.cuda.synchronize()
    minus1 = False
    for b in range(B):
        n = counts[b]
        want = pybow.compute_bow(voc, desc[b, :n], levelsup)
        got = out.keyframe(b)
        assert_keyframe(got, want)
        assert_keyframe(fv_only.keyframe(b), want, bow=False)
        assert_keyframe(got, host_transform(v, desc[b, :n], levelsup))
        assert_keyframe(full.keyframe(b), pybow.compute_bow(voc, desc[b], levelsup))
        minus1 |= bool((got["node"] == -1).any())
        if n > 100:
            assert abs(got["value"].sum() - 1.0) < 1e-12 and len(got["word"]) < n
    assert out.keyframe(1)["ptr"].tolist() == [0] and len(out.keyframe(1)["word"]) == 0
    assert minus1 == (ragged and levelsup == 2), minus1


def test_compute_bow_stopped_words_and_reuse():
    """A vocabulary with half its leaves stopped (weight 0) and one with all of them stopped (no word, no node), a second call of
    a smaller batch on the same handle (no new scratch), and a larger one after it (grown scratch)."""
    import torch
    voc = make_voc(8, 4, seed=4)
    half, none = dict(voc), dict(voc)
    half["weight"] = voc["weight"].copy(); none["weight"] = voc["weight"].copy()
    leaves = np.flatnonzero(voc["word_id"] >= 0)
    half["weight"][leaves[::2]] = 0.0
    none["weight"][leaves] = 0.0
    cap = 500
    for vd in (half, none):
        v = voc_handle(vd)
        for B in (5, 2, 9):
            counts = np.array([cap - 50 * (b % 4) for b in range(B)], np.int32)
            desc = np.stack([make_features(vd, cap, seed=200 + b) for b in range(B)])
            out = BowOut(B, cap)
            out.run(v, dev(desc), dev(counts), 2)
            torch.cuda.synchronize()
            for b in range(B):
                want = pybow.compute_bow(vd, desc[b, :counts[b]], 2)
                assert_keyframe(out.keyframe(b), want)
                if vd is none:
                    assert len(want["word"]) == 0 and want["ptr"].tolist() == [0]


# ---------------------------------------------------------------------------------------------- SearchByBoW batch
def side(kfs, cap, seed=0):
    """Keyframe dicts (make_bow_case's) -> host arrays in slots of cap: keypoints with the angle, descriptors, has_mp and the
    FeatureVector; every slot past a keyframe's entries filled with copies of real entries."""
    rng = np.random.default_rng(seed)
    S = len(kfs)
    kp = np.zeros((S, cap), KP_DTYPE); desc = rng.integers(0, 256, (S, cap, 32), dtype=np.uint8)
    mp = (rng.random((S, cap)) < 0.5).astype(np.uint8)
    node = np.full((S, cap), 1 << 30, np.int32); ptr = np.zeros((S, cap + 1), np.int32); feat = np.zeros((S, cap), np.int32)
    nn = np.zeros(S, np.int32)
    for s_, k in enumerate(kfs):
        n, K = len(k["angle"]), len(k["node"])
        kp["angle"][s_] = rng.uniform(0, 360, cap).astype(np.float32)
        kp["angle"][s_, :n] = k["angle"]; kp["x"][s_] = rng.uniform(0, 640, cap); desc[s_, :n] = k["desc"]; mp[s_, :n] = k["has_mp"]
        if n:
            desc[s_, n:] = k["desc"][np.arange(cap - n) % n]
        node[s_, :K] = k["node"]; ptr[s_, :K + 1] = k["ptr"]; ptr[s_, K + 1:] = k["ptr"][-1]; feat[s_, :len(k["feat"])] = k["feat"]
        nn[s_] = K
    return dict(kp=kp, desc=desc, has_mp=mp, node=node, ptr=ptr, feat=feat, n_node=nn, cap=cap)


def dev_side(s, has_mp=True):
    t = {k: dev(v) for k, v in s.items() if k != "cap"}
    return t, ORBmatcher.BowBatchSide(t["kp"], t["desc"], s["cap"], t["node"], t["ptr"], t["feat"], t["n_node"],
                                      has_mp=t["has_mp"] if has_mp else None)


def batched(mt, B, side1, side2, cap1, slot2=None, mp_only=True, has_mp=True):
    import torch
    t1, k1 = dev_side(side1, has_mp)
    t2, k2 = dev_side(side2, has_mp)
    d_m, d_nm = dev(np.full((B, cap1), 7, np.int32)), dev(np.full(B, 7, np.int32))
    d_slot = dev(np.asarray(slot2, np.int32)) if slot2 is not None else None
    launches = counted(lambda: mt.SearchByBoWBatchDevice(B, k1, k2, d_m, d_nm, d_slot2=d_slot, bIfMPOnly=mp_only, stream=stream()))
    torch.cuda.synchronize()
    return host(d_m), host(d_nm), launches


def bow_pairs():
    """eight pairs: seeds, the steal chain that overflows the claim table, a pair with no common node, an empty FeatureVector
    on side 1 and a keyframe without features on side 2"""
    pairs = [make_bow_case(seed=s_) for s_ in (3, 4, 5, 6)]
    pairs.append(make_bow_case(seed=13, chain=48))
    a, b = make_bow_case(seed=7)
    b = dict(b, node=b["node"] + 100000)
    pairs.append((a, b))
    a, b = make_bow_case(seed=8)
    pairs.append((dict(a, node=a["node"][:0], ptr=a["ptr"][:1], feat=a["feat"][:0]), b))
    a, b = make_bow_case(seed=9)
    e = np.zeros(0, np.int32)
    pairs.append((a, dict(angle=np.zeros(0, np.float32), desc=np.zeros((0, 32), np.uint8), has_mp=np.zeros(0, np.uint8), node=e,
                          ptr=np.zeros(1, np.int32), feat=e)))
    return pairs


def check_pairs(pairs, m_b, nm_b, mp_only, ori, host_mt):
    for b, (k1, k2) in enumerate(pairs):
        n1 = len(k1["angle"])
        n_o, m_o = pyoracle.search_by_bow(k1, k2, mp_only, RATIO, ori)
        assert nm_b[b] == n_o, (b, nm_b[b], n_o)
        np.testing.assert_array_equal(m_b[b, :n1], m_o)
        assert (m_b[b, n1:] == -1).all(), b
        n_h, m_h = host_mt.SearchByBoW(k1, k2, mp_only)
        assert n_h == n_o and np.array_equal(m_h, m_o), b


@pytest.mark.parametrize("mp_only,ori", [(1, 1), (1, 0), (0, 1), (0, 0)])
def test_search_by_bow_batch_of_eight_pairs(mp_only, ori):
    """Every pair equals the oracle and the host entry; the chain pair alone takes the sequential fallback; four launches."""
    pairs = bow_pairs()
    cap1 = max(len(k1["angle"]) for k1, _ in pairs)
    cap2 = max(len(k2["angle"]) for _, k2 in pairs)
    s1, s2 = side([p[0] for p in pairs], cap1, 1), side([p[1] for p in pairs], cap2, 2)
    mt = ORBmatcher(RATIO, bool(ori), max_queries=cap1, max_db=cap2, max_batch=8)
    m_b, nm_b, launches = batched(mt, 8, s1, s2, cap1, mp_only=mp_only, has_mp=bool(mp_only))
    assert launches == 4
    rounds, fallback = mt.last_rounds_batch(8)
    assert fallback.tolist() == [False] * 4 + [True] + [False] * 3, fallback
    assert (nm_b[:5] > 20).all() and (nm_b[5:] == 0).all(), nm_b
    check_pairs(pairs, m_b, nm_b, mp_only, bool(ori), ORBmatcher(RATIO, bool(ori), max_queries=cap1, max_db=cap2))


def test_search_by_bow_batch_large_database():
    """Side-2 keyframes of 16 384 and 6 000 features (n2_extra): no claim table at cap2 = 16 384, so the resolve is not
    launched (three launches) and every pair runs the sequential kernel."""
    pairs = [make_bow_case(seed=14, n=2000, n2_extra=14384), make_bow_case(seed=15, n=1500, n2_extra=4500)]
    cap1, cap2 = 2000, 16384
    s1, s2 = side([p[0] for p in pairs], cap1, 3), side([p[1] for p in pairs], cap2, 4)
    mt = ORBmatcher(RATIO, True, max_queries=cap1, max_db=cap2, max_batch=2)
    m_b, nm_b, launches = batched(mt, 2, s1, s2, cap1)
    assert launches == 3
    rounds, fallback = mt.last_rounds_batch(2)
    assert fallback.all() and (rounds == 0).all(), (fallback, rounds)
    check_pairs(pairs, m_b, nm_b, True, True, ORBmatcher(RATIO, True, max_queries=cap1, max_db=cap2))


def test_search_by_bow_batch_slot2():
    """Five side-2 keyframes matched by eleven pairs through d_slot2 give the results of side-2 copies laid out per pair."""
    base = [make_bow_case(seed=s_) for s_ in (21, 22, 23, 24, 25)]
    slot2 = [3, 0, 0, 4, 1, 2, 3, 3, 1, 4, 0]
    B = len(slot2)
    pairs = [(make_bow_case(seed=30 + b)[0] if b % 2 else base[slot2[b]][0], base[slot2[b]][1]) for b in range(B)]
    cap1 = max(len(p[0]["angle"]) for p in pairs); cap2 = max(len(k["angle"]) for _, k in base)
    s1 = side([p[0] for p in pairs], cap1, 5)
    mt = ORBmatcher(RATIO, True, max_queries=cap1, max_db=cap2, max_batch=B)
    m_s, nm_s, l_s = batched(mt, B, s1, side([k for _, k in base], cap2, 6), cap1, slot2=slot2)
    m_c, nm_c, l_c = batched(mt, B, s1, side([p[1] for p in pairs], cap2, 6), cap1)
    assert l_s == l_c == 4
    assert m_s.tobytes() == m_c.tobytes() and nm_s.tobytes() == nm_c.tobytes()
    check_pairs(pairs, m_s, nm_s, True, True, ORBmatcher(RATIO, True, max_queries=cap1, max_db=cap2))


# ---------------------------------------------------------------------------------------------- chain, launches, capture
def test_extract_compute_bow_search_on_device():
    """2B frames through se2gpu_orb_extract_device, one compute_bow_device over all of them, then the pair batch (frame b
    against frame B + b through d_slot2) as the extractor left its buffers: the oracle chain on the downloaded keypoints and
    descriptors gives the same FeatureVectors and matches, and nothing is copied between host and device in between."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    from se2lam_b200.orb import ORBextractor
    B, nf, H, W, levelsup = 8, 1000, 480, 640, 2
    voc = make_voc(10, 4, seed=4)
    v = voc_handle(voc)
    ref = [synth.orb_frame(4000 + b) for b in range(B)]
    cur = [np.roll(f, (1 + b % 3, -2 + b % 5), axis=(0, 1)) for b, f in enumerate(ref)]
    e = ORBextractor(nf, 1.2, 8, max_batch=2 * B)
    d_kps = torch.zeros(2 * B * nf * 28, dtype=torch.uint8, device="cuda:0")
    d_desc = torch.zeros(2 * B * nf * 32, dtype=torch.uint8, device="cuda:0")
    d_cnt = torch.zeros(2 * B, dtype=torch.int32, device="cuda:0")
    e.extract_device(dev(np.stack(ref + cur)), 2 * B, H, W, d_kps, d_desc, d_cnt, stream=stream())
    mp = dev((np.random.default_rng(9).random((2 * B, nf)) < 0.7).astype(np.uint8))
    out = BowOut(2 * B, nf, bow=False)
    mt = ORBmatcher(RATIO, True, max_queries=nf, max_db=nf, max_batch=B)
    side_ = ORBmatcher.BowBatchSide(d_kps, d_desc, nf, out.node, out.ptr, out.feat, out.nn, has_mp=mp)
    slot2 = dev(np.arange(B, 2 * B, dtype=np.int32))
    d_m, d_nm = dev(np.full((B, nf), 7, np.int32)), dev(np.full(B, 7, np.int32))
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        out.run(v, d_desc, d_cnt, levelsup)
        mt.SearchByBoWBatchDevice(B, side_, side_, d_m, d_nm, d_slot2=slot2, stream=stream())
        torch.cuda.synchronize()
    copies = [ev.name for ev in prof.events() if "Memcpy" in ev.name and ("HtoD" in ev.name or "DtoH" in ev.name)]
    assert not copies, copies
    c = host(d_cnt)
    kps = host(d_kps).view(KP_DTYPE).reshape(2 * B, nf)
    dsc = host(d_desc).reshape(2 * B, nf, 32)
    hm = host(mp)
    kf = []
    for f in range(2 * B):
        n = c[f]
        want = pybow.compute_bow(voc, dsc[f, :n], levelsup)
        assert_keyframe(out.keyframe(f), want, bow=False)
        kf.append(dict(angle=kps[f, :n]["angle"], desc=dsc[f, :n], has_mp=hm[f, :n], node=want["node"], ptr=want["ptr"], feat=want["feat"]))
    m, nm = host(d_m), host(d_nm)
    for b in range(B):
        n_o, m_o = pyoracle.search_by_bow(kf[b], kf[B + b], True, RATIO, True)
        assert nm[b] == n_o and n_o > 20, (b, nm[b], n_o)
        np.testing.assert_array_equal(m[b, :c[b]], m_o)
        assert (m[b, c[b]:] == -1).all()


def test_launch_counts_and_graph_capture():
    """Two launches for compute_bow and four for the pair batch at B = 1, 8 and 64, each pair equal to its B = 8 result; a
    CUDA graph captured from both calls replays to the eager outputs."""
    import torch
    voc = make_voc(10, 3, seed=3)
    v = voc_handle(voc)
    cap, base = 600, 8
    desc8 = np.stack([make_features(voc, cap, seed=300 + b) for b in range(2 * base)])
    flips = np.random.default_rng(2)
    desc8[base:] = desc8[:base] ^ (flips.integers(0, 256, desc8[:base].shape, dtype=np.uint8) &
                                   flips.integers(0, 256, desc8[:base].shape, dtype=np.uint8) &
                                   flips.integers(0, 256, desc8[:base].shape, dtype=np.uint8) &
                                   flips.integers(0, 256, desc8[:base].shape, dtype=np.uint8))   # the pair's keyframe seen again
    cnt8 = np.array([cap - 23 * b for b in range(2 * base)], np.int32)
    mt = ORBmatcher(RATIO, True, max_queries=cap, max_db=cap, max_batch=64)
    kp = np.zeros((2 * 64, cap), KP_DTYPE)
    kp["angle"] = np.random.default_rng(1).uniform(0, 360, kp.shape).astype(np.float32)
    kp[base:2 * base] = kp[:base]
    results = {}
    for B in (1, 8, 64):
        idx = np.concatenate([np.arange(B) % base, base + np.arange(B) % base])
        d_desc, d_n, d_kp = dev(desc8[idx]), dev(cnt8[idx]), dev(kp[idx])
        out = BowOut(2 * B, cap, bow=False)
        assert counted(lambda: out.run(v, d_desc, d_n, 3)) == 2
        side_ = ORBmatcher.BowBatchSide(d_kp, d_desc, cap, out.node, out.ptr, out.feat, out.nn)
        slot2 = dev(np.arange(B, 2 * B, dtype=np.int32))
        d_m, d_nm = dev(np.full((B, cap), 7, np.int32)), dev(np.full(B, 7, np.int32))
        assert counted(lambda: mt.SearchByBoWBatchDevice(B, side_, side_, d_m, d_nm, d_slot2=slot2, bIfMPOnly=False,
                                                         stream=stream())) == 4
        torch.cuda.synchronize()
        results[B] = (host(d_m), host(d_nm))
        if B == 8:
            eager = out.arrays() + [host(d_m), host(d_nm)]
            for t in (out.node, out.ptr, out.feat, out.nn, d_m, d_nm):
                t.fill_(7)
            g = torch.cuda.CUDAGraph()
            s_ = torch.cuda.Stream()
            s_.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(s_):
                with torch.cuda.graph(g, stream=s_):
                    out.run(v, d_desc, d_n, 3)
                    mt.SearchByBoWBatchDevice(B, side_, side_, d_m, d_nm, d_slot2=slot2, bIfMPOnly=False, stream=stream())
            torch.cuda.synchronize()
            for t in (out.node, out.ptr, out.feat, out.nn, d_m, d_nm):
                t.fill_(7)
            g.replay()
            torch.cuda.synchronize()
            replay = out.arrays() + [host(d_m), host(d_nm)]
            assert all(a.tobytes() == b_.tobytes() for a, b_ in zip(eager, replay))
    m8, nm8 = results[8]
    assert (nm8 > 20).all(), nm8
    for B in (1, 64):
        m, nm = results[B]
        for b in range(B):
            assert m[b].tobytes() == m8[b % base].tobytes() and nm[b] == nm8[b % base], (B, b)


# ---------------------------------------------------------------------------------------------- errors
def test_errors_leave_the_handles_usable():
    """Capacities above the context's or the assembly's shared memory are SE2GPU_ERR_CAPACITY; B < 0, NULL required pointers
    and a partial BowVector output set are SE2GPU_ERR_INVALID. A refused call launches nothing and writes nothing, and the
    next call on the same handles is right. B = 0 does nothing."""
    import torch
    L = lib()
    pairs = [make_bow_case(seed=s_) for s_ in (41, 42, 43, 44)]
    cap1 = max(len(p[0]["angle"]) for p in pairs); cap2 = max(len(p[1]["angle"]) for p in pairs)
    s1, s2 = side([p[0] for p in pairs], cap1, 7), side([p[1] for p in pairs], cap2, 8)
    mt = ORBmatcher(RATIO, True, max_queries=cap1, max_db=cap2, max_batch=4)
    host_mt = ORBmatcher(RATIO, True, max_queries=cap1, max_db=cap2)
    t1, k1 = dev_side(s1)
    t2, k2 = dev_side(s2)
    m, nm = dev(np.full((4, cap1), 7, np.int32)), dev(np.full(4, 7, np.int32))
    h, sp = C.c_void_p(mt.h), C.c_void_p(stream())

    def search(B, a=k1, b=k2, out=m, mp_only=1):
        return L.se2gpu_search_by_bow_batch_device(h, B, C.byref(a) if a is not None else None, C.byref(b) if b is not None else None,
                                                   None, mp_only, RATIO, 1, out.data_ptr() if out is not None else None, nm.data_ptr(), sp)

    def with_(k, **kw):
        f = {n: getattr(k, n) for n, _ in k._fields_}
        f.update(kw)
        return type(k)(**f)

    def good():
        m_b, nm_b, _ = batched(mt, 4, s1, s2, cap1)
        check_pairs(pairs, m_b, nm_b, True, True, host_mt)

    voc = make_voc(10, 3, seed=3)
    v = voc_handle(voc)
    cap = 500
    desc = np.stack([make_features(voc, cap, seed=500 + b) for b in range(3)])
    d_desc, d_n = dev(desc), dev(np.array([cap, 10, 0], np.int32))
    out = BowOut(3, cap)

    def bow(B=3, c=cap, word=out.word, value=out.value, nw=out.nw, node=out.node, ptr=out.ptr):
        p = lambda t: t.data_ptr() if t is not None else None
        return L.se2gpu_voc_compute_bow_device(C.c_void_p(v.h), B, d_desc.data_ptr(), c, d_n.data_ptr(), 2, p(word), p(value), p(nw),
                                               p(node), p(ptr), p(out.feat), p(out.nn), sp)

    def good_bow():
        out.run(v, d_desc, d_n, 2)
        torch.cuda.synchronize()
        for b, n in enumerate((cap, 10, 0)):
            assert_keyframe(out.keyframe(b), pybow.compute_bow(voc, desc[b, :n], 2))

    good()
    good_bow()
    failing = [(lambda: search(5), ERR_CAPACITY), (lambda: search(2, a=with_(k1, cap=cap1 + 1)), ERR_CAPACITY),
               (lambda: search(2, b=with_(k2, cap=cap2 + 1)), ERR_CAPACITY), (lambda: search(-1), ERR_INVALID),
               (lambda: search(2, a=with_(k1, cap=-1)), ERR_INVALID), (lambda: search(2, a=None), ERR_INVALID),
               (lambda: search(2, out=None), ERR_INVALID), (lambda: search(2, a=with_(k1, kp=None)), ERR_INVALID),
               (lambda: search(2, b=with_(k2, feat=None)), ERR_INVALID), (lambda: search(2, b=with_(k2, n_node=None)), ERR_INVALID),
               (lambda: search(2, a=with_(k1, has_mp=None)), ERR_INVALID),
               (lambda: L.se2gpu_search_by_bow_batch_device(None, 1, C.byref(k1), C.byref(k2), None, 1, RATIO, 1, None, None, None), ERR_INVALID),
               (lambda: bow(c=7000), ERR_CAPACITY), (lambda: bow(B=-1), ERR_INVALID), (lambda: bow(value=None), ERR_INVALID),
               (lambda: bow(node=None), ERR_INVALID), (lambda: bow(ptr=None), ERR_INVALID),
               (lambda: L.se2gpu_voc_compute_bow_device(None, 1, None, cap, None, 2, None, None, None, None, None, None, None, None),
                ERR_INVALID)]
    for k, (call, code) in enumerate(failing):
        m.fill_(7); nm.fill_(7)
        for t in (out.word, out.value, out.nw, out.node, out.ptr, out.feat, out.nn):
            t.fill_(7)
        assert counted(call) == 0, k
        assert call() == code, k
        torch.cuda.synchronize()
        assert (host(m) == 7).all() and (host(nm) == 7).all(), k
        assert all((a == 7).all() for a in out.arrays()), k
        good()
        good_bow()
    assert search(2, a=with_(k1, has_mp=None), mp_only=0) == 0              # has_mp may be NULL when mp_only == 0
    assert counted(lambda: search(0, a=with_(k1, kp=None))) == 0 and search(0, a=with_(k1, kp=None)) == 0
    assert bow(B=0, word=None, value=None, nw=None, node=None, ptr=None) == 0
