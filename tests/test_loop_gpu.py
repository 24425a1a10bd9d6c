"""GPU: loop closure on the device (se2gpu_detect_loop_device, se2gpu_verify_loop_device) against the CPU oracle chain
(oracle/pyloop.py) and DBoW2's own scores (tests/golden/l1_score_golden.npz), byte for byte."""
import ctypes as C

import numpy as np
import pytest

from oracle import pybow, pyloop
from se2lam_b200 import loop as gl
from se2lam_b200._capi import KP_DTYPE, lib
from se2lam_b200.matcher import ORBmatcher
from tests import loop_cases as lc
from tests.bow_cases import make_features, make_voc
from tests.test_bow_batch_gpu import BowOut, counted, dev, host, stream, voc_handle
from tests.test_loop_oracle import golden

pytestmark = pytest.mark.gpu

ERR_INVALID, ERR_CAPACITY = -3, -4


def bows(vecs, cap):
    w = np.full((len(vecs), cap), 7, np.int32); v = np.full((len(vecs), cap), 0.5); n = np.zeros(len(vecs), np.int32)
    for k, (a, b) in enumerate(vecs):
        w[k, :len(a)] = a; v[k, :len(a)] = b; n[k] = len(a)
    return w, v, n


class Detect:
    """device inputs and sentinel-filled outputs of one detect call"""

    def __init__(self, q, db, q_id=None, db_id=None, cap_q=None, cap_db=None):
        import torch
        self.B, self.N = len(q[2]), len(db[2])
        self.cap_q, self.cap_db = cap_q or q[0].shape[1], cap_db or db[0].shape[1]
        self.q = [dev(a) for a in q]; self.db = [dev(a) for a in db]
        self.q_id = dev(q_id) if q_id is not None else None
        self.db_id = dev(db_id) if db_id is not None else None
        self.scores = torch.full((max(self.B * self.N, 1),), 7.0, dtype=torch.float64, device="cuda:0")
        self.loop = torch.full((self.B,), 7, dtype=torch.int32, device="cuda:0")
        self.best = torch.full((self.B,), 7.0, dtype=torch.float64, device="cuda:0")

    def run(self, params):
        gl.detect_loop_device(self.B, *self.q, self.cap_q, self.N, *self.db, self.cap_db, self.scores, self.loop, self.best,
                              d_q_id=self.q_id, d_db_id=self.db_id, params=params, stream=stream())

    def out(self):
        import torch
        torch.cuda.synchronize()
        return host(self.scores)[:self.B * self.N].reshape(self.B, self.N), host(self.loop), host(self.best)


def assert_detect(d, q, db, q_id, db_id, params):
    scores, loop, best = d.out()
    s_o, l_o, b_o = pyloop.detect(*q, *db, q_id, db_id, params)
    assert scores.tobytes() == s_o.tobytes()
    assert loop.tobytes() == l_o.tobytes() and best.tobytes() == b_o.tobytes(), (loop, l_o, best, b_o)
    return scores, loop, best


def test_detect_scores_equal_dbow2_golden():
    pairs, want = golden()
    cap = max(max(len(a[0]), len(b[0])) for a, b in pairs)
    q, db = bows([a for a, _ in pairs], cap), bows([b for _, b in pairs], cap)
    d = Detect(q, db)
    d.run(gl.DETECT_LOCALIZER)
    scores, _, _ = assert_detect(d, q, db, None, None, gl.DETECT_LOCALIZER)
    assert np.diagonal(scores).copy().tobytes() == want.tobytes()


def synthetic_db(B, N, cap, seed):
    """N keyframes of up to cap words from a 20 000-word vocabulary; query b shares part of keyframe (37 b mod N)'s words,
    some queries and keyframes are empty, and two keyframes are copies (equal scores)"""
    rng = np.random.default_rng(seed)
    db = [lc.random_bow(rng, int(rng.integers(1, cap + 1)), vocab=20000) for _ in range(N)]
    if N > 3:
        db[1] = (np.zeros(0, np.int32), np.zeros(0)); db[3] = db[2]
    q = []
    for b in range(B):
        w, _ = db[(37 * b) % N]
        keep = w[rng.random(len(w)) < 0.6]
        extra = rng.choice(20000, max(0, min(cap - len(keep), 40)), replace=False)
        ww = np.unique(np.concatenate([keep, extra]))[:cap].astype(np.int32)
        v = rng.uniform(0.1, 1, len(ww))
        q.append((ww, v / v.sum()))
    if B > 2:
        q[2] = (np.zeros(0, np.int32), np.zeros(0))
    return q, db


@pytest.mark.parametrize("B,N", [(1, 1), (1, 37), (8, 37), (64, 37), (1, 2000), (8, 2000), (64, 2000)])
def test_detect_sizes(B, N):
    q, db = synthetic_db(B, N, 300, seed=B * 7 + N)
    qa, da = bows(q, 300), bows(db, 300)
    q_id = np.arange(B, dtype=np.int32) * 13 % max(N, 1); db_id = np.arange(N, dtype=np.int32)
    d = Detect(qa, da, q_id, db_id)
    for params in (gl.DETECT_GLOBAL_MAPPER, gl.DETECT_LOCALIZER, (3, 0.0)):
        assert counted(lambda: d.run(params)) == 2
        _, loop, _ = assert_detect(d, qa, da, q_id, db_id, params)
    assert N < 37 or (loop >= 0).sum() >= B // 2


def test_detect_query_at_the_shared_memory_limit():
    """cap_q = 19 370 words (12 bytes each in 227 KB) is accepted, one more is SE2GPU_ERR_CAPACITY"""
    import torch
    cap = torch.cuda.get_device_properties(0).shared_memory_per_block_optin // 12
    rng = np.random.default_rng(9)
    q = [lc.random_bow(rng, cap, vocab=400000), lc.random_bow(rng, 500, vocab=400000)]
    db = [lc.random_bow(rng, int(n), vocab=400000) for n in (cap, 1, 3000, 0, 20000)]
    cd = max(len(a) for a, _ in db)
    qa, da = bows(q, cap), bows(db, cd)
    d = Detect(qa, da)
    d.run(gl.DETECT_LOCALIZER)
    assert_detect(d, qa, da, None, None, gl.DETECT_LOCALIZER)
    L = lib()
    params = gl.LoopDetectParams(0, 0.05)
    rc = L.se2gpu_detect_loop_device(2, d.q[0].data_ptr(), d.q[1].data_ptr(), d.q[2].data_ptr(), cap + 1, d.N, d.db[0].data_ptr(),
                                     d.db[1].data_ptr(), d.db[2].data_ptr(), cd, None, None, C.byref(params), d.scores.data_ptr(),
                                     d.loop.data_ptr(), d.best.data_ptr(), C.c_void_p(stream()))
    assert rc == ERR_CAPACITY


@pytest.mark.parametrize("k,levels,ragged", [(10, 4, False), (7, 5, True), (10, 6, False)])
def test_detect_on_compute_bow_vectors(k, levels, ragged):
    """BowVectors compute_bow_device writes, of the bow_cases vocabulary shapes: keyframes that see one scene again score it
    highest"""
    import torch
    voc = make_voc(k, levels, seed=levels, ragged=ragged)
    v = voc_handle(voc)
    N, B, cap = 40, 8, 500
    desc = np.stack([make_features(voc, cap, seed=900 + n) for n in range(N)])
    qd = desc[(np.arange(B) * 5) % N].copy()
    rng = np.random.default_rng(4)
    qd ^= (rng.integers(0, 256, qd.shape, dtype=np.uint8) & rng.integers(0, 256, qd.shape, dtype=np.uint8) &
           rng.integers(0, 256, qd.shape, dtype=np.uint8) & rng.integers(0, 256, qd.shape, dtype=np.uint8))
    outs = []
    for dsc in (qd, desc):
        o = BowOut(len(dsc), cap)
        o.run(v, dev(dsc), None, 2)
        outs.append(o)
    torch.cuda.synchronize()
    q_id = (np.arange(B) * 5 + 3).astype(np.int32); db_id = np.arange(N, dtype=np.int32)
    for params in (gl.DETECT_GLOBAL_MAPPER, gl.DETECT_LOCALIZER):
        d = Detect([host(outs[0].word), host(outs[0].value), host(outs[0].nw)], [host(outs[1].word), host(outs[1].value), host(outs[1].nw)],
                   q_id, db_id)
        d.q = [outs[0].word, outs[0].value, outs[0].nw]; d.db = [outs[1].word, outs[1].value, outs[1].nw]
        d.run(params)
        qa = [host(outs[0].word), host(outs[0].value), host(outs[0].nw)]; da = [host(outs[1].word), host(outs[1].value), host(outs[1].nw)]
        for b in range(B):
            assert pybow.compute_bow(voc, qd[b], 2)["word"].tolist() == qa[0][b, :qa[2][b]].tolist()
        _, loop, _ = assert_detect(d, qa, da, q_id, db_id, params)
        if params == gl.DETECT_LOCALIZER:
            assert (loop == (np.arange(B) * 5) % N).mean() > 0.5, loop


# ---------------------------------------------------------------------------------------------- verify
def verify_side(kfs, cap, seed):
    """keyframe dicts (tests/loop_cases.loop_pair's) -> slots of cap: keypoints (x, y, angle), descriptors, hasObservation as
    has_mp and the FeatureVector; every slot past a keyframe's entries holds copies of real ones"""
    from tests.test_bow_batch_gpu import side
    s = side([dict(k, has_mp=k["obs"]) for k in kfs], cap, seed)
    for i, k in enumerate(kfs):
        n = len(k["angle"])
        if n:
            s["kp"]["x"][i] = k["x"][np.arange(cap) % n]; s["kp"]["y"][i] = k["y"][np.arange(cap) % n]
            s["kp"]["angle"][i, :n] = k["angle"]
    return s


def verify_cases():
    pairs = [lc.loop_pair(s) for s in (3, 4, 6)] + [lc.loop_pair(5, collinear=True)]
    a, b = lc.loop_pair(7, n=300)
    pairs.append((a, dict(b, node=b["node"] + 100001)))                   # no common node: no raw match
    a, b = lc.loop_pair(8, n=60, outliers=0.0)
    pairs.append((a, b))                                                   # a small pair
    return pairs


def run_verify(mt, pairs, loop, params, n_mps, cap1=None, cap2=None):
    import torch
    B = len(pairs)
    cap1 = cap1 or max(len(p[0]["angle"]) for p in pairs); cap2 = cap2 or max(len(p[1]["angle"]) for p in pairs)
    s1 = verify_side([p[0] for p in pairs], cap1, 1)
    map_kfs = [pairs[j][1] for j in range(B)]
    s2 = verify_side(map_kfs, cap2, 2)
    from tests.test_bow_batch_gpu import dev_side
    t1, k1 = dev_side(s1); t2, k2 = dev_side(s2)
    z = lambda *sh, t=torch.int32: torch.full(sh, 7, dtype=t, device="cuda:0")
    o = dict(raw=z(B, cap1), good=z(B, cap1), mp=z(B, cap1), counts=z(B, 3), verified=z(B, t=torch.uint8))
    d_loop = dev(np.asarray(loop, np.int32)); d_n = dev(np.asarray(n_mps, np.int32))
    launches = counted(lambda: gl.verify_loop_device(mt, B, k1, k2, d_loop, o["raw"], o["good"], o["mp"], o["counts"], o["verified"],
                                                     d_n_mps_cur=d_n, params=params, stream=stream()))
    torch.cuda.synchronize()
    return {k: host(t) for k, t in o.items()}, launches, (t1, t2, k1, k2, d_loop, d_n, o)


def check_verify(out, pairs, loop, params, n_mps):
    for b, (cur, _) in enumerate(pairs):
        n1 = len(cur["angle"])
        if loop[b] < 0:
            assert (out["raw"][b] == -1).all() and (out["good"][b] == -1).all() and (out["mp"][b] == -1).all()
            assert out["counts"][b].tolist() == [0, 0, 0] and out["verified"][b] == 0
            continue
        raw, good, mp, counts, ok = pyloop.verify(cur, pairs[loop[b]][1], params, n_mps[b])
        assert out["raw"][b, :n1].tolist() == raw.tolist(), b
        assert out["good"][b, :n1].tolist() == good.tolist(), b
        assert out["mp"][b, :n1].tolist() == mp.tolist(), b
        assert (out["raw"][b, n1:] == -1).all() and (out["good"][b, n1:] == -1).all() and (out["mp"][b, n1:] == -1).all()
        assert out["counts"][b].tolist() == counts.tolist() and bool(out["verified"][b]) == ok, (b, out["counts"][b], counts)


@pytest.mark.parametrize("params", [gl.VERIFY_GLOBAL_MAPPER, gl.VERIFY_LOCALIZER])
def test_verify_matches_the_oracle_chain(params):
    """raw, good, MP, counts and verdict of every pair equal the oracle chain; a pair with d_loop = -1 is empty; the
    collinear pair's RANSAC finds no model; a pair with no common node has no raw match"""
    pairs = verify_cases()
    B = len(pairs)
    loop = list(range(B)); loop[2] = -1
    n_mps = [500, 5000, 300, 0, 400, 0]
    mt = ORBmatcher(0.6, True, max_queries=800, max_db=800, max_batch=B)
    out, launches, _ = run_verify(mt, pairs, loop, params, n_mps)
    assert launches == 6
    check_verify(out, pairs, loop, params, n_mps)
    c = out["counts"]
    assert c[3, 0] > 100 and c[3, 1] == 0 and c[4, 0] == 0
    assert out["verified"][0] == 1 and out["verified"][3] == 0


def test_verify_pairs_through_d_loop():
    """map keyframes in other slots than their queries: d_loop picks the slot, and a query against the wrong scene fails"""
    p = verify_cases()[:4]
    # slot j of the map holds the j-th of these loop keyframes; query b is matched against slot loop[b]
    both = [(p[0][0], p[2][1]), (p[1][0], p[3][1]), (p[3][0], p[1][1]), (p[2][0], p[0][1])]
    loop = [3, -1, 1, 0]
    mt = ORBmatcher(0.6, True, max_queries=800, max_db=800, max_batch=4)
    out, _, _ = run_verify(mt, both, loop, gl.VERIFY_GLOBAL_MAPPER, [500] * 4)
    check_verify(out, both, loop, gl.VERIFY_GLOBAL_MAPPER, [500] * 4)
    assert out["verified"].tolist() == [1, 0, 0, 1], out["counts"]


def test_negative_slot2_gives_an_empty_pair():
    from tests.matcher_cases import make_bow_case
    from tests.test_bow_batch_gpu import batched, side
    pairs = [make_bow_case(seed=s_) for s_ in (3, 4, 5)]
    cap1 = max(len(p[0]["angle"]) for p in pairs); cap2 = max(len(p[1]["angle"]) for p in pairs)
    s1, s2 = side([p[0] for p in pairs], cap1, 1), side([p[1] for p in pairs], cap2, 2)
    mt = ORBmatcher(0.6, True, max_queries=cap1, max_db=cap2, max_batch=3)
    m, nm, launches = batched(mt, 3, s1, s2, cap1, slot2=[0, -1, 2])
    m0, nm0, _ = batched(mt, 3, s1, s2, cap1)
    assert launches == 4
    assert (m[1] == -1).all() and nm[1] == 0 and nm0[1] > 20
    assert m[0].tobytes() == m0[0].tobytes() and m[2].tobytes() == m0[2].tobytes() and nm[[0, 2]].tolist() == nm0[[0, 2]].tolist()


# ---------------------------------------------------------------------------------------------- chain, launches, capture
def test_extract_compute_bow_detect_verify_on_device():
    """ORB -> compute_bow_device (map and queries) -> detect -> verify with no host copy in between equals the oracle chain
    on the downloaded keypoints and descriptors"""
    import torch
    from torch.profiler import ProfilerActivity, profile
    from se2lam_b200.orb import ORBextractor
    from tools import synth
    M, B, nf, H, W = 12, 4, 1000, 480, 640
    voc = make_voc(10, 4, seed=4)
    v = voc_handle(voc)
    maps = [synth.orb_frame(5000 + k) for k in range(M)]
    qs = [np.roll(maps[(3 * b + 1) % M], (2 + b, -3 + b), axis=(0, 1)) for b in range(B)]
    e = ORBextractor(nf, 1.2, 8, max_batch=M + B)
    d_kps = torch.zeros((M + B) * nf * 28, dtype=torch.uint8, device="cuda:0")
    d_desc = torch.zeros((M + B) * nf * 32, dtype=torch.uint8, device="cuda:0")
    d_cnt = torch.zeros(M + B, dtype=torch.int32, device="cuda:0")
    obs = dev((np.random.default_rng(3).random((M + B, nf)) < 0.6).astype(np.uint8))
    n_mps = dev(np.full(B, 400, np.int32))
    ids = dev(np.concatenate([np.arange(M) * 3, np.array([40, 41, 42, 25])]).astype(np.int32))
    e.extract_device(dev(np.stack(maps + qs)), M + B, H, W, d_kps, d_desc, d_cnt, stream=stream())
    torch.cuda.synchronize()
    bo = BowOut(M + B, nf)
    mt = ORBmatcher(0.6, True, max_queries=nf, max_db=nf, max_batch=B)
    scores = torch.zeros(B * M, dtype=torch.float64, device="cuda:0")
    loop = torch.zeros(B, dtype=torch.int32, device="cuda:0"); best = torch.zeros(B, dtype=torch.float64, device="cuda:0")
    z = lambda *sh, t=torch.int32: torch.full(sh, 7, dtype=t, device="cuda:0")
    o = dict(raw=z(B, nf), good=z(B, nf), mp=z(B, nf), counts=z(B, 3), verified=z(B, t=torch.uint8))
    q_off = lambda t, per: t.view(-1)[M * per:]
    map_side = ORBmatcher.BowBatchSide(d_kps, d_desc, nf, bo.node, bo.ptr, bo.feat, bo.nn, has_mp=obs)
    cur_side = ORBmatcher.BowBatchSide(q_off(d_kps, nf * 28), q_off(d_desc, nf * 32), nf, q_off(bo.node, nf), q_off(bo.ptr, nf + 1),
                                       q_off(bo.feat, nf), q_off(bo.nn, 1), has_mp=q_off(obs, nf))
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        bo.run(v, d_desc, d_cnt, 4)
        gl.detect_loop_device(B, q_off(bo.word, nf), q_off(bo.value, nf), q_off(bo.nw, 1), nf, M, bo.word, bo.value, bo.nw, nf,
                              scores, loop, best, d_q_id=q_off(ids, 1), d_db_id=ids, params=gl.DETECT_GLOBAL_MAPPER, stream=stream())
        gl.verify_loop_device(mt, B, cur_side, map_side, loop, o["raw"], o["good"], o["mp"], o["counts"], o["verified"],
                              d_n_mps_cur=n_mps, params=gl.VERIFY_GLOBAL_MAPPER, stream=stream())
        torch.cuda.synchronize()
    copies = [ev.name for ev in prof.events() if "Memcpy" in ev.name and ("HtoD" in ev.name or "DtoH" in ev.name)]
    assert not copies, copies
    c = host(d_cnt); kps = host(d_kps).view(KP_DTYPE).reshape(M + B, nf); dsc = host(d_desc).reshape(M + B, nf, 32)
    hobs = host(obs); hid = host(ids)
    kf = []
    for f in range(M + B):
        want = pybow.compute_bow(voc, dsc[f, :c[f]], 4)
        kf.append(dict(want, angle=kps[f, :c[f]]["angle"], x=kps[f, :c[f]]["x"], y=kps[f, :c[f]]["y"], desc=dsc[f, :c[f]],
                       obs=hobs[f, :c[f]]))
    qa = bows([(kf[M + b]["word"], kf[M + b]["value"]) for b in range(B)], nf)
    da = bows([(kf[k]["word"], kf[k]["value"]) for k in range(M)], nf)
    s_o, l_o, b_o = pyloop.detect(*qa, *da, hid[M:], hid[:M], gl.DETECT_GLOBAL_MAPPER)
    assert host(scores).reshape(B, M).tobytes() == s_o.tobytes()
    lp = host(loop)
    assert lp.tobytes() == l_o.tobytes() and host(best).tobytes() == b_o.tobytes()
    assert lp[:3].tolist() == [1, 4, 7] and lp[3] != 10, lp        # query 3's scene is 5 ids away: excluded
    out = {k: host(t) for k, t in o.items()}
    for b in range(B):
        n1 = c[M + b]
        if lp[b] < 0:
            assert out["counts"][b].tolist() == [0, 0, 0]
            continue
        raw, good, mp, counts, ok = pyloop.verify(kf[M + b], kf[lp[b]], gl.VERIFY_GLOBAL_MAPPER, 400)
        assert out["raw"][b, :n1].tolist() == raw.tolist() and out["good"][b, :n1].tolist() == good.tolist(), b
        assert out["mp"][b, :n1].tolist() == mp.tolist() and out["counts"][b].tolist() == counts.tolist(), b
        assert bool(out["verified"][b]) == ok
    assert out["verified"][:3].all(), out["counts"]


def test_launch_counts_and_graph_capture():
    """two launches for detect and six for verify at B = 1, 8 and 64, each query's result equal to its B = 8 one; a CUDA
    graph captured from both replays to the eager bytes"""
    import torch
    base = verify_cases()[:4]
    N = 37
    q, db = synthetic_db(8, N, 300, seed=5)
    results = {}
    mt = ORBmatcher(0.6, True, max_queries=800, max_db=800, max_batch=64)
    for B in (1, 8, 64):
        idx = np.arange(B) % 8
        qa = bows([q[i] for i in idx], 300); da = bows(db, 300)
        d = Detect(qa, da, (idx * 3).astype(np.int32), np.arange(N, dtype=np.int32))
        assert counted(lambda: d.run(gl.DETECT_GLOBAL_MAPPER)) == 2
        pairs = [base[i % 4] for i in range(B)]
        loop = [(i % 4) if i % 4 != 1 else -1 for i in range(B)]
        out, launches, keep = run_verify(mt, pairs, loop, gl.VERIFY_GLOBAL_MAPPER, [500] * B)
        assert launches == 6
        results[B] = (d.out(), out)
        if B == 8:
            t1, t2, k1, k2, d_loop, d_n, o = keep
            eager = [host(d.scores), host(d.loop), host(d.best)] + [host(t) for t in o.values()]
            for t in [d.scores, d.best] + list(o.values()) + [d.loop]:
                t.fill_(7)
            g = torch.cuda.CUDAGraph()
            s_ = torch.cuda.Stream()
            s_.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(s_):
                with torch.cuda.graph(g, stream=s_):
                    d.run(gl.DETECT_GLOBAL_MAPPER)
                    gl.verify_loop_device(mt, B, k1, k2, d_loop, o["raw"], o["good"], o["mp"], o["counts"], o["verified"],
                                          d_n_mps_cur=d_n, params=gl.VERIFY_GLOBAL_MAPPER, stream=stream())
            torch.cuda.synchronize()
            for t in [d.scores, d.best] + list(o.values()) + [d.loop]:
                t.fill_(7)
            g.replay()
            torch.cuda.synchronize()
            replay = [host(d.scores), host(d.loop), host(d.best)] + [host(t) for t in o.values()]
            assert all(a.tobytes() == b_.tobytes() for a, b_ in zip(eager, replay))
    (s8, l8, b8), o8 = results[8]
    for B in (1, 64):
        (s, l, bb), o = results[B]
        for b in range(B):
            assert s[b].tobytes() == s8[b % 8].tobytes() and l[b] == l8[b % 8] and bb[b] == b8[b % 8]
            for k in o:
                assert o[k][b].tobytes() == o8[k][b % 8].tobytes(), (B, b, k)


def test_refused_calls_write_nothing():
    """capacities above the matcher's or the outlier kernel's, NULL required pointers and negative sizes are refused before
    anything is launched or written, and the next call on the same handles is right"""
    import torch
    L = lib()
    pairs = verify_cases()[:3]
    loop = [0, 1, 2]
    mt = ORBmatcher(0.6, True, max_queries=800, max_db=800, max_batch=3)
    out, _, keep = run_verify(mt, pairs, loop, gl.VERIFY_GLOBAL_MAPPER, [500] * 3)
    t1, t2, k1, k2, d_loop, d_n, o = keep
    gm, loc = gl.LoopVerifyParams(*gl.VERIFY_GLOBAL_MAPPER), gl.LoopVerifyParams(*gl.VERIFY_LOCALIZER)
    sp = C.c_void_p(stream())

    def with_(k, **kw):
        f = {n: getattr(k, n) for n, _ in k._fields_}
        f.update(kw)
        return type(k)(**f)

    def verify(B=3, h=mt.h, a=k1, b=k2, params=gm, n_mps=d_n, raw=o["raw"], mp=o["mp"]):
        p = lambda t: t.data_ptr() if t is not None else None
        return L.se2gpu_verify_loop_device(C.c_void_p(h) if h else None, B, C.byref(a) if a is not None else None,
                                           C.byref(b) if b is not None else None, d_loop.data_ptr(), p(n_mps),
                                           C.byref(params) if params is not None else None, p(raw), o["good"].data_ptr(), p(mp),
                                           o["counts"].data_ptr(), o["verified"].data_ptr(), sp)
    small = ORBmatcher(0.6, True, max_queries=100, max_db=800, max_batch=3)
    failing = [(lambda: verify(B=4), ERR_CAPACITY), (lambda: verify(a=with_(k1, cap=801)), ERR_CAPACITY),
               (lambda: verify(b=with_(k2, cap=801)), ERR_CAPACITY), (lambda: verify(h=small.h), ERR_CAPACITY),
               (lambda: verify(a=with_(k1, cap=8193)), ERR_CAPACITY), (lambda: verify(B=-1), ERR_INVALID),
               (lambda: verify(h=None), ERR_INVALID), (lambda: verify(a=None), ERR_INVALID), (lambda: verify(params=None), ERR_INVALID),
               (lambda: verify(n_mps=None), ERR_INVALID), (lambda: verify(raw=None), ERR_INVALID), (lambda: verify(mp=None), ERR_INVALID),
               (lambda: verify(a=with_(k1, has_mp=None)), ERR_INVALID), (lambda: verify(b=with_(k2, has_mp=None)), ERR_INVALID),
               (lambda: verify(a=with_(k1, cap=-1)), ERR_INVALID)]
    q, db = synthetic_db(3, 37, 300, seed=8)
    qa, da = bows(q, 300), bows(db, 300)
    d = Detect(qa, da, np.zeros(3, np.int32), np.arange(37, dtype=np.int32))
    dp = gl.LoopDetectParams(*gl.DETECT_GLOBAL_MAPPER)

    def detect(B=3, cap_q=300, ids=True, scores=True):
        return L.se2gpu_detect_loop_device(B, d.q[0].data_ptr(), d.q[1].data_ptr(), d.q[2].data_ptr(), cap_q, 37, d.db[0].data_ptr(),
                                           d.db[1].data_ptr(), d.db[2].data_ptr(), 300, d.q_id.data_ptr() if ids else None,
                                           d.db_id.data_ptr() if ids else None, C.byref(dp),
                                           d.scores.data_ptr() if scores else None, d.loop.data_ptr(), d.best.data_ptr(), sp)
    failing += [(lambda: detect(cap_q=100000), ERR_CAPACITY), (lambda: detect(B=-1), ERR_INVALID), (lambda: detect(ids=False), ERR_INVALID),
                (lambda: detect(scores=False), ERR_INVALID)]
    tensors = list(o.values()) + [d.scores, d.loop, d.best]
    for k, (call, code) in enumerate(failing):
        for t in tensors:
            t.fill_(7)
        assert counted(call) == 0, k
        assert call() == code, k
        torch.cuda.synchronize()
        assert all((host(t) == 7).all() for t in tensors), k
        assert verify() == 0 and detect() == 0
        torch.cuda.synchronize()
        check_verify({n: host(t) for n, t in o.items()}, pairs, loop, gl.VERIFY_GLOBAL_MAPPER, [500] * 3)
        assert_detect(d, qa, da, np.zeros(3, np.int32), np.arange(37, dtype=np.int32), gl.DETECT_GLOBAL_MAPPER)
    # the Localizer's verdict reads neither has_mp nor numMPsCurrent; B == 0 does nothing
    assert verify(params=loc, n_mps=None, a=with_(k1, has_mp=None), b=with_(k2, has_mp=None)) == 0
    assert counted(lambda: verify(B=0, raw=None)) == 0 and verify(B=0, raw=None) == 0
    assert counted(lambda: detect(B=0)) == 0
