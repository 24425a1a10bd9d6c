"""GPU: loop closure at the edges of its decisions and at the capacities include/se2gpu.h states, against the CPU oracle
(oracle/pyloop.py, oracle/pybow.py) byte for byte and against the slot or verdict each case is built to give.

Detect: equal best scores split across the argmax's threads and warps, the id exclusion at |id difference| 19 and 20,
scores exactly on the presets' thresholds, no positive score, the 32-word chunks of the score kernel's walk, the extreme
word ids, N = 0, N = 1 048 560 and one more, clamped counts. Verify: 9, 10, 14 and 15 raw matches around the RANSAC gate,
the verdict's comparisons at equality, cur->cap = 8192, map->cap = 16 384 (SearchByBoW without a claim table) and
FeatureVectors holding node -1. compute_bow_device at the assembly's shared-memory limit and one feature above it.
The inputs are the ones tests/test_loop_paths_oracle.py pins on the CPU."""
import ctypes as C
import re

import numpy as np
import pytest

from oracle import pybow, pyloop
from se2lam_b200 import loop as gl
from se2lam_b200._capi import last_error, lib
from se2lam_b200.matcher import ORBmatcher
from tests import loop_cases as lc
from tests.bow_cases import make_features, make_voc
from tests.test_bow_batch_gpu import BowOut, assert_keyframe, counted, dev, dev_side, host, stream, voc_handle
from tests.test_loop_gpu import Detect, assert_detect, bows, check_verify, run_verify, verify_side

pytestmark = pytest.mark.gpu

ERR_CAPACITY = -4
PRESETS = [gl.DETECT_GLOBAL_MAPPER, gl.DETECT_LOCALIZER, (3, 0.0)]
MAX_N = 65535 * 16


def run(d, params):
    """fill every output of `d` with the sentinel, then detect: two launches"""
    for t in (d.scores, d.loop, d.best):
        t.fill_(7)
    assert counted(lambda: d.run(params)) == 2


# ---------------------------------------------------------------------------------------------- detect: selection
@pytest.mark.parametrize("params", PRESETS)
def test_detect_ties_across_threads_and_warps(params):
    """N = 1 100, one query per tie layout: the lowest slot of the shared best wins, or the next one when the id offset
    excludes it; scoreBest is 0.25 bit for bit"""
    layouts = lc.tie_layouts(1100)
    q, db, q_id, db_id = lc.selection_case(layouts)
    qa, da = bows(q, 1), bows(db, len(layouts))
    d = Detect(qa, da, q_id, db_id)
    run(d, params)
    _, loop, best = assert_detect(d, qa, da, q_id, db_id, params)
    assert loop.tolist() == [lc.expected_slot(lay, db_id, params[0]) for lay in layouts], loop
    assert (best == 0.25).all()
    assert loop[5] == (700 if params[0] > 1 else 3) and loop[7] == (1 if params[0] > 1 else 0)


@pytest.mark.parametrize("params", PRESETS)
def test_detect_id_exclusion_at_19_and_20(params):
    """the best keyframe 19 ids from the query, above or below, is excluded by GlobalMapper's offset of 20; 20 ids away it
    is not"""
    layouts = lc.exclusion_layouts()
    q, db, q_id, db_id = lc.selection_case(layouts)
    qa, da = bows(q, 1), bows(db, len(layouts))
    d = Detect(qa, da, q_id, db_id)
    run(d, params)
    _, loop, best = assert_detect(d, qa, da, q_id, db_id, params)
    gm = params == gl.DETECT_GLOBAL_MAPPER
    assert loop.tolist() == ([900, 600, 900, 600] if gm else [600] * 4)
    assert best.tolist() == ([0.2421875, 0.25] * 2 if gm else [0.25] * 4)


def reword(pair, w):
    return tuple((np.array([w], np.int32), v) for _, v in pair)


def test_detect_thresholds_on_exact_scores():
    """{w: t} against itself scores t exactly: at each preset's threshold no loop is detected and scoreBest holds t; one
    ulp above, the loop is the keyframe. {w: 0.005} against {w: 1.0} scores s, which no value near 0.005 makes exactly
    0.005: min_score = s rejects it and nextafter(s, 0) accepts it."""
    at5, up5 = lc.threshold_pair(0.005)
    at50, up50 = lc.threshold_pair(0.05)
    pairs = [reword(p, 10 + k) for k, p in enumerate([at5, up5, at50, up50, (lc.single(7, 0.005), lc.single(7, 1.0))])]
    s = lc.py_score(*pairs[4][0], *pairs[4][1])
    qa, da = bows([p[0] for p in pairs], 1), bows([p[1] for p in pairs], 1)
    q_id, db_id = np.full(5, lc.FAR, np.int32), np.arange(5, dtype=np.int32)
    d = Detect(qa, da, q_id, db_id)
    want_best = np.array([0.005, np.nextafter(0.005, 1), 0.05, np.nextafter(0.05, 1), s])
    for params, want in [(gl.DETECT_GLOBAL_MAPPER, [-1, 1, 2, 3, 4]), (gl.DETECT_LOCALIZER, [-1, -1, -1, 3, -1]),
                         ((20, s), [-1, -1, 2, 3, -1]), ((20, np.nextafter(s, 0)), [-1, -1, 2, 3, 4])]:
        run(d, params)
        _, loop, best = assert_detect(d, qa, da, q_id, db_id, params)
        assert loop.tolist() == want, (params, loop)
        assert best.tobytes() == want_best.tobytes()


def test_detect_no_positive_score():
    """disjoint and empty vectors score -0.0 and a common word of value 0 scores -0.0 too: no loop, scoreBest +0.0"""
    e = (np.zeros(0, np.int32), np.zeros(0))
    q = [lc.single(300, 1.0), e, lc.single(100, 0.0), lc.random_bow(np.random.default_rng(2), 40, vocab=1000)]
    q[3] = (q[3][0] + 3000, q[3][1])
    db = [lc.single(100, 1.0), e, lc.single(200, 0.5), (np.arange(2000, 2040, dtype=np.int32), np.full(40, 0.025))]
    qa, da = bows(q, 40), bows(db, 40)
    q_id, db_id = np.zeros(4, np.int32), np.arange(4, dtype=np.int32) * 100 + 100
    d = Detect(qa, da, q_id, db_id)
    for params in PRESETS:
        run(d, params)
        scores, loop, best = assert_detect(d, qa, da, q_id, db_id, params)
        assert (scores == 0).all() and np.signbit(scores).all()
        assert (loop == -1).all() and best.tobytes() == np.zeros(4).tobytes()


# ---------------------------------------------------------------------------------------------- detect: scoring
def test_detect_scoring_chunks_and_word_extremes():
    """keyframes of 31, 32, 33, 64 and 65 words whose one common word with the query is at lane 31 of a chunk, lane 0 of
    the next, the first or the last; words 0 and 2^31 - 1; queries below and above every word"""
    q, db, hits = lc.chunk_case()
    qa, da = bows(q, max(len(w) for w, _ in q)), bows(db, 65)
    d = Detect(qa, da)
    run(d, gl.DETECT_LOCALIZER)
    scores, _, _ = assert_detect(d, qa, da, None, None, gl.DETECT_LOCALIZER)
    for b, n in hits:
        assert scores[b, n] == lc.py_score(*q[b], *db[n]) > 0, (b, n)
    assert scores[-4, 5] > 0 and scores[-3, 5] > 0
    assert (scores[-2:] == 0).all() and np.signbit(scores[-2:]).all()


# ---------------------------------------------------------------------------------------------- detect: sizes and counts
def test_detect_without_database_keyframes():
    """N = 0: two launches, no loop and scoreBest 0.0, with NULL scores and database pointers"""
    import torch
    rng = np.random.default_rng(4)
    qa = bows([lc.random_bow(rng, 50), lc.random_bow(rng, 3), (np.zeros(0, np.int32), np.zeros(0))], 50)
    q = [dev(a) for a in qa]
    hq_id = np.array([5, 6, 7], np.int32)
    q_id = dev(hq_id)
    loop = torch.full((3,), 7, dtype=torch.int32, device="cuda:0")
    best = torch.full((3,), 7.0, dtype=torch.float64, device="cuda:0")
    empty = (np.zeros((0, 4), np.int32), np.zeros((0, 4)), np.zeros(0, np.int32))
    for params in PRESETS:
        loop.fill_(7); best.fill_(7)
        assert counted(lambda: gl.detect_loop_device(3, *q, 50, 0, None, None, None, 4, None, loop, best, d_q_id=q_id, params=params,
                                                     stream=stream())) == 2
        torch.cuda.synchronize()
        _, l_o, b_o = pyloop.detect(*qa, *empty, hq_id, None, params)
        assert host(loop).tolist() == l_o.tolist() == [-1] * 3
        assert host(best).tobytes() == b_o.tobytes() == np.zeros(3).tobytes()


def test_detect_at_the_keyframe_limit():
    """N = 1 048 560 = 65 535 x 16 one-word keyframes, B = 2: query 0's unique best is the last slot, query 1's best is
    shared by slot N - 17 (the previous score CTA row) and the last; every score equals the oracle's. N + 1 is
    SE2GPU_ERR_CAPACITY and writes nothing, though every buffer holds N + 1 keyframes."""
    import torch
    N = MAX_N
    rng = np.random.default_rng(12)
    dw = rng.integers(0, 128, (N + 1, 1)).astype(np.int32)
    dv = rng.uniform(0.01, 0.2, (N + 1, 1))
    dw[N - 1], dv[N - 1] = 200, 0.25
    dw[N - 17], dv[N - 17] = 201, 0.25
    dn = np.ones(N + 1, np.int32)
    qw = np.stack([np.concatenate([np.arange(64), [200, 300]]), np.arange(64, 130)]).astype(np.int32)
    qw[1, -2:] = [200, 201]
    qa = (qw, np.ones(qw.shape), np.full(2, qw.shape[1], np.int32))
    q_id, db_id = np.full(2, -1000, np.int32), np.arange(N + 1, dtype=np.int32)
    d = Detect(qa, (dw, dv, dn), q_id, db_id)
    d.N = N
    for params in (gl.DETECT_GLOBAL_MAPPER, gl.DETECT_LOCALIZER):
        run(d, params)
        _, loop, best = assert_detect(d, qa, (dw[:N], dv[:N], dn[:N]), q_id, db_id[:N], params)
        assert loop.tolist() == [N - 1, N - 17] and (best == 0.25).all()
    for t in (d.scores, d.loop, d.best):
        t.fill_(7)
    p = gl.LoopDetectParams(*gl.DETECT_GLOBAL_MAPPER)
    call = lambda: lib().se2gpu_detect_loop_device(
        2, d.q[0].data_ptr(), d.q[1].data_ptr(), d.q[2].data_ptr(), qw.shape[1], N + 1, d.db[0].data_ptr(), d.db[1].data_ptr(),
        d.db[2].data_ptr(), 1, d.q_id.data_ptr(), d.db_id.data_ptr(), C.byref(p), d.scores.data_ptr(), d.loop.data_ptr(),
        d.best.data_ptr(), C.c_void_p(stream()))
    assert counted(call) == 0 and call() == ERR_CAPACITY
    assert "1048560" in last_error()
    torch.cuda.synchronize()
    assert d.scores.numel() == 2 * (N + 1) and all((host(t) == 7).all() for t in (d.scores, d.loop, d.best))


def test_detect_clamps_counts():
    """counts above cap read cap words and counts below 0 read none, as the oracle does on the clamped counts"""
    rng = np.random.default_rng(6)
    cap = 40
    qa = bows([lc.random_bow(rng, cap, vocab=300) for _ in range(4)], cap)
    da = bows([lc.random_bow(rng, cap, vocab=300) for _ in range(6)], cap)
    qa[2][:] = [cap + 1, 2 ** 31 - 1, -1, -2 ** 31]
    da[2][:] = [cap + 5, 0, -7, 2 ** 31 - 1, cap, 17]
    q_id, db_id = np.full(4, lc.FAR, np.int32), np.arange(6, dtype=np.int32)
    d = Detect(qa, da, q_id, db_id)
    clamp = lambda a: (a[0], a[1], np.clip(a[2], 0, cap).astype(np.int32))
    for params in PRESETS:
        run(d, params)
        scores, loop, best = assert_detect(d, clamp(qa), clamp(da), q_id, db_id, params)
        assert (scores[:2, [0, 3, 4]] > 0).all() and np.signbit(scores[2:]).all() and np.signbit(scores[:, [1, 2]]).all()
        assert loop[2:].tolist() == [-1, -1] and loop[0] >= 0


# ---------------------------------------------------------------------------------------------- verify
GM, LOC = gl.VERIFY_GLOBAL_MAPPER, gl.VERIFY_LOCALIZER


def test_verify_ransac_gate():
    """pairs of exactly 9, 10, 14 and 15 raw matches: 9 clear every match without an estimate (counts [9, 0, 0]); 10 to
    14 keep LMedS's mask and 15 RANSAC's, as RemoveMatchOutlierRansac does"""
    pairs = [lc.trimmed_pair(k) for k in (9, 10, 14, 15)]
    loop = [0, 1, 2, 3]
    mt = ORBmatcher(0.6, True, max_queries=400, max_db=400, max_batch=4)
    for params in (GM, LOC):
        out, launches, _ = run_verify(mt, pairs, loop, params, [100] * 4)
        assert launches == 6
        check_verify(out, pairs, loop, params, [100] * 4)
        assert out["counts"][:, 0].tolist() == [9, 10, 14, 15]
        assert out["counts"][0].tolist() == [9, 0, 0] and (out["good"][0] == -1).all() and (out["mp"][0] == -1).all()
        for b in (1, 2, 3):
            a, m = pairs[b]
            good = pyloop.remove_match_outlier_ransac(np.stack([a["x"], a["y"]], 1), np.stack([m["x"], m["y"]], 1), out["raw"][b])
            assert out["good"][b].tolist() == good.tolist() and out["counts"][b, 1] > 0, b


def test_verify_verdict_at_equality():
    """copies of one pair whose hasObservation flags make nMP 14, 15 or 0, with numMPsCurrent 100, 300 (15 / 300 is
    0.05 exactly), 301 and 0, under the presets, min_match_kp = G and G + 1, and ratio 0 (0 / 0 fails)"""
    a, m = lc.loop_pair(4)
    mt = ORBmatcher(0.6, True, max_queries=800, max_db=800, max_batch=8)
    m = dict(m, obs=np.ones(len(m["angle"]), np.uint8))
    first, _, _ = run_verify(mt, [(a, m)], [0], GM, [100])
    check_verify(first, [(a, m)], [0], GM, [100])
    G = int(first["counts"][0, 1])
    gi = np.flatnonzero(first["good"][0] >= 0)
    assert G == len(gi) >= 45

    def cur(n_mp):
        obs = np.zeros(len(a["angle"]), np.uint8)
        obs[gi[:n_mp]] = 1
        return dict(a, obs=obs)
    copies = [(14, 100), (15, 100), (15, 300), (15, 301), (15, 0), (0, 0), (0, 1)]
    pairs = [(cur(k), m) for k, _ in copies]
    n_mps = [n for _, n in copies]
    loop = [0] * len(copies)
    for params, want in [(GM, [0, 1, 1, 0, 1, 0, 0]), ((0, 0, 0, 0.0), [1, 1, 1, 1, 1, 0, 1]), ((0, 15, G, 0.05), [0, 1, 1, 0, 1, 0, 0]),
                         ((0, 15, G + 1, 0.05), [0] * 7), ((1, 0, G, 0.0), [1] * 7), ((1, 0, G + 1, 0.0), [0] * 7)]:
        out, _, _ = run_verify(mt, pairs, loop, params, n_mps)
        check_verify(out, pairs, loop, params, n_mps)
        assert out["verified"].tolist() == want, (params, out["counts"])
        assert out["counts"][:, 1].tolist() == [G] * 7
        assert out["counts"][:, 2].tolist() == ([14, 15, 15, 15, 15, 0, 0] if not params[0] else [0] * 7)
    # the Localizer's preset on pairs of exactly 45 and 44 good matches
    pairs = [lc.good_pair(45), lc.good_pair(44)]
    out, _, _ = run_verify(mt, pairs, [0, 1], LOC, [0, 0])
    check_verify(out, pairs, [0, 1], LOC, [0, 0])
    assert out["counts"][:, 1].tolist() == [45, 44] and out["verified"].tolist() == [1, 0]


def test_verify_at_the_outlier_kernels_capacity():
    """cur->cap = max_queries = 8192 (the outlier kernel's limit) with an 8 000-feature pair of thousands of raw matches"""
    a, m = lc.loop_pair(9, n=8000)
    mt = ORBmatcher(0.6, True, max_queries=8192, max_db=8192, max_batch=1)
    for params in (GM, LOC):
        out, launches, _ = run_verify(mt, [(a, m)], [0], params, [3000], cap1=8192, cap2=8192)
        check_verify(out, [(a, m)], [0], params, [3000])
        assert out["counts"][0, 0] > 1000 and out["counts"][0, 1] > 1000 and out["verified"][0] == 1


def test_verify_on_a_large_map():
    """map->cap = 16 384: SearchByBoW runs without its claim table (three launches), so verify takes five; one loop
    keyframe holds 14 000 more features than its query matched against"""
    pairs = [lc.loop_pair(s_) for s_ in (3, 4, 6)]
    pairs.append((pairs[0][0], lc.extended(pairs[0][1], 14000, seed=1)))
    loop = [3, 1, -1, 2]
    mt = ORBmatcher(0.6, True, max_queries=800, max_db=16384, max_batch=4)
    out, launches, _ = run_verify(mt, pairs, loop, GM, [500] * 4, cap2=16384)
    assert launches == 5
    check_verify(out, pairs, loop, GM, [500] * 4)
    assert out["verified"].tolist() == [1, 1, 0, 0] and out["counts"][0, 0] > 100


def test_verify_on_feature_vectors_with_node_minus_one():
    """a ragged vocabulary at levelsup 2, where some features sit at leaves above the node level: compute_bow_device
    writes node -1 into both sides' FeatureVectors, and verify on those device FeatureVectors equals the oracle chain"""
    import torch
    voc = make_voc(7, 5, seed=5, ragged=True)
    v = voc_handle(voc)
    n, seeds = 500, (3, 4, 6)
    pairs = []
    for s_ in seeds:
        a, m = lc.loop_pair(s_, n=n)
        d1 = make_features(voc, n, seed=700 + s_)
        rng = np.random.default_rng(s_)
        d2 = d1[lc.loop_perm(s_, n)] ^ (rng.integers(0, 256, (n, 32), dtype=np.uint8) & rng.integers(0, 256, (n, 32), dtype=np.uint8) &
                                        rng.integers(0, 256, (n, 32), dtype=np.uint8) & rng.integers(0, 256, (n, 32), dtype=np.uint8))
        a, m = dict(a, desc=d1), dict(m, desc=d2)
        for k in (a, m):
            k.update({f: pybow.compute_bow(voc, k["desc"], 2)[f] for f in ("node", "ptr", "feat")})
        pairs.append((a, m))
    B = len(pairs)
    sides = []
    for j in (0, 1):
        t, _ = dev_side(verify_side([p[j] for p in pairs], n, j + 1))
        bo = BowOut(B, n, bow=False)
        bo.run(v, t["desc"], None, 2)
        sides.append((t, bo, ORBmatcher.BowBatchSide(t["kp"], t["desc"], n, bo.node, bo.ptr, bo.feat, bo.nn, has_mp=t["has_mp"])))
    torch.cuda.synchronize()
    for j in (0, 1):
        for b in range(B):
            assert_keyframe(sides[j][1].keyframe(b), pairs[b][j], bow=False)
        assert any((pairs[b][j]["node"] == -1).any() for b in range(B)), j
    z = lambda *sh, t=torch.int32: torch.full(sh, 7, dtype=t, device="cuda:0")
    o = dict(raw=z(B, n), good=z(B, n), mp=z(B, n), counts=z(B, 3), verified=z(B, t=torch.uint8))
    loop, n_mps = [0, 1, 2], [300] * B
    mt = ORBmatcher(0.6, True, max_queries=n, max_db=n, max_batch=B)
    gl.verify_loop_device(mt, B, sides[0][2], sides[1][2], dev(np.array(loop, np.int32)), o["raw"], o["good"], o["mp"], o["counts"],
                          o["verified"], d_n_mps_cur=dev(np.array(n_mps, np.int32)), params=GM, stream=stream())
    torch.cuda.synchronize()
    out = {k: host(t) for k, t in o.items()}
    check_verify(out, pairs, loop, GM, n_mps)
    assert (out["counts"][:, 0] > 50).all(), out["counts"]


# ---------------------------------------------------------------------------------------------- compute_bow at its limit
def test_compute_bow_at_the_assembly_limit():
    """cap = the assembly's shared memory / 36 bytes (6 400 features on an H100), read from a refused call's message and
    from the device's opt-in shared memory: keyframes at full count, one with duplicate words and one (on a vocabulary
    with half its words stopped) equal the oracle byte for byte; one feature more is SE2GPU_ERR_CAPACITY and writes
    nothing into buffers that hold it"""
    import torch
    voc = make_voc(10, 4, seed=4)
    half = dict(voc, weight=voc["weight"].copy())
    half["weight"][np.flatnonzero(voc["word_id"] >= 0)[::2]] = 0.0
    v, vh = voc_handle(voc), voc_handle(half)
    cap = (torch.cuda.get_device_properties(0).shared_memory_per_block_optin - 2048) // 36
    desc = np.stack([make_features(voc, cap + 1, seed=40 + b) for b in range(3)])
    desc[1, 1::3] = desc[0, 0::3][: len(desc[1, 1::3])]
    desc[1, 0::3] = desc[0, 0::3]
    big = BowOut(3, cap + 1)
    d_big = dev(desc)
    rc = lib().se2gpu_voc_compute_bow_device(C.c_void_p(v.h), 3, d_big.data_ptr(), cap + 1, None, 2, big.word.data_ptr(),
                                             big.value.data_ptr(), big.nw.data_ptr(), big.node.data_ptr(), big.ptr.data_ptr(),
                                             big.feat.data_ptr(), big.nn.data_ptr(), C.c_void_p(stream()))
    assert rc == ERR_CAPACITY
    assert int(re.search(r"at most (\d+)", last_error()).group(1)) == cap
    torch.cuda.synchronize()
    assert all((a == 7).all() for a in big.arrays())
    d = dev(np.ascontiguousarray(desc[:, :cap]))
    for voc_, h, rows in ((voc, v, (0, 1, 2)), (half, vh, (2,))):
        out = BowOut(len(rows), cap)
        dd = d if len(rows) == 3 else dev(np.ascontiguousarray(desc[2:, :cap]))
        assert counted(lambda: out.run(h, dd, dev(np.full(len(rows), cap, np.int32)), 2)) == 2
        torch.cuda.synchronize()
        for k, b in enumerate(rows):
            want = pybow.compute_bow(voc_, desc[b, :cap], 2)
            assert_keyframe(out.keyframe(k), want)
            assert want["ptr"][-1] > (cap // 3 if voc_ is half else cap * 9 // 10), (b, want["ptr"][-1])
    assert len(pybow.compute_bow(voc, desc[1, :cap], 2)["word"]) < len(pybow.compute_bow(voc, desc[0, :cap], 2)["word"])
