"""CPU: the loop-closure oracle (oracle/loop_oracle.cpp, oracle/pyloop.py) against DBoW2's own L1 score (the golden file,
and oracle/_ref/libdbow2_l1.so when it was built) and against the Python restatements of tests/loop_cases.py, on the
boundaries of the selection, the RANSAC gate and both verdicts."""
import os

import numpy as np
import pytest

from oracle import pyfundam, pyloop
from tests import loop_cases as lc

GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "l1_score_golden.npz")


def golden():
    g = np.load(GOLDEN)
    off = g["offsets"]
    vec = [(g["words"][off[k]:off[k + 1]], g["values"][off[k]:off[k + 1]]) for k in range(len(off) - 1)]
    return [(vec[2 * k], vec[2 * k + 1]) for k in range(len(vec) // 2)], g["scores"]


def test_scores_equal_the_golden_bytes():
    pairs, scores = golden()
    assert len(pairs) == len(lc.golden_pairs())
    for k, ((w1, v1), (w2, v2)) in enumerate(pairs):
        got = np.float64(pyloop.score(w1, v1, w2, v2))
        assert got.tobytes() == scores[k].tobytes(), k
        assert np.float64(lc.py_score(w1, v1, w2, v2)).tobytes() == scores[k].tobytes(), k
    # disjoint and empty sides give -0.0; identical vectors 1 up to rounding; the order-sensitive pairs differ from a tree sum
    assert all(np.signbit(scores[k]) and scores[k] == 0 for k in (1, 2, 3, 4, 6))
    assert abs(scores[0] - 1.0) < 1e-12
    for (a, b), s in zip(pairs[-3:], scores[-3:]):
        assert lc.pairwise_score(*a, *b) != s


def test_scores_equal_dbow2_on_fresh_seeds():
    if pyloop.dbow2_score([1], [1.0], [1], [1.0]) is None:
        pytest.skip("oracle/_ref/libdbow2_l1.so was not built (no reference tree)")
    rng = np.random.default_rng(123)
    for k in range(40):
        n1, n2 = (int(x) for x in rng.integers(0, 900, 2))
        a, b = lc.overlapping(rng, n1, n2, int(rng.integers(0, min(n1, n2) + 1)), vocab=5000)
        want = np.float64(pyloop.dbow2_score(*a, *b))
        assert np.float64(pyloop.score(*a, *b)).tobytes() == want.tobytes(), k


def bows(vecs, cap):
    w = np.zeros((len(vecs), cap), np.int32); v = np.zeros((len(vecs), cap)); n = np.zeros(len(vecs), np.int32)
    for k, (a, b) in enumerate(vecs):
        w[k, :len(a)] = a; v[k, :len(a)] = b; n[k] = len(a)
    return w, v, n


def check_detect(queries, db, q_id, db_id, params):
    cap = max([len(a) for a, _ in queries + db] + [1])
    scores, loop, best = pyloop.detect(*bows(queries, cap), *bows(db, cap), q_id, db_id, params)
    for b, (qw, qv) in enumerate(queries):
        for n, (dw, dv) in enumerate(db):
            assert scores[b, n].tobytes() == np.float64(lc.py_score(qw, qv, dw, dv)).tobytes()
        want = lc.select(scores[b], q_id[b], db_id, *params)
        assert (loop[b], best[b]) == want, (b, loop[b], best[b], want)
    return scores, loop, best


def test_selection_boundaries():
    rng = np.random.default_rng(3)
    q = lc.random_bow(rng, 80)
    near = (q[0][:40], q[1][:40])                           # shares half of q's words
    far = (q[0][:20], q[1][:20])
    other = (np.array([10**6], np.int32), np.array([1.0]))
    # |id difference| 19 is excluded and 20 is not (GlobalMapper); the Localizer excludes none
    db = [near, far, other]
    ids = np.array([119, 80, 60], np.int32)
    _, loop, _ = check_detect([q], db, np.array([100], np.int32), ids, pyloop.DETECT_GLOBAL_MAPPER)
    assert loop[0] == 1
    _, loop, _ = check_detect([q], db, np.array([100], np.int32), np.array([120, 80, 60], np.int32), pyloop.DETECT_GLOBAL_MAPPER)
    assert loop[0] == 0
    _, loop, _ = check_detect([q], db, np.array([100], np.int32), ids, pyloop.DETECT_LOCALIZER)
    assert loop[0] == 0
    # a best score equal to min_score is rejected, and scoreBest still reported
    s_far = lc.py_score(*q, *far)
    _, loop, best = check_detect([q], [far], np.array([0]), np.array([100]), (20, s_far))
    assert loop[0] == -1 and best[0] == s_far
    _, loop, _ = check_detect([q], [far], np.array([0]), np.array([100]), (20, np.nextafter(s_far, 0)))
    assert loop[0] == 0
    # equal best scores: the first slot wins
    _, loop, _ = check_detect([q], [far, near, near, far], np.zeros(1, np.int32), np.arange(4, dtype=np.int32) + 50, (20, 0.005))
    assert loop[0] == 1
    # every score <= 0 (disjoint: -0.0, empty): no loop and scoreBest 0.0
    e = (np.zeros(0, np.int32), np.zeros(0))
    _, loop, best = check_detect([q, e], [other, e], np.zeros(2, np.int32), np.array([40, 50], np.int32), (20, 0.005))
    assert (loop == -1).all() and best.tobytes() == np.zeros(2).tobytes()


def test_ransac_gate_and_lmeds_boundaries():
    """9 raw matches clear everything without an estimate; 10 to 14 run LMedS, 15 RANSAC (the hypothesis counts differ);
    the good matches are the mask's"""
    a, b = lc.loop_pair(seed=6, n=400)
    xy1 = np.stack([a["x"], a["y"]], 1); xy2 = np.stack([b["x"], b["y"]], 1)
    full = np.full(400, -1, np.int32)
    rng_mb = np.random.default_rng(6)
    rng_mb.integers(0, 256, (400, 32), dtype=np.uint8); rng_mb.uniform(0, 360, 400); rng_mb.integers(0, 120, 400)
    perm = rng_mb.permutation(400)
    full[perm] = np.arange(400)                               # KF1 feature perm[j] is KF2 feature j
    for k in (9, 10, 12, 14, 15):
        m = np.full(400, -1, np.int32)
        idx = np.sort(np.random.default_rng(k).choice(400, k, replace=False))
        m[idx] = full[idx]
        good = pyloop.remove_match_outlier_ransac(xy1, xy2, m)
        if k < 10:
            assert (good == -1).all()
            continue
        mask, _, iters = pyfundam.find_fundamental_mat(xy1[idx], xy2[m[idx]])
        want = np.full(400, -1, np.int32)
        if mask is not None:
            want[idx[mask.astype(bool)]] = m[idx[mask.astype(bool)]]
        assert good.tolist() == want.tolist(), k


def tail(n_good, n_mp, n_mps_cur, params, n=400):
    """verify_tail on n_good good matches of which the first n_mp have observations on both sides"""
    raw = np.full(n, -1, np.int32); good = raw.copy()
    raw[:n_good + 5] = np.arange(n_good + 5); good[:n_good] = np.arange(n_good)
    o1 = np.zeros(n, np.uint8); o2 = np.zeros(n, np.uint8)
    o1[:n_mp] = 1; o2[:n_mp] = 1
    o1[n_mp:n_good:2] = 1; o2[n_mp + 1:n_good:2] = 1            # one side only: erased
    import ctypes as C
    mp = np.zeros(n, np.int32); counts = np.zeros(3, np.int32)
    p = lambda x: x.ctypes.data_as(C.c_void_p)
    ok = pyloop.lib().loop_oracle_verify_tail(n, p(raw), p(good), p(o1), n, p(o2), int(params[0]), int(params[1]), int(params[2]),
                                              float(params[3]), int(n_mps_cur), p(mp), p(counts))
    assert counts.tolist() == [n_good + 5, n_good, 0 if params[0] else n_mp]
    assert mp.tolist() == ([-1] * n if params[0] else list(range(n_mp)) + [-1] * (n - n_mp))
    assert bool(ok) == lc.verdict(n_good, n_mp if not params[0] else 0, n_mps_cur, params)
    return bool(ok)


def test_verdict_boundaries():
    gm, loc = pyloop.VERIFY_GLOBAL_MAPPER, pyloop.VERIFY_LOCALIZER
    assert not tail(29, 20, 100, gm) and tail(30, 20, 100, gm)
    assert not tail(40, 14, 100, gm) and tail(40, 15, 100, gm)
    assert tail(40, 15, 300, gm) and not tail(40, 15, 301, gm)          # 15 / 300 == 0.05 exactly
    assert tail(40, 15, 0, gm)                                          # x / 0 = +inf passes
    assert not tail(40, 0, 0, (0, 0, 0, 0.0)) and tail(40, 0, 1, (0, 0, 0, 0.0))   # 0 / 0 = NaN fails
    assert not tail(44, 10, 100, loc) and tail(45, 10, 100, loc)


@pytest.mark.parametrize("seed,collinear", [(3, False), (4, False), (5, True)])
def test_verify_chain(seed, collinear):
    """the composed chain on a two-view pair: raw matches, a RANSAC that keeps most of them (or, collinear, finds no model)"""
    a, b = lc.loop_pair(seed, collinear=collinear)
    raw, good, mp, counts, ok = pyloop.verify(a, b, pyloop.VERIFY_GLOBAL_MAPPER, 500)
    assert counts[0] == (raw >= 0).sum() > 100
    assert counts[1] == (good >= 0).sum() and counts[2] == (mp >= 0).sum()
    assert ((good == raw) | (good == -1)).all() and ((mp == good) | (mp == -1)).all()
    assert (mp[mp >= 0] >= 0).all() and a["obs"][mp >= 0].all() and b["obs"][mp[mp >= 0]].all()
    assert ok == (not collinear) and (counts[1] == 0) == collinear


def test_detect_entry_refuses_bad_arguments_and_reports_no_device():
    """The handle-less entry checks its arguments before it looks for a device, and without one it fails loudly."""
    import ctypes as C
    import torch
    from se2lam_b200 import _capi
    L = _capi.lib()
    gm = _capi.LoopDetectParams(20, 0.005)
    buf = (C.c_double * 8)()
    call = lambda B, N, cap_q, params=C.byref(gm), q_n=buf, loop=buf: L.se2gpu_detect_loop_device(
        B, buf, buf, q_n, cap_q, N, buf, buf, buf, 4, buf, buf, params, buf, loop, buf, None)
    assert call(1, 1, 4, params=None) == -3
    assert call(-1, 1, 4) == -3 and call(1, -1, 4) == -3 and call(1, 1, -4) == -3
    assert call(1, 1, 4, q_n=None) == -3 and call(1, 1, 4, loop=None) == -3
    assert L.se2gpu_detect_loop_device(1, buf, buf, buf, 4, 1, buf, buf, buf, 4, None, None, C.byref(gm), buf, buf, buf, None) == -3
    if not torch.cuda.is_available():
        assert call(1, 1, 4) == -1 and "device" in _capi.last_error()
