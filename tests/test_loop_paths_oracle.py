"""CPU: the crafted inputs of tests/test_loop_paths_gpu.py, pinned to the loop-closure oracle (oracle/pyloop.py), to the
Python restatements of tests/loop_cases.py and, when oracle/_ref/libdbow2_l1.so was built, to DBoW2's own score: the
threshold pairs, the exact tie and exclusion layouts, the scoring chunk boundaries and the trimmed verification pairs."""
import numpy as np
import pytest

from oracle import pyloop
from tests import loop_cases as lc
from tests.test_loop_oracle import bows, check_detect

PRESETS = [pyloop.DETECT_GLOBAL_MAPPER, pyloop.DETECT_LOCALIZER, (3, 0.0)]


def same_score(pair, want):
    """the pair scores `want` bit for bit in the oracle, the restatement and (when built) DBoW2"""
    (a, b) = pair
    got = [np.float64(pyloop.score(*a, *b)), np.float64(lc.py_score(*a, *b))]
    ref = pyloop.dbow2_score(*a, *b)
    if ref is not None:
        got.append(np.float64(ref))
    assert all(g.tobytes() == np.float64(want).tobytes() for g in got), (got, want)


@pytest.mark.parametrize("t", [0.005, 0.05])
def test_threshold_pairs_score_exactly(t):
    """No one-word value near t scores exactly t against {w: 1.0} (those scores are multiples of 2^-54), so the pair
    against 1.0 gives min_score = s and nextafter(s, 0); a one-word vector against itself scores its value exactly, so
    the presets' own thresholds are met exactly by {w: t} and one ulp above by {w: nextafter(t, 1)}."""
    assert lc.against_one(t) is None
    s = lc.py_score(*lc.single(7, t), *lc.single(7, 1.0))
    same_score((lc.single(7, t), lc.single(7, 1.0)), s)
    q, k = lc.single(7, t), lc.single(7, 1.0)
    _, loop, best = check_detect([q], [k], np.zeros(1, np.int32), np.array([100], np.int32), (20, s))
    assert loop[0] == -1 and best[0] == s
    _, loop, _ = check_detect([q], [k], np.zeros(1, np.int32), np.array([100], np.int32), (20, np.nextafter(s, 0)))
    assert loop[0] == 0
    at, above = lc.threshold_pair(t)
    same_score(at, t)
    same_score(above, np.nextafter(t, 1.0))
    for params in (pyloop.DETECT_GLOBAL_MAPPER, pyloop.DETECT_LOCALIZER):
        if params[1] != t:
            continue
        _, loop, best = check_detect([at[0], above[0]], [at[1], above[1]], np.zeros(2, np.int32), np.array([100, 200], np.int32), params)
        assert loop.tolist() == [-1, 1] and best.tolist() == [t, np.nextafter(t, 1.0)]


def test_dyadic_pairs_score_exactly():
    """values 0.25, 0.2421875 and 0.125 against 1.0 score themselves exactly; 0.25 against 0.5 scores 0.25"""
    for v in (0.25, 0.2421875, 0.125):
        same_score((lc.single(3, 1.0), lc.single(3, v)), v)
    same_score((lc.single(3, 0.5), lc.single(3, 0.25)), 0.25)


@pytest.mark.parametrize("params", PRESETS)
def test_tie_and_exclusion_layouts(params):
    """the oracle's selection equals lc.select and each layout's named slot; the shared best is 0.25 bit for bit"""
    for layouts in (lc.tie_layouts(), lc.exclusion_layouts()):
        q, db, q_id, db_id = lc.selection_case(layouts)
        scores, loop, best = pyloop.detect(*bows(q, 1), *bows(db, len(layouts)), q_id, db_id, params)
        for b, lay in enumerate(layouts):
            assert (scores[b, lay[0]] == 0.25).all() and (scores[b, lay[2]] == 0.2421875).all()
            assert (loop[b], best[b]) == lc.select(scores[b], q_id[b], db_id, *params), b
            assert loop[b] == lc.expected_slot(lay, db_id, params[0]), (b, loop[b])
    # the ties are won by the lowest slot; the excluded lowest slot hands the loop to the next one
    _, loop, _ = pyloop.detect(*bows(q, 1), *bows(db, 4), q_id, db_id, params)
    gm = params == pyloop.DETECT_GLOBAL_MAPPER
    assert loop.tolist() == ([900, 600, 900, 600] if gm else [600] * 4)


def test_layout_scores_equal_the_restatement():
    """every score of the tie layouts' database equals lc.py_score, bit for bit (spot check of 60 slots per query)"""
    q, db, _, _ = lc.selection_case(lc.tie_layouts())
    rng = np.random.default_rng(1)
    for b, qv in enumerate(q):
        for n in rng.choice(len(db), 60, replace=False):
            same_score((qv, db[n]), lc.py_score(*qv, *db[n]))


def test_chunk_case_scores():
    """each one-word query scores its keyframe above 0 and every other chunk keyframe -0.0; the queries below and above
    every word score -0.0 against the chunk keyframes"""
    q, db, hits = lc.chunk_case()
    cap = max(len(w) for w, _ in q + db)
    scores, _, _ = pyloop.detect(*bows(q, cap), *bows(db, cap), None, None, pyloop.DETECT_LOCALIZER)
    for b, (w, v) in enumerate(q):
        for n, (dw, dv) in enumerate(db):
            assert scores[b, n].tobytes() == np.float64(lc.py_score(w, v, dw, dv)).tobytes()
    for b, n in hits:
        assert scores[b, n] > 0
        others = [m for m in range(5) if m != n]
        assert np.signbit(scores[b, others]).all() and (scores[b, others] == 0).all()
    assert scores[-4, 5] > 0 and scores[-3, 5] > 0
    assert np.signbit(scores[-2:, :5]).all() and (scores[-2:, :] == 0).all()


@pytest.mark.parametrize("k", [9, 10, 14, 15])
def test_trimmed_pairs_give_k_raw_matches(k):
    """the gate pairs: exactly k raw matches; 9 clear every match, 10 to 15 keep what RemoveMatchOutlierRansac keeps"""
    a, b = lc.trimmed_pair(k)
    raw, good, mp, counts, _ = pyloop.verify(a, b, pyloop.VERIFY_GLOBAL_MAPPER, 100)
    assert counts[0] == k == (raw >= 0).sum() == len(a["angle"])
    want = pyloop.remove_match_outlier_ransac(np.stack([a["x"], a["y"]], 1), np.stack([b["x"], b["y"]], 1), raw)
    assert good.tolist() == want.tolist()
    assert (counts[1] == 0) == (k < 10)


@pytest.mark.parametrize("G", [44, 45])
def test_good_pairs_sit_on_the_localizer_threshold(G):
    a, b = lc.good_pair(G)
    _, _, _, counts, ok = pyloop.verify(a, b, pyloop.VERIFY_LOCALIZER, 0)
    assert counts[1] == G and ok == (G >= 45)


def test_subset_keeps_the_feature_vector():
    """subset renumbers the kept features and drops the nodes it empties; the full set is the keyframe itself"""
    a, _ = lc.loop_pair(6, n=400)
    full = lc.subset(a, np.arange(400))
    assert all(np.array_equal(full[k], a[k]) for k in ("node", "ptr", "feat", "angle", "x"))
    keep = np.array([3, 50, 51, 399])
    s = lc.subset(a, keep)
    node_of = {int(f): int(a["node"][k]) for k in range(len(a["node"])) for f in a["feat"][a["ptr"][k]:a["ptr"][k + 1]]}
    got = {int(f): int(s["node"][k]) for k in range(len(s["node"])) for f in s["feat"][s["ptr"][k]:s["ptr"][k + 1]]}
    assert got == {i: node_of[int(o)] for i, o in enumerate(keep)} and s["ptr"][-1] == 4
