"""BowVectors, keyframe pairs and Python restatements for the loop-closure tests (tests/test_loop_oracle.py,
tests/test_loop_gpu.py) and tools/loop_bench.py."""
import numpy as np

f32 = np.float32


def random_bow(rng, n, vocab=100000):
    """n distinct ascending words with L1-normalised positive values"""
    w = np.sort(rng.choice(vocab, n, replace=False)).astype(np.int32)
    v = rng.uniform(0.1, 1.0, n)
    return w, v / v.sum()


def overlapping(rng, n1, n2, common, vocab=100000):
    """two BowVectors of n1 and n2 words sharing `common` of them"""
    w = rng.choice(vocab, n1 + n2 - common, replace=False)
    a, b = np.sort(w[:n1]), np.sort(np.concatenate([w[:common], w[n1:]]))
    va, vb = rng.uniform(0.1, 1.0, n1), rng.uniform(0.1, 1.0, n2)
    return (a.astype(np.int32), va / va.sum()), (b.astype(np.int32), vb / vb.sum())


def py_score(w1, v1, w2, v2):
    """L1Scoring::score restated: the common words in ascending order, score += fabs(vi - wi) - fabs(vi) - fabs(wi)"""
    d2 = dict(zip(np.asarray(w2).tolist(), np.asarray(v2).tolist()))
    s = 0.0
    for w, vi in zip(np.asarray(w1).tolist(), np.asarray(v1).tolist()):
        if w in d2:
            wi = d2[w]
            s += abs(vi - wi) - abs(vi) - abs(wi)
    return -s / 2.0


def pairwise_score(w1, v1, w2, v2):
    """the same terms summed as a tree (what a parallel reduction would do)"""
    d2 = dict(zip(np.asarray(w2).tolist(), np.asarray(v2).tolist()))
    t = [abs(vi - d2[w]) - abs(vi) - abs(d2[w]) for w, vi in zip(np.asarray(w1).tolist(), np.asarray(v1).tolist()) if w in d2]
    while len(t) > 1:
        t = [t[i] + t[i + 1] if i + 1 < len(t) else t[i] for i in range(0, len(t), 2)]
    return -(t[0] if t else 0.0) / 2.0


def order_sensitive_pairs(seed=5, count=3):
    """pairs whose ascending fold differs from the pairwise sum of the same terms"""
    rng = np.random.default_rng(seed)
    out = []
    while len(out) < count:
        a, b = overlapping(rng, 300, 280, 150)
        if py_score(*a, *b) != pairwise_score(*a, *b):
            out.append((a, b))
    return out


def golden_pairs():
    """the BowVector pairs of tests/golden/l1_score_golden.npz"""
    rng = np.random.default_rng(11)
    e = (np.zeros(0, np.int32), np.zeros(0))
    a = random_bow(rng, 50)
    pairs = [(a, a), overlapping(rng, 40, 30, 0), (e, a), (a, e), (e, e),
             ((np.array([7], np.int32), np.array([1.0])), (np.array([7], np.int32), np.array([0.25]))),
             ((np.array([7], np.int32), np.array([1.0])), (np.array([8], np.int32), np.array([1.0])))]
    pairs += [overlapping(rng, 700, 700, c) for c in (1, 90, 400)]
    pairs += [overlapping(rng, 700, 60, 30), overlapping(rng, 60, 700, 30)]
    pairs += order_sensitive_pairs()
    return pairs


def select(scores, q_id, db_id, min_id_offset, min_score):
    """DetectLoopClose's selection restated for one query: (loop slot or -1, scoreBest)"""
    best, kf = 0.0, -1
    for n, s in enumerate(scores):
        if abs(int(db_id[n]) - int(q_id)) < min_id_offset:
            continue
        if s > best:
            best, kf = s, n
    return (kf if kf >= 0 and best > min_score else -1), best


def verdict(n_good, n_mp, n_mps_cur, params):
    """VerifyLoopClose's acceptance restated"""
    localizer, min_mp, min_kp, ratio = params
    if localizer:
        return n_good >= min_kp
    r = n_mp * 1.0 / n_mps_cur if n_mps_cur else (float("nan") if n_mp == 0 else float("inf"))
    return n_mp >= min_mp and n_good >= min_kp and r >= ratio


def loop_pair(seed=3, n=800, outliers=0.3, collinear=False):
    """A keyframe pair of tests/matcher_cases.make_bow_case with keyPointsUn from two views of one 3D scene (KF2 feature j is
    KF1 feature perm[j] seen again; a fraction of KF2's points moved at random), and hasObservation flags.
    collinear=True puts every KF1 point on one image row, so RANSAC finds no model."""
    from tests.matcher_cases import make_bow_case
    k1, k2 = make_bow_case(seed=seed, n=n)
    rng = np.random.default_rng((seed, 77))
    rng_mb = np.random.default_rng(seed)                 # make_bow_case's permutation: its draws before it, then it
    rng_mb.integers(0, 256, (n, 32), dtype=np.uint8); rng_mb.uniform(0, 360, n); rng_mb.integers(0, 120, n)
    perm = rng_mb.permutation(n)
    P = np.stack([rng.uniform(-3, 3, n), rng.uniform(-2, 2, n), rng.uniform(3, 9, n)], 1)
    ang = 0.05
    R = np.array([[np.cos(ang), 0, np.sin(ang)], [0, 1, 0], [-np.sin(ang), 0, np.cos(ang)]])
    t = np.array([0.4, 0.05, 0.1])
    proj = lambda X: np.stack([400 * X[:, 0] / X[:, 2] + 320, 400 * X[:, 1] / X[:, 2] + 240], 1)
    xy1 = proj(P)
    xy2 = proj(P @ R.T + t)[perm] + rng.normal(0, 0.3, (n, 2))
    bad = rng.random(n) < outliers
    xy2[bad] = rng.uniform(0, 640, (bad.sum(), 2))
    if collinear:
        xy1[:, 1] = 240.0
    for k, xy in ((k1, xy1), (k2, xy2)):
        k["x"], k["y"] = xy[:, 0].astype(f32), xy[:, 1].astype(f32)
        k["obs"] = (rng.random(n) < 0.7).astype(np.uint8)
    return k1, k2
