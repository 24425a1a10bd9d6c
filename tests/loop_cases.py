"""BowVectors, keyframe pairs and Python restatements for the loop-closure tests (tests/test_loop_oracle.py,
tests/test_loop_gpu.py, tests/test_loop_paths_oracle.py, tests/test_loop_paths_gpu.py) and tools/loop_bench.py."""
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


def single(word, value):
    """the one-word BowVector {word: value}"""
    return np.array([word], np.int32), np.array([value], np.float64)


def threshold_pair(t):
    """(at, above): {7: v} against itself for v = t and the next double above t. L1Scoring scores such a pair v exactly:
    |v - v| - |v| - |v| = -2v and -(-2v) / 2 = v, every step exact in double."""
    up = np.nextafter(t, 1.0)
    return (single(7, t), single(7, t)), (single(7, up), single(7, up))


def against_one(t, steps=4096):
    """a value v within `steps` doubles of t whose {7: v} scores exactly t against {7: 1.0}, or None. There is none at
    0.005 or 0.05: that score is ((1 - v) - v - 1) / -2, a multiple of 2^-54, and neither threshold is one."""
    for d in (1.0, 0.0):
        v = t
        for _ in range(steps):
            if py_score(*single(7, v), *single(7, 1.0)) == t:
                return v
            v = np.nextafter(v, d)
    return None


# selection layouts: query b is {b: 1.0}; database keyframe n holds word b with 0.25 at layout b's `best` slots (a score
# of 0.25 exactly), 0.2421875 at its `second` slots (exact too) and a value in [0.01, 0.2) elsewhere. Keyframe n's id is
# 40 n, so a query id of 10^6 excludes none.
FAR = 10 ** 6


def tie_layouts(N=1100):
    """(best slots, q_id, second slots) with the best score shared across the argmax's threads and warps"""
    return [([5, 261], FAR, []),                     # one thread's first and second stride
            ([31, 32], FAR, []),                     # the last lane of warp 0 and the first of warp 1
            ([255, 256, 511], FAR, []),              # the last thread, then thread 0's second and third strides
            ([1040, 40], FAR, []),                   # the lower slot in a higher thread
            ([0, N - 1], FAR, []),                   # the first slot and the last, in the score kernel's partial row
            ([3, 700], 3 * 40 + 1, []),              # the lowest slot 1 id from the query: excluded by any offset > 1
            ([100, 612, 1099], FAR, []),
            (list(range(N)), 1, [])]                 # every slot: slot 0 (id 0) is excluded by any offset > 1


def exclusion_layouts():
    """slot 600 (id 24 000) holds the best score, slot 900 the second; the query id is 19 or 20 above or below 24 000"""
    return [([600], 24000 + d, [900]) for d in (19, 20, -19, -20)]


def selection_case(layouts, N=1100, seed=0):
    """(queries, database, q_id, db_id) of the layouts"""
    rng = np.random.default_rng(seed)
    B = len(layouts)
    val = rng.uniform(0.01, 0.2, (N, B))
    for b, (best, _, second) in enumerate(layouts):
        val[second, b] = 0.2421875
        val[best, b] = 0.25
    q = [single(b, 1.0) for b in range(B)]
    db = [(np.arange(B, dtype=np.int32), val[n].copy()) for n in range(N)]
    return q, db, np.array([l[1] for l in layouts], np.int32), np.arange(N, dtype=np.int32) * 40


def expected_slot(layout, db_id, min_id_offset):
    """the slot a layout's query selects: the lowest best slot the offset keeps, else the lowest kept second slot"""
    best, q_id, second = layout
    kept = lambda s: [n for n in s if min_id_offset <= 0 or abs(int(db_id[n]) - q_id) >= min_id_offset]
    return min(kept(best) or kept(second))


def chunk_case():
    """Database keyframes of 31, 32, 33, 64 and 65 words (keyframe n: 1000 (n + 1) + 2 i), one holding words 0 and
    2^31 - 1, and queries that share one word with one keyframe: at position 0, 31 (the last lane of a 32-word chunk),
    32 (the first lane of the next), 63, 64 or the last, among odd words of that keyframe's range. Then queries holding
    0 and 2^31 - 1, 2^31 - 1 alone, and queries whose words all lie below or all above every keyframe word but those two.
    Returns (queries, database, [(query, keyframe)] of the one-word queries)."""
    rng = np.random.default_rng(31)
    top = 2 ** 31 - 1
    lengths = [31, 32, 33, 64, 65]
    db = [((1000 * (n + 1) + 2 * np.arange(L)).astype(np.int32), rng.uniform(0.01, 1, L)) for n, L in enumerate(lengths)]
    db.append((np.array([0, 5, top - 1, top], np.int32), rng.uniform(0.01, 1, 4)))
    q, hits = [], []
    for n, L in enumerate(lengths):
        for p in sorted({0, 31, 32, 63, 64, L - 1} & set(range(L))):
            w = np.sort(np.concatenate([db[n][0][p:p + 1], db[n][0] + 1])).astype(np.int32)
            hits.append((len(q), n))
            q.append((w, rng.uniform(0.01, 1, len(w))))
    q.append((np.array([0, 7, top], np.int32), rng.uniform(0.01, 1, 3)))
    q.append((np.array([top], np.int32), rng.uniform(0.01, 1, 1)))
    q.append((np.arange(10, 60, 3, dtype=np.int32), rng.uniform(0.01, 1, 17)))          # below
    q.append((np.arange(top - 60, top - 10, 3, dtype=np.int32), rng.uniform(0.01, 1, 17)))  # above
    return q, db, hits


def loop_perm(seed, n):
    """loop_pair's correspondence: KF2 feature j is KF1 feature perm[j]"""
    rng_mb = np.random.default_rng(seed)
    rng_mb.integers(0, 256, (n, 32), dtype=np.uint8); rng_mb.uniform(0, 360, n); rng_mb.integers(0, 120, n)
    return rng_mb.permutation(n)


def subset(kf, keep):
    """keyframe dict restricted to the features `keep` (ascending), renumbered 0.., its FeatureVector rebuilt"""
    keep = np.asarray(keep)
    new = np.full(len(kf["angle"]), -1, np.int64); new[keep] = np.arange(len(keep))
    out = {k: np.asarray(v)[keep] for k, v in kf.items() if k not in ("node", "ptr", "feat")}
    node, ptr, feat = [], [0], []
    for k, nd in enumerate(kf["node"]):
        f = new[kf["feat"][kf["ptr"][k]:kf["ptr"][k + 1]]]
        f = f[f >= 0]
        if len(f):
            node.append(nd); feat.extend(f.tolist()); ptr.append(len(feat))
    return dict(out, node=np.asarray(node, np.int32), ptr=np.asarray(ptr, np.int32), feat=np.asarray(feat, np.int32))


def extended(kf, extra, seed=0):
    """keyframe dict with `extra` more features: random descriptors, angles, positions and flags in its own nodes"""
    rng = np.random.default_rng(seed)
    n = len(kf["angle"])
    node_of = np.empty(n + extra, np.int32)
    for k, nd in enumerate(kf["node"]):
        node_of[kf["feat"][kf["ptr"][k]:kf["ptr"][k + 1]]] = nd
    node_of[n:] = rng.choice(kf["node"], extra)
    more = dict(angle=rng.uniform(0, 360, extra).astype(f32), desc=rng.integers(0, 256, (extra, 32), dtype=np.uint8),
                x=rng.uniform(0, 640, extra).astype(f32), y=rng.uniform(0, 480, extra).astype(f32),
                obs=(rng.random(extra) < 0.7).astype(np.uint8), has_mp=(rng.random(extra) < 0.7).astype(np.uint8))
    out = {k: np.concatenate([kf[k], more[k]]) for k in more}
    nodes = np.unique(node_of)
    feat = [np.flatnonzero(node_of == nd) for nd in nodes]
    return dict(out, node=nodes.astype(np.int32), ptr=np.cumsum([0] + [len(f) for f in feat]).astype(np.int32),
                feat=np.concatenate(feat).astype(np.int32))


def trimmed_pair(k, seed=6, n=400, want_good=None, tries=200):
    """a loop_pair whose KF1 is trimmed to k features that match, so that SearchByBoW gives exactly k raw matches (and,
    with want_good, RemoveMatchOutlierRansac keeps exactly want_good of them); the first subset of seeded draws that does,
    or None"""
    from oracle import pyloop
    a, b = loop_pair(seed, n=n)
    raw, _, _, _, _ = pyloop.verify(a, b, (1, 0, 0, 0.0), 0)
    matched = np.flatnonzero(raw >= 0)
    for t in range(tries):
        keep = np.sort(np.random.default_rng((seed, k, t)).choice(matched, k, replace=False))
        c = subset(a, keep)
        counts = pyloop.verify(c, b, (1, 0, 0, 0.0), 0)[3]
        if counts[0] == k and (want_good is None or counts[1] == want_good):
            return c, b
    return None


def good_pair(G, seed=6, n=400):
    """a trimmed loop_pair whose verification keeps exactly G good matches"""
    for k in range(G, 2 * G):
        p = trimmed_pair(k, seed, n, want_good=G, tries=8)
        if p is not None:
            return p
    raise AssertionError(f"no trimmed pair with {G} good matches")


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
