"""CPU: the BowVector / FeatureVector assembly oracle (oracle/bow_assembly_oracle.cpp) against an independent pure-Python
restatement of DBoW2's transform(features, v, fv, levelsup) bookkeeping (TemplatedVocabulary.h:1170-1190, BowVector.cpp:62-84),
value bytes and feature lists exactly."""
import numpy as np
import pytest

from oracle import pybow, pyoracle
from tests.bow_cases import make_features, make_voc


def dict_assembly(word, weight, node):
    """v[word] += w in feature order for the features with w > 0, fv[node].append(i); L1 norm summed in ascending word order,
    applied when > 0. Node -1 is an ordinary key."""
    v, fv = {}, {}
    for i in range(len(word)):
        w = float(weight[i])
        if not w > 0.0:
            continue
        k = int(word[i])
        v[k] = v[k] + w if k in v else w
        fv.setdefault(int(node[i]), []).append(i)
    norm = 0.0
    for k in sorted(v):
        norm += abs(v[k])
    if norm > 0.0:
        v = {k: x / norm for k, x in v.items()}
    words = sorted(v)
    nodes = sorted(fv)
    ptr = np.cumsum([0] + [len(fv[n]) for n in nodes]).astype(np.int32)
    return dict(word=np.asarray(words, np.int32), value=np.asarray([v[k] for k in words], np.float64),
                node=np.asarray(nodes, np.int32), ptr=ptr, feat=np.asarray([i for n in nodes for i in fv[n]], np.int32))


def assert_same(got, want):
    assert got["word"].tobytes() == want["word"].tobytes()
    assert got["value"].tobytes() == want["value"].tobytes()          # float64 bytes: bit-identical
    assert got["node"].tobytes() == want["node"].tobytes()
    assert got["ptr"].tobytes() == want["ptr"].tobytes()
    assert got["feat"].tobytes() == want["feat"].tobytes()


@pytest.mark.parametrize("k,levels,ragged,levelsup,n", [(10, 3, False, 1, 600), (10, 3, False, 4, 600), (6, 4, True, 2, 800),
                                                        (3, 5, True, 4, 500)])
def test_assembly_on_vocabulary_descents(k, levels, ragged, levelsup, n):
    """Seeded keyframes through the descent oracle: the plain keyframe, one with every other descriptor repeated (duplicate
    words), one with a third of the leaves stopped (weight 0), and the empty keyframe."""
    voc = make_voc(k, levels, seed=k + levels, ragged=ragged)
    stopped = dict(voc)
    stopped["weight"] = voc["weight"].copy()
    leaves = np.flatnonzero(voc["word_id"] >= 0)
    stopped["weight"][leaves[::3]] = 0.0
    f = make_features(voc, n, seed=levels)
    dup = np.repeat(f[: n // 2], 2, axis=0)
    seen_minus1 = False
    for v, feats in ((voc, f), (voc, dup), (stopped, f), (voc, f[:0])):
        word, weight, node = pyoracle.voc_transform(v, feats, levelsup)
        got = pybow.assemble(word, weight, node)
        assert_same(got, dict_assembly(word, weight, node))
        assert_same(pybow.compute_bow(v, feats, levelsup), got)
        seen_minus1 |= bool((got["node"] == -1).any())
        if len(feats):
            assert len(got["word"]) < (weight > 0).sum() or v is stopped      # some words collect several features
    if ragged and levelsup == 2:
        assert seen_minus1                                                      # a leaf above the requested level


def test_assembly_sums_in_feature_and_word_order():
    """Weights whose double sums depend on the order: a word's features 1, 1e16, 1 sum to 1e16 in feature order (2 + 1e16
    otherwise), and the norm over words in ascending order differs from other orders."""
    word = np.array([7, 7, 7, 3, 9, 3, 5], np.int32)
    weight = np.array([1.0, 1e16, 1.0, 0.1, 0.2, 0.3, 0.0])
    node = np.array([2, -1, 2, 0, -1, 5, 1], np.int32)
    got = pybow.assemble(word, weight, node)
    assert_same(got, dict_assembly(word, weight, node))
    assert got["word"].tolist() == [3, 7, 9] and got["node"].tolist() == [-1, 0, 2, 5]
    assert got["feat"].tolist() == [1, 4, 3, 0, 2, 5]
    s7 = (1.0 + 1e16) + 1.0
    norm = ((0.1 + 0.3) + s7) + 0.2
    assert got["value"].tolist() == [(0.1 + 0.3) / norm, s7 / norm, 0.2 / norm]


@pytest.mark.parametrize("seed", range(6))
def test_assembly_on_random_triples(seed):
    """Random triples over few words and nodes (many repeats), weights spread over 12 decades with a fifth of them 0 or
    negative-zero, node -1 among the keys; and all-stopped keyframes (norm 0: no word, no node)."""
    rng = np.random.default_rng(seed)
    n = int(rng.integers(1, 3000))
    word = rng.integers(0, 40, n).astype(np.int32)
    weight = 10.0 ** rng.uniform(-6, 6, n)
    weight[rng.random(n) < 0.1] = 0.0
    weight[rng.random(n) < 0.1] = -0.0
    node = rng.integers(-1, 25, n).astype(np.int32)
    got = pybow.assemble(word, weight, node)
    assert_same(got, dict_assembly(word, weight, node))
    assert abs(got["value"].sum() - 1.0) < 1e-12
    none = pybow.assemble(word, np.zeros(n), node)
    assert len(none["word"]) == 0 and len(none["node"]) == 0 and none["ptr"].tolist() == [0]
