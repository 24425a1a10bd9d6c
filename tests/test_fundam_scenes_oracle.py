"""CPU checks that the scene families of tests/fundam_scenes.py reach the estimator branches they are there for, on the
oracle (oracle/fundam_oracle.cpp): zero motion with and without a model, first-draw and later getSubset give-ups,
keypoint-lattice coordinates and full capacity. tests/test_fundam_paths_gpu.py holds the GPU to the oracle on them."""
import numpy as np
import pytest

from oracle import pyfundam
from tests import fundam_scenes as fs


@pytest.fixture(scope="module")
def scenes():
    return fs.all_scenes()


@pytest.fixture(scope="module")
def results(scenes):
    return [pyfundam.find_fundamental_mat(s.p1, s.p2) for s in scenes]


def _final_niters(n, good):
    """niters when the RANSAC loop ends: every accepted model lowers it, the best (last accepted) model sets it."""
    return min(1000, pyfundam.niters((n - good) / n)) if good > 6 else 1000


def test_keypoint_dtype_is_the_abi_one():
    from se2lam_b200._capi import KP_DTYPE
    assert fs.KP_DTYPE == KP_DTYPE


@pytest.mark.parametrize("family", ["static", "lattice", "collinear", "duplicate", "giveup"])
def test_each_scene_reaches_its_branch(scenes, results, family):
    sel = [(s, r) for s, r in zip(scenes, results) if s.family == family]
    assert sel
    for s, (mask, F, it) in sel:
        tag = (repr(s), s.n, it)
        assert mask is not None and len(mask) == s.n, tag
        good = int(mask.sum())
        if s.expect in ("static", "static-none", "static-model"):
            assert np.array_equal(s.p1, s.p2), tag
            if s.n == 7:
                assert good == 7 and it == 1, tag
            elif good == 0:
                # every hypothesis ran and none produced a model: each elimination stopped at its pivot test
                assert it == (300 if s.branch == "lmeds" else 1000) and len(F) == 0, tag
            else:
                # a model through every point; RANSAC stops on its niters update (LMedS always runs its 300)
                assert good == s.n and len(F) == 3 and 0 < it <= 1000, tag
            if s.expect == "static-none":
                assert good == 0, tag
            if s.expect == "static-model":
                assert good == s.n and it < 1000, tag
        elif s.expect == "ransac":
            assert s.branch == "ransac" and good > 6 and len(F) == 3 and 0 < it <= 1000, tag
        elif s.expect == "lmeds":
            # all 300 hypotheses, and a model the median threshold keeps at least 7 pairs of
            assert s.branch == "lmeds" and it == 300 and good >= 7 and len(F) == 3, tag
        elif s.expect == "first-draw":
            # getSubset exhausts its attempts before the first hypothesis: no estimate, an empty F, the mask all zeros
            assert it == 0 and good == 0 and len(F) == 0, tag
        elif s.expect == "giveup":
            # getSubset gave up after some hypotheses and before the iteration count reached niters
            assert s.n >= 1000 and good > 6 and len(F) == 3, tag
            assert 0 < it < _final_niters(s.n, good), tag
        else:
            assert s.expect == "any", tag


def test_zero_motion_takes_both_outcomes(scenes, results):
    got = {(s.branch, int(r[0].sum()) > 0) for s, r in zip(scenes, results) if s.family == "static" and s.expect != "ransac"}
    assert {("ransac", False), ("ransac", True), ("lmeds", False), ("lmeds", True)} <= got


def test_first_draw_give_ups_on_both_estimators(scenes, results):
    first = {s.branch for s, r in zip(scenes, results) if s.expect == "first-draw" and r[2] == 0}
    assert first == {"lmeds", "ransac"}


def test_hypothesis_counts_span_the_wave_edges(scenes, results):
    """The device scores 32 hypotheses per wave: the counts include ones below a wave, ones that end mid-wave, and 1000."""
    its = [r[2] for s, r in zip(scenes, results) if s.n > 7]
    assert any(0 < i < 32 for i in its)
    assert any(i % 32 and i > 32 for i in its)
    assert 1000 in its and 0 in its
    giveups = [r[2] for s, r in zip(scenes, results) if s.expect == "giveup"]
    assert min(giveups) < 32 and max(giveups) > 32 and any(i % 32 for i in giveups)


def test_lattice_coordinates_are_keypoint_like(scenes):
    for s in scenes:
        if s.family != "lattice":
            continue
        for p in (s.p1, s.p2):
            on = np.zeros(s.n, bool)
            for level in range(8):
                step = np.float32(np.float64(fs.SCALE) ** level)
                k = np.round(p / step)
                on |= ((k.astype(np.float32) * step) == p).all(1)
            assert on.all(), repr(s)
        if s.n >= 1000:
            # shared rows (equal y) are common, which is what makes collinear redraws and error ties likely
            assert len(np.unique(s.p1[:, 1])) < 0.8 * s.n, repr(s)


def test_capacity_scenes():
    full = [s for s in fs.all_scenes() if s.n == fs.MAX_PAIRS]
    assert {s.family for s in full} == {"static", "lattice"}
    for s in full:
        kp1, kp2, m = s.keypoints()
        assert len(kp1) == fs.MAX_PAIRS and (m >= 0).all() and len(kp2) <= fs.MAX_PAIRS
    kp1, kp2, m = fs.sparse_capacity_pair()
    assert len(kp1) == len(kp2) == fs.MAX_PAIRS and (m >= 0).sum() == 20


def test_remove_outliers_ignores_the_interleaving(scenes, results):
    """The same matched pairs surrounded by other unmatched keypoints give the same result, and it is the mask of
    findFundamentalMat with the 10-inlier rule."""
    for s, (mask, F, it) in zip(scenes, results):
        out = []
        for variant in (0, 1):
            kp1, kp2, m = s.keypoints(variant=variant)
            nin, m2, F2, it2 = pyfundam.remove_outliers(kp1, kp2, m)
            slots = np.flatnonzero(m >= 0)
            assert np.array_equal(m2[m < 0], m[m < 0]), repr(s)
            kept = m2[slots] >= 0
            assert np.array_equal(m2[slots][kept], m[slots][kept]), repr(s)
            out.append((nin, kept, F2.tobytes(), it2))
        assert out[0][0] == out[1][0] and np.array_equal(out[0][1], out[1][1]), repr(s)
        assert out[0][2:] == out[1][2:], repr(s)
        want = mask.astype(bool) if mask.sum() >= 10 else np.zeros(s.n, bool)
        assert np.array_equal(out[0][1], want) and out[0][0] == int(want.sum()) and out[0][3] == it, repr(s)
        assert out[0][2] == (F[:3] if len(F) else np.zeros((3, 3))).tobytes(), repr(s)


def test_lmeds_errors_of_the_returned_model_are_not_nan(scenes, results):
    """A NaN epipolar error would enter the LMedS median by its bit pattern, which differs between x86 and the GPU."""
    for s, (mask, F, it) in zip(scenes, results):
        if s.branch != "lmeds" or len(F) == 0:
            continue
        x1 = np.c_[s.p1.astype(np.float64), np.ones(s.n)]; x2 = np.c_[s.p2.astype(np.float64), np.ones(s.n)]
        l2, l1 = x1 @ F.T, x2 @ F            # epipolar lines in image 2 and image 1
        with np.errstate(all="ignore"):
            e1 = np.sum(x1 * l1, 1) ** 2 / (l1[:, 0] ** 2 + l1[:, 1] ** 2)
            e2 = np.sum(x2 * l2, 1) ** 2 / (l2[:, 0] ** 2 + l2[:, 1] ** 2)
        assert not np.isnan(e1).any() and not np.isnan(e2).any(), repr(s)
