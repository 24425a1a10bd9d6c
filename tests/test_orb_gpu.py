"""GPU parity of the ORB front-end against the CPU oracle and the committed golden vectors, through the C ABI.

Bar (BASELINE.md section 4): bit-exact keypoints (x, y, octave, response, angle, size) in identical order and
bit-exact 32-byte descriptors.
"""
import os

import numpy as np
import pytest

from oracle import pyoracle
from tools import synth
from se2lam_b200.orb import ORBextractor

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = np.load(os.path.join(ROOT, "tests", "golden", "orb_golden.npz"))
CASES = {
    "synth1000": lambda: synth.orb_frame(1000), "synth1001": lambda: synth.orb_frame(1001),
    "constant": lambda: synth.orb_adversarial("constant"), "noise": lambda: synth.orb_adversarial("noise"),
    "lowcontrast": lambda: synth.orb_adversarial("lowcontrast"), "gradient": lambda: synth.orb_adversarial("gradient"),
    "small_320x240": lambda: synth.orb_frame(5, 320, 240), "odd_501x377": lambda: synth.orb_frame(6, 501, 377),
}


def assert_same(kg, dg, ko, do_, what=""):
    assert len(kg) == len(ko), f"{what}: {len(kg)} vs {len(ko)} keypoints"
    for field in ("octave", "x", "y", "response", "angle", "size", "class_id"):
        bad = np.flatnonzero(kg[field].view(np.int32) != ko[field].view(np.int32))
        assert bad.size == 0, f"{what}: {field} differs at {bad[:5]} ({kg[field][bad[:5]]} vs {ko[field][bad[:5]]})"
    bad = np.flatnonzero((dg != do_).any(axis=1))
    assert bad.size == 0, f"{what}: {bad.size} descriptors differ, first at {bad[:5]}"


@pytest.fixture(scope="module")
def ext():
    return ORBextractor(1000, 1.2, 8, fastTh=20, max_width=640, max_height=480, max_batch=8)


@pytest.mark.parametrize("name", sorted(CASES))
def test_matches_golden_vectors(ext, name):
    img = CASES[name]()
    kps, desc = ext(img)
    assert_same(kps, desc, GOLD[name + "_kps"], GOLD[name + "_desc"], name)


def test_pyramid_and_blur_planes_bit_exact(ext):
    img = synth.orb_frame(1003)
    o = pyoracle.OrbOracle()
    ko, do_ = o.extract(img)
    kg, dg = ext(img)
    for level in range(8):
        po, w, h = o.level(level, False)
        pg, wg, hg = ext.level(0, level, False)
        assert (w, h) == (wg, hg)
        np.testing.assert_array_equal(pg[:, :w + 32], po[:, :w + 32], err_msg=f"plain level {level}")
        bo, _, _ = o.level(level, True)
        if bo is not None:
            bg, _, _ = ext.level(0, level, True)
            np.testing.assert_array_equal(bg[:, :w + 32], bo[:, :w + 32], err_msg=f"blurred level {level}")
    assert_same(kg, dg, ko, do_, "synth1003")


def test_batch_equals_single_frames_and_oracle(ext):
    imgs = synth.orb_batch(8, first_seed=2000)
    kps, desc, counts = ext.extract_batch(imgs)
    o = pyoracle.OrbOracle()
    for i in range(8):
        ko, do_ = o.extract(imgs[i])
        assert counts[i] == len(ko)
        assert_same(kps[i, :counts[i]], desc[i, :counts[i]], ko, do_, f"batch frame {i}")


@pytest.mark.parametrize("params", [dict(nfeatures=500, scaleFactor=1.2, nlevels=8, fastTh=20),
                                    dict(nfeatures=2000, scaleFactor=1.15, nlevels=6, fastTh=12),
                                    dict(nfeatures=800, scaleFactor=1.3, nlevels=5, fastTh=5),
                                    dict(nfeatures=1000, scaleFactor=1.2, nlevels=8, fastTh=40)])
def test_other_parameters(params):
    img = synth.orb_frame(77)
    e = ORBextractor(params["nfeatures"], params["scaleFactor"], params["nlevels"], fastTh=params["fastTh"])
    o = pyoracle.OrbOracle(params["nfeatures"], params["scaleFactor"], params["nlevels"], params["fastTh"])
    ko, do_ = o.extract(img)
    kg, dg = e(img)
    assert_same(kg, dg, ko, do_, str(params))


def test_strided_input_and_empty_image(ext):
    big = np.zeros((480, 704), np.uint8)
    img = synth.orb_frame(1004)
    big[:, 32:672] = img
    view = big[:, 32:672]
    kps = np.zeros((1, 1000), pyoracle.KP_DTYPE)
    from se2lam_b200._capi import lib, ptr, check
    desc = np.zeros((1, 1000, 32), np.uint8); counts = np.zeros(1, np.int32)
    check(lib().se2gpu_orb_extract(ext.h, view.ctypes.data, 1, 640, 480, big.strides[0], 0, ptr(kps), ptr(desc), ptr(counts)), "strided")
    ko, do_ = pyoracle.OrbOracle().extract(img)
    assert_same(kps[0, :counts[0]], desc[0, :counts[0]], ko, do_, "strided")
    k0, d0 = ext(np.zeros((0, 0), np.uint8))
    assert len(k0) == 0 and d0.shape == (0, 32)


def test_full_batch_properties():
    """BASELINE configs[1] size (64 frames): determinism (two runs identical), frame independence (a frame's
    result does not depend on its batch neighbours), every frame returns exactly nfeatures keypoints."""
    imgs = synth.orb_batch(64)
    e = ORBextractor(1000, 1.2, 8, max_batch=64)
    k1, d1, c1 = e.extract_batch(imgs)
    k2, d2, c2 = e.extract_batch(imgs[::-1].copy())
    assert np.all(c1 == 1000)
    assert k1.tobytes() == k2[::-1].tobytes() and d1.tobytes() == d2[::-1].tobytes()
    o = pyoracle.OrbOracle()
    for i in (0, 31, 63):
        ko, do_ = o.extract(imgs[i])
        assert_same(k1[i], d1[i], ko, do_, f"frame {i} of 64")


def test_warp_nth_element_matches_std_nth_element():
    """The warp-cooperative introselect must produce libstdc++'s permutation (ties decide which keypoints survive
    retainBest, ORBextractor.cpp:692/:708): thousands of tie-heavy lists against the oracle's real std::nth_element."""
    from se2lam_b200 import _capi
    rng = np.random.default_rng(7)
    lists, nths = [], []
    for case in range(1500):
        kind = case % 5
        n = int(rng.integers(1, 40)) if kind == 0 else int(rng.integers(40, 3000))
        if kind == 1:
            sc = rng.integers(0, 3, n)                    # almost everything tied
        elif kind == 2:
            sc = np.sort(rng.integers(0, 256, n))[::-1]   # already ordered
        elif kind == 3:
            sc = np.sort(rng.integers(0, 256, n))         # reversed
        else:
            sc = rng.integers(0, int(rng.integers(2, 256)), n)
        lists.append(sc.astype(np.uint32))
        nths.append(int(rng.integers(0, n)))
    # organ-pipe / sawtooth lists exercise the depth limit (heap-select fallback)
    for n in (64, 257, 1024, 2048):
        half = np.arange(n // 2, dtype=np.uint32) % 251
        lists.append(np.concatenate([half, half[::-1]])); nths.append(n // 2)
        lists.append((np.arange(n, dtype=np.uint32) * 37 % 17)); nths.append(n - 2)
    offs = np.zeros(len(lists) + 1, np.int32)
    offs[1:] = np.cumsum([len(x) for x in lists])
    packed = np.concatenate([(sc << 24) | np.arange(len(sc), dtype=np.uint32) for sc in lists]).astype(np.uint32)
    got = packed.copy()
    nth = np.asarray(nths, np.int32)
    _capi.check(_capi.lib().se2gpu_orb_debug_nth_element(got.ctypes.data, offs.ctypes.data, nth.ctypes.data, len(lists), 0), "nth")
    for k, sc in enumerate(lists):
        ids = pyoracle.nth_element(sc.astype(np.float32), nths[k])
        want = packed[offs[k]:offs[k + 1]][ids]
        assert np.array_equal(got[offs[k]:offs[k + 1]], want), f"list {k} (n={len(sc)}, nth={nths[k]})"


def test_hd_frame_big_cells():
    """1920x1080 with 1000 features has 470 x 150 px grid cells: too large for the compacting FAST kernel's shared-memory
    candidate list, so the one-thread-per-pixel fallback kernel runs; results must still be bit-exact. 1280x720 with 1000
    features (level-0 cells 312 x 99 px) exceeds the 256 px TMA box and takes the plain-load instantiation of the compacting
    kernel; 1024x768 with 1500 features takes its TMA instantiation."""
    img = synth.orb_frame(4242, 1920, 1080)
    ext = ORBextractor(1000, 1.2, 8, fastTh=20, max_width=1920, max_height=1080, max_batch=1)
    kg, dg = ext(img)
    ko, do_ = pyoracle.OrbOracle(1000, 1.2, 8, 20).extract(img)
    assert_same(kg, dg, ko, do_, "1080p")
    img1 = synth.orb_frame(4244, 1280, 720)
    ext1 = ORBextractor(1000, 1.2, 8, fastTh=20, max_width=1280, max_height=720, max_batch=1)
    kg1, dg1 = ext1(img1)
    ko1, do1 = pyoracle.OrbOracle(1000, 1.2, 8, 20).extract(img1)
    assert_same(kg1, dg1, ko1, do1, "720p")
    img2 = synth.orb_frame(4243, 1024, 768)
    ext2 = ORBextractor(1500, 1.2, 8, fastTh=20, max_width=1024, max_height=768, max_batch=1)
    kg2, dg2 = ext2(img2)
    ko2, do2 = pyoracle.OrbOracle(1500, 1.2, 8, 20).extract(img2)
    assert_same(kg2, dg2, ko2, do2, "1024x768")


def test_undistort_folded_into_level0():
    """se2gpu_orb_set_undistort: raw frame in, keypoints/descriptors of cv::undistort(frame) out (reference Frame.cpp:22-25),
    checked against oracle undistort -> oracle extract, and the level-0 plane against copyMakeBorder(undistorted)."""
    K = np.array([[520.9, 0, 325.1], [0, 521.0, 249.7], [0, 0, 1]], np.float32)
    D = np.array([0.2312, -0.7849, -0.0033, -0.0001, 0.9172], np.float32)
    ext = ORBextractor(1000, 1.2, 8, fastTh=20, max_width=640, max_height=480, max_batch=4)
    orc = pyoracle.OrbOracle(1000, 1.2, 8, 20)
    raw = synth.orb_frame(1000)
    ext.set_undistort(K, D)
    kg, dg = ext(raw)
    und = pyoracle.undistort(raw, K, D)
    ko, do_ = orc.extract(und)
    assert_same(kg, dg, ko, do_, "undistort 640x480")
    plane, w, h = ext.level(0, 0)
    assert np.array_equal(plane[16:16 + h, 16:16 + w], und)
    # batch through the pipelined host path, other coefficient counts and an odd frame size
    batch = np.stack([synth.orb_frame(1000 + i) for i in range(4)])
    kps, desc, counts = ext.extract_batch(batch)
    for i in range(4):
        ko, do_ = orc.extract(pyoracle.undistort(batch[i], K, D))
        assert_same(kps[i, :counts[i]], desc[i, :counts[i]], ko, do_, f"undistort batch frame {i}")
    K2 = np.array([[700.0, 0, 250.5], [0, 701.0, 188.5], [0, 0, 1]], np.float32)
    D2 = np.array([0.05, 0.0, 0.0, 0.0, 0.0, 0.01, 0.0, 0.0], np.float32)
    ext.set_undistort(K2, D2)
    raw2 = synth.orb_frame(6, 501, 377)
    kg, dg = ext(raw2)
    ko, do_ = orc.extract(pyoracle.undistort(raw2, K2, D2))
    assert_same(kg, dg, ko, do_, "undistort 501x377")
    ext.set_undistort(None)                      # off again: plain extraction
    kg, dg = ext(raw)
    ko, do_ = orc.extract(raw)
    assert_same(kg, dg, ko, do_, "undistort off")


def test_submit_wait_pipeline_matches_synchronous_extract():
    """se2gpu_orb_submit / _wait (two batches in flight on twin contexts) returns exactly what se2gpu_orb_extract returns."""
    n = 6
    batches = [synth.orb_batch(n, first_seed=3000 + 10 * k) for k in range(5)]
    e = ORBextractor(1000, 1.2, 8, max_batch=n)
    ref = [e.extract_batch(b) for b in batches]
    outs = [(np.zeros((n, 1000), pyoracle.KP_DTYPE), np.zeros((n, 1000, 32), np.uint8), np.zeros(n, np.int32)) for _ in range(2)]
    got = []
    for k, b in enumerate(batches):
        e.submit(b, *outs[k & 1])
        if k >= 1:
            e.wait()
            got.append(tuple(a.copy() for a in outs[(k - 1) & 1]))
    e.wait()
    got.append(tuple(a.copy() for a in outs[(len(batches) - 1) & 1]))
    with pytest.raises(Exception):
        e.submit(batches[0], *outs[0]); e.submit(batches[1], *outs[1]); e.submit(batches[2], *outs[0])    # a third batch in flight is refused
    e.wait(); e.wait()
    for (kr, dr, cr), (kg, dg, cg) in zip(ref, got):
        np.testing.assert_array_equal(cg, cr)
        for i in range(n):
            assert kg[i, :cr[i]].tobytes() == kr[i, :cr[i]].tobytes() and dg[i, :cr[i]].tobytes() == dr[i, :cr[i]].tobytes()
