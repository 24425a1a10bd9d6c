"""The image pyramid (orb_pyr0 + orb_resize_w) against the CPU oracle: every plain level plane, ROI and 16 px border, byte for
byte, and zero pitch padding. Covers every frame of a batch (a launch writing the wrong frame or level), the chunked host path
(frame offset != 0) and submit / wait, frame sizes whose tiles fall differently, scale factors up to the byte path of the
horizontal pass (above ~2.6), level 0 from orb_pyr0_undistort, unaligned input rows (the bytewise level-0 path), and a batch of
one frame next to a larger batch."""
import numpy as np
import pytest
import torch

from oracle import pyoracle
from tools import synth
from se2lam_b200 import _capi
from se2lam_b200.orb import ORBextractor

pytestmark = pytest.mark.gpu


def assert_planes(ext, frame, orc, nlevels, what):
    for level in range(nlevels):
        po, w, h = orc.level(level, False)
        pg, wg, hg = ext.level(frame, level, False)
        assert (wg, hg) == (w, h), f"{what}: level {level} size"
        np.testing.assert_array_equal(pg[:, :w + 32], po[:, :w + 32], err_msg=f"{what}: plain level {level}")
        assert not pg[:, w + 32:].any(), f"{what}: pitch padding of level {level} is not zero"


def check_batch(ext, imgs, nfeatures, scale, nlevels, what, frames=None):
    orc = pyoracle.OrbOracle(nfeatures, scale, nlevels, 20)
    for i in (range(len(imgs)) if frames is None else frames):
        orc.extract(imgs[i])
        assert_planes(ext, i, orc, nlevels, f"{what} frame {i}")


def test_every_frame_of_a_batch():
    imgs = synth.orb_batch(8, first_seed=4100)
    ext = ORBextractor(1000, 1.2, 8, fastTh=20, max_width=640, max_height=480, max_batch=8)
    ext.extract_batch(imgs)      # host path in chunks over the pipeline lanes: frame offsets 0 and != 0
    check_batch(ext, imgs, 1000, 1.2, 8, "640x480 chunked")
    d = torch.from_numpy(imgs).cuda()
    kps = torch.empty(8 * 1000 * 28, dtype=torch.uint8, device="cuda")
    desc = torch.empty(8 * 1000 * 32, dtype=torch.uint8, device="cuda")
    counts = torch.zeros(8, dtype=torch.int32, device="cuda")
    ext.extract_device(d, 8, 480, 640, kps, desc, counts)      # one launch for the batch
    torch.cuda.synchronize()
    check_batch(ext, imgs, 1000, 1.2, 8, "640x480 device")


def test_submit_wait():
    imgs = synth.orb_batch(4, first_seed=4200)
    ext = ORBextractor(1000, 1.2, 8, max_batch=4)
    kps = np.zeros((4, 1000), _capi.KP_DTYPE)
    desc = np.zeros((4, 1000, 32), np.uint8)
    counts = np.zeros(4, np.int32)
    ext.submit(imgs, kps, desc, counts)
    ext.wait()
    check_batch(ext, imgs, 1000, 1.2, 8, "submit")


@pytest.mark.parametrize("w,h", [(320, 240), (501, 377), (1280, 720), (1920, 1080)])
def test_frame_sizes(w, h):
    imgs = np.stack([synth.orb_frame(s, w, h) for s in (41, 42)])
    ext = ORBextractor(1000, 1.2, 8, fastTh=20, max_width=w, max_height=h, max_batch=2)
    ext.extract_batch(imgs)
    check_batch(ext, imgs, 1000, 1.2, 8, f"{w}x{h}")


@pytest.mark.parametrize("scale,nlevels", [(1.15, 8), (1.3, 6), (3.0, 3)])
def test_scale_factors(scale, nlevels):
    imgs = np.stack([synth.orb_frame(s, 640, 480) for s in (51, 52)])
    ext = ORBextractor(1000, scale, nlevels, fastTh=20, max_width=640, max_height=480, max_batch=2)
    ext.extract_batch(imgs)
    check_batch(ext, imgs, 1000, scale, nlevels, f"scale {scale}")


def test_undistort_skips_level0():
    K = np.array([[520.9, 0, 325.1], [0, 521.0, 249.7], [0, 0, 1]], np.float32)
    D = np.array([0.2312, -0.7849, -0.0033, -0.0001, 0.9172], np.float32)
    raw = synth.orb_batch(3, first_seed=4300)
    ext = ORBextractor(1000, 1.2, 8, max_batch=3)
    ext.set_undistort(K, D)
    ext.extract_batch(raw)
    und = np.stack([pyoracle.undistort(raw[i], K, D) for i in range(3)])
    check_batch(ext, und, 1000, 1.2, 8, "undistort")


def test_unaligned_rows():
    w, h, stride = 640, 480, 643
    imgs = synth.orb_batch(2, first_seed=4400)
    padded = np.zeros((2, h, stride), np.uint8)
    padded[:, :, :w] = imgs
    d = torch.from_numpy(padded).cuda()
    ext = ORBextractor(1000, 1.2, 8, max_batch=2)
    kps = torch.empty(2 * 1000 * 28, dtype=torch.uint8, device="cuda")
    desc = torch.empty(2 * 1000 * 32, dtype=torch.uint8, device="cuda")
    counts = torch.zeros(2, dtype=torch.int32, device="cuda")
    ext.extract_device(d, 2, h, w, kps, desc, counts, stride=stride, frame_stride=h * stride)
    torch.cuda.synchronize()
    check_batch(ext, imgs, 1000, 1.2, 8, "unaligned rows")


@pytest.mark.parametrize("n", [1, 16])
def test_batch_sizes(n):
    imgs = synth.orb_batch(n, first_seed=4500)
    ext = ORBextractor(1000, 1.2, 8, max_batch=n)
    d = torch.from_numpy(imgs).cuda()
    kps = torch.empty(n * 1000 * 28, dtype=torch.uint8, device="cuda")
    desc = torch.empty(n * 1000 * 32, dtype=torch.uint8, device="cuda")
    counts = torch.zeros(n, dtype=torch.int32, device="cuda")
    ext.extract_device(d, n, 480, 640, kps, desc, counts)
    torch.cuda.synchronize()
    check_batch(ext, imgs, 1000, 1.2, 8, f"batch {n}", frames=sorted({0, n // 2, n - 1}))
