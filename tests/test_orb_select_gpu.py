"""GPU parity of the two-launch keypoint selection (orb_select_cells: quota redistribution + retainBest per cell, one warp per
cell; orb_select_levels: retainBest per level) against the CPU oracle, level by level: which tied keypoints survive and their
order come from libstdc++'s nth_element permutation, so every level's keypoints must match in order, bit for bit.

Frames: 'noise' (quota saturation, massive ties), 'lowcontrast' (the threshold-7 fallback everywhere), 'constant' (no keypoint),
and a few features on noise, whose 4-cell level 0 puts thousands of candidates in each cell list (longer than the per-warp
shared-memory stage, so those lists are selected in place in global memory). Batches of 1 and 64, through the device entry
point (the blur on its side stream) and through the chunked host path (launch groups with a frame offset), FAST and Harris
scores."""
import numpy as np
import pytest
import torch

from oracle import pyharris, pyoracle
from se2lam_b200.orb import FAST_SCORE, HARRIS_SCORE, ORBextractor
from tools import synth

pytestmark = pytest.mark.gpu

FIELDS = ("octave", "x", "y", "response", "angle", "size", "class_id")
FRAMES = {
    "noise": lambda: synth.orb_adversarial("noise"), "lowcontrast": lambda: synth.orb_adversarial("lowcontrast"),
    "constant": lambda: synth.orb_adversarial("constant"), "synth1000": lambda: synth.orb_frame(1000),
}


def oracle(score, nf, sf, nl, th):
    return pyharris.HarrisOrbOracle(nf, sf, nl, th) if score == HARRIS_SCORE else pyoracle.OrbOracle(nf, sf, nl, th)


def assert_levels_same(kg, dg, ko, do_, nlevels, what):
    for level in range(nlevels):
        g, o = kg["octave"] == level, ko["octave"] == level
        assert g.sum() == o.sum(), f"{what} level {level}: {g.sum()} vs {o.sum()} keypoints"
        for field in FIELDS:
            a, b = kg[field][g].view(np.int32), ko[field][o].view(np.int32)
            bad = np.flatnonzero(a != b)
            assert bad.size == 0, f"{what} level {level}: {field} differs at {bad[:5]}"
        bad = np.flatnonzero((dg[g] != do_[o]).any(axis=1))
        assert bad.size == 0, f"{what} level {level}: {bad.size} descriptors differ"
    assert len(kg) == len(ko), f"{what}: {len(kg)} vs {len(ko)} keypoints"
    np.testing.assert_array_equal(kg["octave"], ko["octave"], err_msg=f"{what}: level order")


def device_extract(ext, imgs, nf):
    """se2gpu_orb_extract_device on a batch already on the GPU (frame offset 0, blur on the side stream)."""
    n, h, w = imgs.shape
    dev = torch.device("cuda", 0)
    d_imgs = torch.from_numpy(np.ascontiguousarray(imgs)).to(dev)
    d_kps = torch.zeros(n * nf * 28, dtype=torch.uint8, device=dev)
    d_desc = torch.zeros(n * nf * 32, dtype=torch.uint8, device=dev)
    d_counts = torch.zeros(n, dtype=torch.int32, device=dev)
    ext.extract_device(d_imgs, n, h, w, d_kps, d_desc, d_counts, stream=torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    from se2lam_b200 import _capi
    kps = d_kps.cpu().numpy().view(_capi.KP_DTYPE).reshape(n, nf)
    return kps, d_desc.cpu().numpy().reshape(n, nf, 32), d_counts.cpu().numpy()


PARAMS = {"default": (1000, 1.2, 8, 20), "few_features": (150, 1.2, 4, 20)}


@pytest.mark.parametrize("score", [FAST_SCORE, HARRIS_SCORE], ids=["fast", "harris"])
@pytest.mark.parametrize("params", sorted(PARAMS))
@pytest.mark.parametrize("name", sorted(FRAMES))
def test_single_frame(score, params, name):
    nf, sf, nl, th = PARAMS[params]
    img = FRAMES[name]()
    ext = ORBextractor(nf, sf, nl, score, th, max_width=640, max_height=480, max_batch=1)
    kg, dg = ext(img)
    ko, do_ = oracle(score, nf, sf, nl, th).extract(img)
    assert_levels_same(kg, dg, ko, do_, nl, f"{name}/{params}")


@pytest.mark.parametrize("score", [FAST_SCORE, HARRIS_SCORE], ids=["fast", "harris"])
@pytest.mark.parametrize("path", ["device", "host_chunked"])
def test_batch_64(score, path):
    nf, sf, nl, th = PARAMS["default"]
    names = sorted(FRAMES)
    distinct = [FRAMES[n]() for n in names] + [synth.orb_frame(3000 + i) for i in range(4)]
    order = [(7 * i) % len(distinct) for i in range(64)]
    imgs = np.stack([distinct[k] for k in order])
    ext = ORBextractor(nf, sf, nl, score, th, max_width=640, max_height=480, max_batch=64)
    if path == "device":
        kps, desc, counts = device_extract(ext, imgs, nf)
    else:
        kps, desc, counts = ext.extract_batch(imgs)      # split into launch groups whose first frame is not frame 0
    o = oracle(score, nf, sf, nl, th)
    ref = [o.extract(img) for img in distinct]
    for i, k in enumerate(order):
        ko, do_ = ref[k]
        assert counts[i] == len(ko), f"frame {i}: {counts[i]} vs {len(ko)} keypoints"
        assert_levels_same(kps[i, :counts[i]], desc[i, :counts[i]], ko, do_, nl, f"{path} frame {i}")
