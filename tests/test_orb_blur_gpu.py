"""orb_blur against the CPU oracle where its strips, column groups and tiles fall differently from 640x480 with 8 levels at scale
1.2 (tests/test_orb_gpu.py::test_pyramid_and_blur_planes_bit_exact): odd and HD frame sizes and another scale factor and level
count. Every level's blurred plane (ROI and the un-blurred 16 px ring) must match bit for bit, for the second frame of a batch."""
import numpy as np
import pytest

from oracle import pyoracle
from tools import synth
from se2lam_b200.orb import ORBextractor

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("w,h,nfeatures,scale,nlevels", [(501, 377, 1000, 1.2, 8), (1280, 720, 1000, 1.2, 8), (800, 600, 1200, 1.3, 5)])
def test_blurred_planes_match_the_oracle(w, h, nfeatures, scale, nlevels):
    imgs = np.stack([synth.orb_frame(s, w, h) for s in (31, 32)])
    ext = ORBextractor(nfeatures, scale, nlevels, fastTh=20, max_width=w, max_height=h, max_batch=2)
    ext.extract_batch(imgs)
    o = pyoracle.OrbOracle(nfeatures, scale, nlevels, 20)
    o.extract(imgs[1])
    for level in range(nlevels):
        bo, lw, lh = o.level(level, True)
        assert bo is not None, f"the oracle did not blur level {level}"   # it blurs levels that keep keypoints
        bg, wg, hg = ext.level(1, level, True)
        assert (wg, hg) == (lw, lh)
        np.testing.assert_array_equal(bg[:, :lw + 32], bo[:, :lw + 32], err_msg=f"{w}x{h} scale {scale}: blurred level {level}")
