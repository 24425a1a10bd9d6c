"""orb_resize_w's tall tiles (RESIZE_TR_TALL rows) against the CPU oracle. run_device picks them only for levels whose grid of
tall tiles fills every resident CTA slot of the GPU, i.e. for large batches, so these cases use batches big enough for the
large levels to take tall tiles and the small levels to keep 32-row tiles. Every plain level plane (ROI and 16 px border) of
the first, a middle and the last frame must match byte for byte, and the pitch padding must be zero."""
import numpy as np
import pytest
import torch

from oracle import pyoracle
from tools import synth
from se2lam_b200.orb import ORBextractor

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("n,w,h,scale,nlevels", [(64, 640, 480, 1.2, 8), (24, 1280, 720, 1.2, 8), (64, 640, 480, 1.3, 6)])
def test_tall_tile_levels_match_the_oracle(n, w, h, scale, nlevels):
    imgs = synth.orb_batch(n, first_seed=4700, w=w, h=h)
    ext = ORBextractor(1000, scale, nlevels, fastTh=20, max_width=w, max_height=h, max_batch=n)
    d = torch.from_numpy(imgs).cuda()
    kps = torch.empty(n * 1000 * 28, dtype=torch.uint8, device="cuda")
    desc = torch.empty(n * 1000 * 32, dtype=torch.uint8, device="cuda")
    counts = torch.zeros(n, dtype=torch.int32, device="cuda")
    ext.extract_device(d, n, h, w, kps, desc, counts)
    torch.cuda.synchronize()
    orc = pyoracle.OrbOracle(1000, scale, nlevels, 20)
    for i in (0, n // 2, n - 1):
        orc.extract(imgs[i])
        for level in range(nlevels):
            po, lw, lh = orc.level(level, False)
            pg, wg, hg = ext.level(i, level, False)
            assert (wg, hg) == (lw, lh)
            np.testing.assert_array_equal(pg[:, :lw + 32], po[:, :lw + 32], err_msg=f"{w}x{h} batch {n} frame {i}: plain level {level}")
            assert not pg[:, lw + 32:].any(), f"{w}x{h} batch {n} frame {i}: pitch padding of level {level} is not zero"
