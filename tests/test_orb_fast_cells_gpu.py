"""orb_fast_cells against the CPU oracle where its candidate lists, its non-maximum suppression and its emission are pushed to
their ends: fastTh 1 (nearly every pixel survives the screen, so the lists are full and cells emit the most keypoints), 60, and
254 (no corner on these frames reaches it, so every cell runs the threshold-7 pass as well), and periodic textures whose equal
scores meet across cell boundaries. 640x480 frames take the TMA-staged instantiation, 1280x720 at 1000 features the plain-load
one. The whole extract_batch output (keypoints, descriptors and counts of every frame) must match bit for bit."""
import numpy as np
import pytest

from oracle import pyoracle
from tools import synth
from se2lam_b200.orb import ORBextractor

pytestmark = pytest.mark.gpu


def assert_batch_matches_oracle(imgs, nfeatures, fast_th):
    h, w = imgs.shape[1:]
    ext = ORBextractor(nfeatures, 1.2, 8, fastTh=fast_th, max_width=w, max_height=h, max_batch=len(imgs))
    kps, desc, counts = ext.extract_batch(imgs)
    o = pyoracle.OrbOracle(nfeatures, 1.2, 8, fast_th)
    for i in range(len(imgs)):
        ko, do_ = o.extract(imgs[i])
        what = f"{w}x{h} fastTh {fast_th} frame {i}"
        assert counts[i] == len(ko), f"{what}: {counts[i]} vs {len(ko)} keypoints"
        assert kps[i, :counts[i]].tobytes() == ko.tobytes(), f"{what}: keypoints differ"
        assert desc[i, :counts[i]].tobytes() == do_.tobytes(), f"{what}: descriptors differ"


def tiled_frames(w, h):
    """Periodic textures: every corner of a tile has the same score as its copies, and the copies meet across cell edges."""
    y, x = np.mgrid[0:h, 0:w]
    squares = np.where((x % 7 < 3) & (y % 6 < 3), 200, 40)                     # 3x3 bright squares on a 7x6 lattice
    checker = np.where(((x // 4) + (y // 4)) % 2 == 0, 180, 60)                  # 4 px checkerboard
    dots = np.where(((x % 5) == 2) & ((y % 5) == 2), 250, 90)                    # isolated bright pixels every 5 px
    rolled = np.roll(squares, (1, 2), axis=(0, 1))
    return np.stack([squares, checker, dots, rolled]).astype(np.uint8)


@pytest.mark.parametrize("fast_th", [1, 60, 254])
@pytest.mark.parametrize("w,h", [(640, 480), (1280, 720)])
def test_extreme_thresholds_match_the_oracle(w, h, fast_th):
    imgs = np.stack([synth.orb_frame(s, w, h) for s in (1000, 1001)] + [synth.orb_adversarial("noise", w, h)])
    assert_batch_matches_oracle(imgs, 1000, fast_th)


@pytest.mark.parametrize("w,h", [(640, 480), (1280, 720)])
def test_equal_scores_across_cell_edges_match_the_oracle(w, h):
    assert_batch_matches_oracle(tiled_frames(w, h), 1000, 20)
