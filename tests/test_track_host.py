"""The tracker's host part (updateFramePose, the pre-integration and needNewKF, run on the host by every step) against
the C++ oracle bit for bit, and the oracle against an independent numpy restatement. No GPU needed."""
import math

import numpy as np
import pytest

from oracle import pytrack, track_numpy
from tools import track_scenes as ts


@pytest.fixture(scope="module")
def cfg():
    from se2lam_b200 import build
    build.build_lib()
    return ts.config()


def _params(cfg):
    from se2lam_b200 import track
    return track.params(cfg["nfeatures"], cfg["scale_factor"], cfg["nlevels"], cfg["K"], cfg["grid"], cfg["lower_depth"],
                        cfg["upper_depth"], cfg["cTb"], cfg["bTc"], cfg["odo_noise"], cfg["max_frames"], cfg["min_frames"])


def odometries(seed, n=400):
    rng = np.random.default_rng(seed)
    out = []
    for k in range(n):
        kind = k % 4
        if kind == 0:     # general
            a = rng.uniform(-3, 3, (3, 3))
        elif kind == 1:   # angles around +-pi: the wrap of normalize_angle
            a = rng.uniform(-0.5, 0.5, (3, 3)); a[:, 2] = rng.choice([math.pi, -math.pi], 3) + rng.uniform(-1e-3, 1e-3, 3)
        elif kind == 2:   # near-zero motion
            base = rng.uniform(-1, 1, 3); a = np.stack([base, base + rng.uniform(-1e-6, 1e-6, 3), base])
        else:             # thresholds of c5 / c6
            a = np.zeros((3, 3)); a[0] = rng.uniform(-1, 1, 3); a[1] = a[0]; a[1, 2] += rng.choice([0.0349, -0.0349, 0.0348, 0.035])
            a[1, 0] += rng.choice([0.0, 0.0523 * 10 * 0.1, 0.05])
        out.append(a.astype(np.float32))
    return out


def test_pose_matches_oracle_and_numpy(cfg):
    from se2lam_b200 import track
    p = _params(cfg)
    for odo, kf, last in odometries(1):
        meas = np.random.default_rng(int(abs(odo[0]) * 1e6)).uniform(-1, 1, 3)
        cov = np.random.default_rng(2).uniform(0, 1e-3, 9)
        T1, m1, c1 = track.host_pose(p, odo, kf, last, meas, cov)
        T2, m2, c2 = pytrack.pose(cfg, odo, kf, last, meas, cov)
        T3, m3, c3 = track_numpy.pose(cfg, odo, kf, last, meas, cov)
        assert T1.tobytes() == T2.tobytes() == T3.tobytes()
        assert m1.tobytes() == m2.tobytes() == m3.tobytes()
        assert c1.tobytes() == c2.tobytes() == c3.tobytes()


def test_decisions_match_oracle_and_numpy(cfg):
    from se2lam_b200 import track
    p = _params(cfg)
    rng = np.random.default_rng(3)
    seen = set()
    for odo, kf, _ in odometries(4):
        for _ in range(4):
            args = (int(rng.integers(0, 20)), int(rng.integers(0, 300)), int(rng.integers(0, 400)), int(rng.integers(0, 90)),
                    int(rng.integers(0, 120)))
            for accept in (True, False):
                r1 = track.host_decide(p, *args, odo, kf, accept)
                r2 = pytrack.decide(cfg, *args, odo, kf, accept)
                r3 = track_numpy.decide(cfg, *args, odo, kf, accept)
                assert r1 == r2 == r3, (args, odo, kf, accept)
                seen.add(r1)
    assert seen == {(False, False), (True, False), (False, True)}
