"""CPU checks of the sequential C++ oracle of the SE(3)-XYZ window BA (oracle/se3_ba_oracle.cpp): it agrees with the
independent numpy restatement (oracle/se3_ba_numpy.py) in both modes, and its own spread — every edge sum reversed, or the
free keyframes eliminated in reversed order — is at least 10x below the bounds tests/test_se3_ba_gpu.py holds the GPU to."""
from __future__ import annotations

import numpy as np
import pytest

from oracle import pyse3ba
from oracle.se3_ba_numpy import Oracle
from tools import se3_window_synth as S

# tests/test_se3_ba_gpu.py: chi2 relative, estimates, per-edge chi2 (relative or absolute)
GPU_CHI2, GPU_EST, GPU_EDGE = 1e-9, 1e-7, 1e-6


def decisions(stats):
    return [(int(s["trials"]), int(s["accepted"]), int(s["terminate"])) for s in stats]


@pytest.mark.parametrize("kw", [{}, dict(with_prior=False, odometry=False), dict(n_ref=2), dict(outlier_frac=0.25)],
                         ids=["loadLocalGraph", "loadLocalGraphOnlyBa", "reference_kfs", "gross_outliers"])
def test_cpp_oracle_agrees_with_the_numpy_restatement(kw):
    prob, w = S.window(6, 200, seed=3, **kw)
    prm = S.window_params(prob)
    c = pyse3ba.run(w, prm)
    o = Oracle(w, prm).optimize()
    assert c["iterations"] == o["iterations"] > 0 and c["status"] == o["status"]
    assert decisions(c["stats"]) == [tuple(int(v) for v in s[4:7]) for s in o["stats"]]
    for s, t in zip(c["stats"], o["stats"]):
        assert abs(s["chi2_after"] - t[1]) <= 1e-8 * t[1]
    # the two routes through the float rotations and the 1e6 prior informations differ at this level
    assert np.abs(c["poses"] - o["poses"]).max() < 2e-7 * max(1.0, np.abs(o["poses"]).max())
    assert np.abs(c["points"] - o["points"]).max() < 2e-7 * max(1.0, np.abs(o["points"]).max())
    assert np.allclose(c["chi2"], o["chi2"], rtol=1e-5, atol=1e-5)
    assert np.array_equal(c["outlier"], o["outlier"])


def test_oracle_spread_is_far_below_the_gpu_bounds():
    worst = np.zeros(3)
    for name, (f, iterations) in S.SCENES.items():
        prob, w = f()
        prm = S.window_params(prob, iterations=iterations)
        a = pyse3ba.run(w, prm)
        for kw in (dict(rev_sums=True), dict(rev_order=True)):
            b = pyse3ba.run(w, prm, **kw)
            assert decisions(a["stats"]) == decisions(b["stats"]), (name, kw)
            chi = max(abs(x["chi2_after"] - y["chi2_after"]) / y["chi2_after"] for x, y in zip(a["stats"], b["stats"]))
            est = max(np.abs(a["poses"] - b["poses"]).max(), np.abs(a["points"] - b["points"]).max())
            edge = (np.abs(a["chi2"] - b["chi2"]) / np.maximum(1.0, np.abs(b["chi2"]))).max()
            worst = np.maximum(worst, [chi, est, edge])
    assert worst[0] * 10 <= GPU_CHI2 and worst[1] * 10 <= GPU_EST and worst[2] * 10 <= GPU_EDGE, worst
