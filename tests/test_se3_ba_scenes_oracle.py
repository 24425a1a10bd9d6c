"""CPU checks of the directly built SE(3) windows (tools/se3_window_synth.DIRECT_SCENES): the C++ oracle agrees with the numpy
restatement on a small version of each, the oracle's own spread on each is at least 10x below the GPU bounds, and the
scenes keep the shapes they exist for — the reduced system's widest envelope column, both off-diagonal odometry codes,
several RCM components (from the kernel's own plan, se3_ba_plan.h, through tests/native/se3_plan_profile.cpp), every
branch of Eigen's Quaterniond(Matrix3d) over the input rotations, the chunk boundaries and a window larger than the H100's 132 SMs x 256."""
from __future__ import annotations

import os
import subprocess

import numpy as np
import pytest

from oracle import pyse3ba
from oracle.se3_ba_numpy import Oracle
from tests.test_se3_ba_cpp_oracle import GPU_CHI2, GPU_EDGE, GPU_EST, decisions
from tools import se3_window_synth as S

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NAMES = sorted(S.DIRECT_SCENES)


def scene(name, small=False):
    f, iterations = S.DIRECT_SCENES[name]
    return f(small), S.direct_params(iterations)


@pytest.mark.parametrize("name", NAMES)
def test_cpp_oracle_agrees_with_the_numpy_restatement(name):
    w, prm = scene(name, small=True)
    c = pyse3ba.run(w, prm)
    o = Oracle(w, prm).optimize()
    N, O, L, E = w.sizes
    assert c["iterations"] == o["iterations"] and c["status"] == o["status"]
    assert (c["iterations"] > 0) == (S.n_free(w) > 0 or E > 0)
    assert decisions(c["stats"]) == [tuple(int(v) for v in s[4:7]) for s in o["stats"]]
    for s, t in zip(c["stats"], o["stats"]):
        assert abs(s["chi2_after"] - t[1]) <= 1e-8 * t[1] + 1e-12
    assert np.abs(c["poses"] - o["poses"]).max() < 2e-7 * max(1.0, np.abs(o["poses"]).max())
    if L:
        assert np.abs(c["points"] - o["points"]).max() < 2e-7 * max(1.0, np.abs(o["points"]).max())
    assert np.allclose(c["chi2"], o["chi2"], rtol=1e-5, atol=1e-5)
    assert np.array_equal(c["outlier"], o["outlier"])


def test_oracle_spread_is_far_below_the_gpu_bounds():
    worst = np.zeros(3)
    for name in NAMES:
        w, prm = scene(name)
        a = pyse3ba.run(w, prm)
        for kw in (dict(rev_sums=True), dict(rev_order=True)):
            b = pyse3ba.run(w, prm, **kw)
            assert decisions(a["stats"]) == decisions(b["stats"]), (name, kw)
            chi = max([abs(x["chi2_after"] - y["chi2_after"]) / y["chi2_after"] for x, y in zip(a["stats"], b["stats"])], default=0.0)
            est = max(np.abs(a["poses"] - b["poses"]).max(), np.abs(a["points"] - b["points"]).max(initial=0.0))
            edge = (np.abs(a["chi2"] - b["chi2"]) / np.maximum(1.0, np.abs(b["chi2"]))).max(initial=0.0)
            worst = np.maximum(worst, [chi, est, edge])
    assert worst[0] * 10 <= GPU_CHI2 and worst[1] * 10 <= GPU_EST and worst[2] * 10 <= GPU_EDGE, worst


@pytest.fixture(scope="module")
def profile(tmp_path_factory):
    exe = str(tmp_path_factory.mktemp("native") / "se3_plan_profile")
    res = subprocess.run(["g++", "-O2", "-std=c++14", "-Wall", "-Werror", os.path.join(ROOT, "tests", "native", "se3_plan_profile.cpp"),
                          "-o", exe], capture_output=True, text=True)
    assert res.returncode == 0, res.stderr

    def run(w):
        topo = [w.sizes, w.fixed, w.prior, np.stack([w.odo_from, w.odo_to], 1).ravel(), np.stack([w.edge_point, w.edge_kf], 1).ravel()]
        text = "\n".join(" ".join(str(int(v)) for v in t) for t in topo) + "\n"
        res = subprocess.run([exe], input=text, capture_output=True, text=True)
        assert res.returncode == 0, res.stderr
        nf, rows, off, off_t, comps = (int(v) for v in res.stdout.split())
        return dict(nf=nf, rows=rows, off=off, off_t=off_t, comps=comps)
    return run


def test_reduced_system_shapes(profile):
    """env_factor's rows-below loops make a second pass once a column holds 8 (x 36 > 256) and 43 (x 6 > 256) rows; the
    off-diagonal odometry gather reads H_ij as it is and transposed; RCM starts more than one component"""
    got = {name: profile(scene(name)[0]) for name in NAMES}
    for name, p in got.items():
        assert p["nf"] == S.n_free(scene(name)[0]), name
    assert got["dense"]["rows"] >= 43, got["dense"]
    assert got["loop_closure"]["rows"] >= 8 and got["large"]["rows"] >= 8
    assert any(p["off"] and p["off_t"] for p in got.values()), got
    assert got["yaw_near_pi"]["off"] and got["yaw_near_pi"]["off_t"], got["yaw_near_pi"]
    assert got["local_graph"]["comps"] > 1, got["local_graph"]


def quat_branch(R):
    """Eigen's Quaterniond(const Matrix3d&) (se2lam_b200/csrc/se3quat.h quat_from_R): the branch it takes, and the sign
    of w before normalisation"""
    t = R[0, 0] + R[1, 1] + R[2, 2]
    if t > 0:
        return "w", 1.0
    i = 0
    if R[1, 1] > R[0, 0]:
        i = 1
    if R[2, 2] > R[i, i]:
        i = 2
    j, k = (i + 1) % 3, (i + 2) % 3
    return "xyz"[i], R[k, j] - R[j, k]


def test_input_rotations_take_every_branch_of_quat_from_R():
    branches, flips = set(), 0
    for name in NAMES:
        w, _ = scene(name)
        for M in np.concatenate([w.Tcw, w.odo_measure]).reshape(-1, 4, 4):
            b, s = quat_branch(M[:3, :3].astype(np.float64))
            branches.add(b)
            flips += s < 0
    assert branches == set("wxyz") and flips > 0, (branches, flips)


def test_layouts():
    w, _ = scene("local_graph")
    n_ref = 3
    assert np.all(w.fixed[-n_ref:] == 1) and np.all(w.prior[-n_ref:] == 0) and np.all(w.prior[:-n_ref] == 1)
    assert w.fixed[0] == 0 and np.count_nonzero(w.fixed[:-n_ref]) == 1
    assert np.all(w.odo_to == w.odo_from + 1)
    assert len(w.odo_from) < len(w.Tcw) - n_ref - 1  # gaps
    assert len(np.setdiff1d(np.arange(len(w.xyz)), w.edge_point)) > 0  # edgeless points
    counts = np.bincount(w.edge_point, minlength=len(w.xyz))
    assert counts.max() == len(w.Tcw) - 1  # a point seen by every keyframe that has edges
    assert (-np.log2(w.inv_sigma2) / np.log2(1.44)).round().max() == S.MAX_OCTAVE
    w, _ = scene("only_ba_x")
    assert not w.prior.any() and len(w.odo_from) == 0
    active = np.zeros(len(w.Tcw), bool); active[w.edge_kf] = True
    assert np.any(~active & (w.fixed == 0))  # free keyframes left out of the graph
    for name, sizes in (("no_points", (0, 0)), ("edgeless", (None, 0)), ("only_ba_no_edges", (None, 0))):
        N, O, L, E = scene(name)[0].sizes
        assert (sizes[0] is None or L == sizes[0]) and E == sizes[1], name
    assert scene("one_kf")[0].sizes[0] == 1 and scene("one_kf_fixed")[0].sizes[0] == 1
    for n in (255, 256, 257):
        N, O, L, E = scene(f"items_{n}")[0].sizes
        assert E + N + O == n
        w = scene(f"points_{n}")[0]
        assert S.n_free(w) + w.sizes[2] == n
    assert scene("large")[0].sizes[3] > 132 * 256
