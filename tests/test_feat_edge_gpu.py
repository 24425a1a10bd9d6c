"""se2gpu_feat_edge against the CPU oracle (oracle/feat_edge_oracle.cpp): the two-keyframe BA's LM trajectory, the outlier
cut, and the marginalised constraint; batch invariance and the host / device entries byte for byte."""
import ctypes as C

import numpy as np
import pytest

from oracle import pyfeat
from se2lam_b200 import _capi, featgraph
from tools import featgraph_synth as S

pytestmark = pytest.mark.gpu

# The information matrix is badly conditioned by construction: H_marginal keeps the pair's six gauge directions at the
# 1e-6 the reference adds, its inverse amplifies them by 1e6, and the forward-difference Jacobian removes them only to the
# accuracy of a forward difference. The CPU oracle run with its per-point sums in ascending and in descending order
# differs by up to 8.1e-4 of max|info| over SCENES (the pure-rotation pair; most are at 1e-5 .. 1e-4, and pairs whose
# eigenvalues all sit on the 1e4 clamp at 1e-16); INFO_ORDER_SPREAD rounds that up. The GPU sums in trees and forms
# H12 H22^-1 H21 in another association; on an H100 it differs from the oracle by up to 2.6e-2 of max|info| (the
# pure-rotation pair again), and is held to fifty times the order spread. That gap is not the kernel's arithmetic: at one and
# the same state the two agree to 1e-6 (test_marginalisation_at_the_start_estimate), and the C++ oracle and its numpy
# restatement, whose LM runs end 1e-8 apart, differ by percent as well (DESIGN.md section 10). ILL_DEFINED names the scenes where the oracle does not even agree with itself: with 3 000 points
# H_marginal spans 1e7 .. 1e-6 and the two summation orders give information matrices that differ by 96 %, so for those the
# information is checked for its eigenvalue range only.
INFO_ORDER_SPREAD = 1e-3
INFO_RTOL = 50 * INFO_ORDER_SPREAD
ILL_DEFINED = {"m0_3000"}
# With both keyframes free and a 1 cm baseline the depth of every point is almost unobservable: LM creeps along that valley
# for all 30 iterations and the two implementations' chi2 separate to 7.5e-7 by the end (trials, accepted and terminate stay
# identical), so this scene is held to chi2 1e-5 and estimates 1e-3 instead.
WEAK_DEPTH = {"m1_baseline_1cm"}

SCENES = {
    # name: (mode, scene keyword arguments)
    "m0_10": (0, dict(seed=11, n_points=10)),
    "m0_50": (0, dict(seed=12, n_points=50)),
    "m0_300": (0, dict(seed=13, n_points=300)),
    "m0_3000": (0, dict(seed=14, n_points=3000)),
    "m1_10": (1, dict(seed=21, n_points=10, noise=0.3)),
    "m1_50": (1, dict(seed=22, n_points=50, noise=0.3)),
    "m1_300": (1, dict(seed=23, n_points=300, noise=0.3)),
    "m1_3000": (1, dict(seed=24, n_points=3000, noise=0.3)),
    "m0_huber": (0, dict(seed=31, n_points=60, outlier_share=0.15, outlier_size=(0.1, 0.3))),
    "m1_outliers": (1, dict(seed=32, n_points=60, noise=0.3, outlier_share=0.2, outlier_size=(0.2, 0.4))),
    "m0_yaw_pi": (0, dict(seed=41, n_points=50, start=(0.5, 0.2, np.pi - 0.01), motion=(0.3, 0.0, 0.03))),
    "m1_yaw_pi": (1, dict(seed=42, n_points=50, noise=0.3, start=(0.5, 0.2, -np.pi + 0.01), motion=(0.3, 0.0, -0.03))),
    "m0_pure_rotation": (0, dict(seed=51, n_points=50, motion=(0.0, 0.0, 0.15))),
    "m0_baseline_1cm": (0, dict(seed=52, n_points=50, motion=(0.01, 0.0, 0.0), pose_noise=(0.002, 0.001))),
    "m1_baseline_1cm": (1, dict(seed=53, n_points=50, noise=0.3, motion=(0.01, 0.0, 0.0), pose_noise=(0.002, 0.001))),
}


def make(name):
    mode, kw = SCENES[name]
    s = S.scene(**kw)
    return mode, s, featgraph.params(s["Tbc"]), pyfeat.params(Tbc=s["Tbc"])


def oracle(mode, s, oprm, **kw):
    return pyfeat.run(mode, s["Tcw0"], s["Tcw1"], s["xyz"], s["z0"], s["z1"], s["info0"], s["info1"], oprm, **kw)


def compared_iterations(st):
    """Iterations held to the LM bar: up to the first whose accepted step lowers chi2 by less than 1e-10 of it."""
    for k in range(len(st)):
        if st["chi2_before"][k] - st["chi2_after"][k] < 1e-10 * st["chi2_before"][k]:
            return k
    return len(st)


def check_parity(g, o, info_defined=True, est_atol=1e-5, chi2_rtol=1e-8):
    assert g["status"] == o["status"]
    if o["status"] == 1:
        return
    n = compared_iterations(o["stats"])
    assert g["iterations"] >= n and (n < o["iterations"] or g["iterations"] == o["iterations"])
    gs, os_ = g["stats"][:n], o["stats"][:n]
    for f in ("trials", "accepted", "terminate"):
        assert np.array_equal(gs[f], os_[f]), f
    # lambda follows rho = (chi2 drop) / scale through (2 rho - 1)^3: once a step lowers chi2 by 1e-5 of it, chi2 values
    # that agree to 1e-8 leave rho, and so lambda, agreeing to 1e-3 only
    np.testing.assert_allclose(gs["lambda"], os_["lambda"], rtol=1e-3)
    np.testing.assert_allclose(gs["chi2_before"], os_["chi2_before"], rtol=chi2_rtol)
    np.testing.assert_allclose(gs["chi2_after"], os_["chi2_after"], rtol=chi2_rtol)
    np.testing.assert_allclose(g["trace"][:n], o["trace"][:n], atol=est_atol)
    # the final state is compared for every scene; where LM stalled before its last iteration the bar is ten times wider
    if n < o["iterations"]:
        est_atol *= 10
    assert g["iterations"] == o["iterations"]
    assert np.array_equal(g["outlier"], o["outlier"])
    np.testing.assert_allclose(g["measure"], o["measure"], atol=max(1e-5, est_atol / 10))
    if True:
        np.testing.assert_allclose(g["poses"], o["poses"], atol=est_atol)
        np.testing.assert_allclose(g["points"], o["points"], atol=10 * est_atol)
        scale = np.abs(o["info"]).max()
        if info_defined:
            assert np.abs(g["info"].astype(np.float64) - o["info"]).max() <= INFO_RTOL * scale


@pytest.mark.parametrize("name", sorted(SCENES))
def test_parity_with_the_oracle(name):
    mode, s, prm, oprm = make(name)
    g = featgraph.CreateFeatEdge(s["Tcw0"], s["Tcw1"], s["xyz"], s["z0"], s["z1"], s["info0"], s["info1"], prm, matched=bool(mode),
                                 trace=True)
    o = oracle(mode, s, oprm)
    rev = oracle(mode, s, oprm, reverse=True)
    spread = np.abs(o["info"].astype(np.float64) - rev["info"]).max() / np.abs(o["info"]).max()
    assert (spread > INFO_ORDER_SPREAD) == (name in ILL_DEFINED), spread
    # with both keyframes free (mode 1) the pair's absolute position is held by the 1e-4 plane-motion prior alone, so the
    # estimates drift along that gauge at 1e-5 while lambda and chi2 agree to 1e-8; the relative pose (measure) does not
    if name in WEAK_DEPTH:
        check_parity(g, o, est_atol=1e-3, chi2_rtol=1e-5)
    else:
        check_parity(g, o, info_defined=name not in ILL_DEFINED, est_atol=1e-4 if mode else 1e-5)
    ev = np.linalg.eigvalsh(g["info"].astype(np.float64))
    assert ev.min() > 0.9e-6 and ev.max() < 1.1e4


COARSE = {   # a coarser sensor (Omega / 1000): the information stays below the 1e4 clamp
    "m0_50_coarse": (0, dict(seed=12, n_points=50, info_scale=1e-3)),
    "m1_50_coarse": (1, dict(seed=22, n_points=50, noise=0.3, info_scale=1e-3)),
    "m1_outliers_coarse": (1, dict(seed=32, n_points=60, noise=0.3, outlier_share=0.2, outlier_size=(6.0, 12.0), info_scale=1e-3)),
}


@pytest.mark.parametrize("name", sorted(SCENES) + sorted(COARSE))
def test_marginalisation_at_the_start_estimate(name):
    """With no LM iteration both sides marginalise at the identical state (the float inputs), which takes LM's drift out of
    the comparison: outlier bytes equal, relative pose to 1e-6, information to 1e-4 of its Frobenius norm where the oracle's
    own summation-order spread is below 1e-5 (elsewhere to ten times that spread)."""
    mode, kw = (SCENES | COARSE)[name]
    s = S.scene(**kw)
    prm = featgraph.params(s["Tbc"], iterations=(0, 0))
    oprm = pyfeat.params(Tbc=s["Tbc"], iterations=(0, 0))
    g = featgraph.CreateFeatEdge(s["Tcw0"], s["Tcw1"], s["xyz"], s["z0"], s["z1"], s["info0"], s["info1"], prm, matched=bool(mode))
    o = oracle(mode, s, oprm)
    rev = oracle(mode, s, oprm, reverse=True)
    assert g["status"] == 0 and g["iterations"] == 0
    assert np.array_equal(g["outlier"], o["outlier"])
    np.testing.assert_allclose(g["measure"], o["measure"], atol=1e-6)
    nrm = np.linalg.norm(o["info"].astype(np.float64))
    spread = np.linalg.norm(o["info"].astype(np.float64) - rev["info"]) / nrm
    assert np.linalg.norm(g["info"].astype(np.float64) - o["info"]) <= max(1e-4, 10 * spread) * nrm, spread


def test_outlier_bytes_match_the_oracle_and_the_planted_set():
    mode, s, prm, oprm = make("m1_outliers")
    g = featgraph.CreateFeatEdge(s["Tcw0"], s["Tcw1"], s["xyz"], s["z0"], s["z1"], s["info0"], s["info1"], prm, matched=True)
    o = oracle(1, s, oprm)
    assert np.array_equal(g["outlier"], o["outlier"])
    assert np.array_equal(g["outlier"] != 0, s["planted"])


def _batch():
    pairs = []
    rng = np.random.default_rng(7)
    for b in range(64):
        n = int(rng.choice([2, 9, 10, 17, 50, 130, 257, 300, 700]))
        pairs.append(S.scene(100 + b, n, noise=0.3, outlier_share=0.1 if b % 3 == 0 else 0.0, outlier_size=(0.15, 0.3)))
    return pairs


@pytest.mark.parametrize("mode", [0, 1])
def test_a_batch_is_its_single_pair_calls_byte_for_byte(mode):
    pairs = _batch()
    prm = featgraph.params(pairs[0]["Tbc"])
    a = featgraph.UpdateFeatGraph(pairs, prm, mode=mode)
    b = featgraph.UpdateFeatGraph(pairs, prm, mode=mode)
    few = 0
    for p, ra, rb in zip(pairs, a, b):
        one = featgraph.UpdateFeatGraph([p], prm, mode=mode)[0]
        assert ra["status"] == one["status"] == rb["status"]
        if ra["status"] == featgraph.TOO_FEW:
            few += 1
            assert ra["measure"] is None and ra["iterations"] == 0
            continue
        for k in ("measure", "info", "outlier", "poses", "points", "stats"):
            assert ra[k].tobytes() == one[k].tobytes() == rb[k].tobytes(), k
    assert few >= 1


def test_too_few_leaves_the_outputs_alone():
    s = S.scene(3, 9)
    prm = featgraph.params(s["Tbc"])
    L = _capi.lib()
    for mode, n in ((0, 9), (1, 2)):
        measure = np.full(16, 7.0, np.float32); info = np.full(36, 7.0, np.float32)
        status = np.zeros(1, np.int32); pp = np.array([0, n], np.int32)
        rc = L.se2gpu_feat_edge(1, mode, _capi.ptr(s["Tcw0"]), _capi.ptr(s["Tcw1"]), _capi.ptr(pp), _capi.ptr(s["xyz"]),
                                _capi.ptr(s["z0"]), _capi.ptr(s["z1"]), _capi.ptr(s["info0"]), _capi.ptr(s["info1"]),
                                C.addressof(prm), _capi.ptr(measure), _capi.ptr(info), _capi.ptr(status), None, None, None, None,
                                None, 0)
        assert rc == 0 and status[0] == featgraph.TOO_FEW
        assert np.all(measure == 7.0) and np.all(info == 7.0)


def test_malformed_input_is_rejected_before_any_launch():
    s = S.scene(3, 12)
    prm = featgraph.params(s["Tbc"])
    L = _capi.lib()
    measure = np.zeros(16, np.float32); info = np.zeros(36, np.float32)

    def call(B, mode, pp, p=prm):
        pp = np.asarray(pp, np.int32)
        return L.se2gpu_feat_edge(B, mode, _capi.ptr(s["Tcw0"]), _capi.ptr(s["Tcw1"]), _capi.ptr(pp), _capi.ptr(s["xyz"]),
                                  _capi.ptr(s["z0"]), _capi.ptr(s["z1"]), _capi.ptr(s["info0"]), _capi.ptr(s["info1"]),
                                  C.addressof(p) if p is not None else None, _capi.ptr(measure), _capi.ptr(info), None, None, None,
                                  None, None, None, 0)

    before = L.se2gpu_launch_count()
    assert call(-1, 0, [0, 12]) == -3
    assert call(1, 2, [0, 12]) == -3
    assert call(1, 0, [1, 12]) == -3
    assert call(2, 0, [0, 12, 5]) == -3
    assert call(1, 0, [0, 12], None) == -3
    bad = featgraph.params(s["Tbc"], iterations=(-1, 30))
    assert call(1, 0, [0, 12], bad) == -3
    assert L.se2gpu_launch_count() == before
    assert "point_ptr" in _capi.last_error() or "iterations" in _capi.last_error()


def test_device_entry_takes_xyz_info_device_output_and_equals_the_host_entry():
    import torch
    mode, s, prm, _ = make("m0_50")
    L = _capi.lib()
    dev = torch.device("cuda:0")
    P = len(s["xyz"])
    # Track::calcSE3toXYZInfo on the device, from keyframe 0's measurement and the two poses
    Tcw = torch.tensor(np.stack([s["Tcw0"], s["Tcw1"]]).reshape(2, 16), device=dev)
    z0 = torch.tensor(s["z0"], device=dev); z1 = torch.tensor(s["z1"], device=dev)
    i0 = torch.zeros(P, dtype=torch.int32, device=dev); i1 = torch.ones(P, dtype=torch.int32, device=dev)
    info0 = torch.zeros(P * 9, dtype=torch.float64, device=dev); info1 = torch.zeros(P * 9, dtype=torch.float64, device=dev)
    p = _capi.ptr
    assert L.se2gpu_xyz_info_device(P, p(z0), p(i0), p(i1), p(Tcw), S.FX, p(info0), p(info1), None) == 0
    xyz = torch.tensor(s["xyz"], device=dev)
    pp = torch.tensor([0, P], dtype=torch.int32, device=dev)
    T0 = Tcw[0].clone(); T1 = Tcw[1].clone()
    measure = torch.zeros(16, dtype=torch.float32, device=dev); info = torch.zeros(36, dtype=torch.float32, device=dev)
    status = torch.zeros(1, dtype=torch.int32, device=dev); iters = torch.zeros(1, dtype=torch.int32, device=dev)
    points = torch.zeros(P * 3, dtype=torch.float64, device=dev); work = torch.zeros(P * 3, dtype=torch.float64, device=dev)
    poses = torch.zeros(14, dtype=torch.float64, device=dev)
    rc = L.se2gpu_feat_edge_device(1, mode, p(T0), p(T1), p(pp), p(xyz), p(z0), p(z1), p(info0), p(info1), C.addressof(prm), p(measure),
                                   p(info), p(status), p(iters), None, None, p(poses), p(points), p(work), None)
    assert rc == 0, _capi.last_error()
    torch.cuda.synchronize()
    h = featgraph.CreateFeatEdge(s["Tcw0"], s["Tcw1"], s["xyz"], s["z0"], s["z1"], info0.cpu().numpy(), info1.cpu().numpy(), prm)
    assert int(status[0]) == h["status"] == 0 and int(iters[0]) == h["iterations"]
    assert measure.cpu().numpy().tobytes() == h["measure"].tobytes()
    assert info.cpu().numpy().tobytes() == h["info"].tobytes()
    assert poses.cpu().numpy().tobytes() == h["poses"].tobytes()
    assert points.cpu().numpy().tobytes() == h["points"].tobytes()
    # and the constraint is the one the oracle derives from the same device-made information
    o = pyfeat.run(mode, s["Tcw0"], s["Tcw1"], s["xyz"], s["z0"], s["z1"], info0.cpu().numpy(), info1.cpu().numpy(),
                   pyfeat.params(Tbc=s["Tbc"]))
    np.testing.assert_allclose(h["measure"], o["measure"], atol=1e-5)
