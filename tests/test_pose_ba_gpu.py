"""GPU parity of the pose-only SE(3) BA (Localizer::DoLocalBA, se2gpu_pose_ba*) against the CPU oracle.

Bar (BASELINE.md section 4): identical trials / accepted / terminate sequences, lambda to 1e-6, chi2 to 1e-8 and the pose after
every iteration within 1e-5 relative. Once LM has converged to the last bits, its accept / reject decisions hinge on chi2
differences at rounding level (an accepted step that lowers chi2 by less than 1e-10 of it), where two correct
implementations that sum in different orders part ways. The sequences are therefore compared over the decisive iterations
before that point; past them the final estimates must still agree within the bar.
"""
import math

import numpy as np
import pytest

from oracle import pypose
from se2lam_b200 import pose as pba
from se2lam_b200._capi import KP_DTYPE
from tools import pose_synth as ps

pytestmark = pytest.mark.gpu

DELTA = math.sqrt(5.991)
ITERS = 30


def prm(iterations=ITERS):
    return pba.params(ps.FX, ps.CX, ps.CY, ps.Tbc_f32(), DELTA, iterations=iterations)


def oracle(p, iterations=ITERS):
    return pypose.run(p["Tcw"], p["xyz"], p["uv"], p["info"], ps.FX, ps.CX, ps.CY, ps.Tbc_f32(), DELTA, iterations=iterations)


def decisive_prefix(st):
    """Leading iterations that accepted a step lowering chi2 by more than 1e-10 of it."""
    for k in range(len(st)):
        if not (st["accepted"][k] and st["chi2_before"][k] - st["chi2_after"][k] > 1e-10 * st["chi2_before"][k]):
            return k
    return len(st)


def check_parity(p, g, b=0, min_decisive=3):
    o = oracle(p)
    P = decisive_prefix(o["stats"])
    st_o, st_g = o["stats"], g["stats"][b][:g["iterations"][b]]
    if P == o["iterations"]:
        assert g["iterations"][b] == o["iterations"]
    assert P >= min_decisive, "test input converges too fast to exercise LM"
    for f in ("trials", "accepted", "terminate"):
        np.testing.assert_array_equal(st_g[f][:P], st_o[f][:P], err_msg=f)
    np.testing.assert_allclose(st_g["lambda"][:P], st_o["lambda"][:P], rtol=1e-6)
    np.testing.assert_allclose(st_g["chi2_before"][:P], st_o["chi2_before"][:P], rtol=1e-8)
    np.testing.assert_allclose(st_g["chi2_after"][:P], st_o["chi2_after"][:P], rtol=1e-8)
    for k in range(P):
        ref = o["trace"][k]
        assert np.abs(g["trace"][b][k] - ref).max() <= 1e-5 * max(1.0, np.abs(ref).max()), k
    # the results: double pose and its float cast (toCvMat)
    assert np.abs(g["pose"][b] - o["pose"]).max() <= 1e-5 * max(1.0, np.abs(o["pose"]).max())
    Tg = g["Tcw"][b]
    assert np.abs(Tg - o["Tcw"]).max() <= 1e-5 * max(1.0, np.abs(o["Tcw"]).max())
    assert g["status"][b] == o["status"] == pba.OK
    return o


CASES = {
    "E1": dict(E=1, seed=11, start_rot=0.002, start_trans=0.01),
    "E7": dict(E=7, seed=12),
    "E31": dict(E=31, seed=13),
    "E300": dict(E=300, seed=14),
    "E1000": dict(E=1000, seed=15),
    # either side of a CTA's 256 edges and of the 1536 edges the batched kernel stages in shared memory (kStageMax)
    "E255": dict(E=255, seed=22),
    "E256": dict(E=256, seed=23),
    "E257": dict(E=257, seed=24),
    "E1536": dict(E=1536, seed=27),
    "E1537": dict(E=1537, seed=26),
    "E5000_streamed": dict(E=5000, seed=16),
    "yaw_near_pi": dict(E=300, seed=17, yaw=math.pi - 1e-4),
    "yaw_near_minus_pi": dict(E=300, seed=18, yaw=-math.pi + 1e-4),
    "zero_rotation": dict(E=300, seed=19, zero_rotation=True),
    "huber_outliers": dict(E=300, seed=20, outliers=0.2),
    "tilted_start": dict(E=300, seed=21, tilt=0.05),
}


@pytest.mark.parametrize("case", sorted(CASES))
def test_problem_matches_oracle(case):
    p = ps.make_problem(**CASES[case])
    g = pba.poseOnlyBA(p["Tcw"][None], [0, len(p["xyz"])], p["xyz"], p["uv"], p["info"], prm(), trace=True)
    o = check_parity(p, g)
    if case == "huber_outliers":
        assert (o["stats"]["chi2_before"][0] > DELTA ** 2)
    if case == "zero_rotation":
        assert np.array_equal(p["Tcw"][:3, :3], np.eye(3, dtype=np.float32))


def test_huber_branch_is_active():
    p = ps.make_problem(**CASES["huber_outliers"])
    T = p["Tcw"].astype(np.float64)
    pc = p["xyz"] @ T[:3, :3].T + T[:3, 3]
    e = p["uv"] - (pc[:, :2] / pc[:, 2:] * ps.FX + np.array([ps.CX, ps.CY]))
    assert ((e ** 2).sum(1) * p["info"] > DELTA ** 2).sum() >= 0.15 * len(e)


def test_no_edges_leaves_the_pose():
    p = ps.make_problem(E=5, seed=3)
    T0 = np.stack([p["Tcw"], p["Tcw"]])
    g = pba.poseOnlyBA(T0, [0, 0, 5], p["xyz"], p["uv"], p["info"], prm())
    assert g["status"][0] == pba.NO_EDGES and g["iterations"][0] == 0
    assert g["Tcw"][0].tobytes() == T0[0].tobytes()
    assert g["status"][1] == pba.OK and g["iterations"][1] > 0
    assert (g["stats"][0]["trials"] == 0).all()


def _mixed(n=64, seed=100):
    rng = np.random.default_rng(seed)
    sizes = [0, 1, 7, 31, 300, 1000, 2000, 5000] + list(rng.integers(1, 1500, n - 8))
    return [ps.make_problem(E=int(E), seed=seed + k, outliers=0.1 if k % 3 == 0 else 0.0,
                            start_rot=0.002 if E < 5 else 0.01, start_trans=0.01 if E < 5 else 0.05) for k, E in enumerate(sizes)]


def test_batch_equals_single_calls_bitwise_and_is_reproducible():
    probs = _mixed()
    T, ptr, x, u, w = ps.batch(probs)
    g1 = pba.poseOnlyBA(T, ptr, x, u, w, prm(), trace=True)
    g2 = pba.poseOnlyBA(T, ptr, x, u, w, prm(), trace=True)
    for k in ("Tcw", "pose", "iterations", "status", "stats", "trace"):
        assert g1[k].tobytes() == g2[k].tobytes(), k
    for b, p in enumerate(probs):
        s = pba.poseOnlyBA(p["Tcw"][None], [0, len(p["xyz"])], p["xyz"], p["uv"], p["info"], prm(), trace=True)
        for k in ("Tcw", "pose", "iterations", "status", "stats", "trace"):
            assert s[k][0].tobytes() == g1[k][b].tobytes(), (b, k)
    # and every problem of the batch holds the oracle bar
    for b in (1, 2, 3, 4, 5, 6, 7, 20):
        check_parity(probs[b], g1, b, min_decisive=1)


def test_device_entry_equals_host_entry():
    import torch
    probs = _mixed(16, seed=300)
    T, ptr, x, u, w = ps.batch(probs)
    h = pba.poseOnlyBA(T, ptr, x, u, w, prm())
    dev = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()
    dT, dp, dx, du, dw = dev(T), dev(ptr), dev(x), dev(u), dev(w)
    B = len(T)
    dst = torch.zeros(B * ITERS * 48, dtype=torch.uint8, device="cuda")
    dit = torch.zeros(B, dtype=torch.int32, device="cuda"); dss = torch.zeros(B, dtype=torch.int32, device="cuda")
    dpose = torch.zeros(B * 7, dtype=torch.float64, device="cuda")
    pba.poseOnlyBADevice(B, dT, dp, dx, du, dw, prm(), dst, dit, dss, dpose, torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    assert dT.cpu().numpy().tobytes() == h["Tcw"].reshape(B, 16).tobytes()
    assert dpose.cpu().numpy().tobytes() == h["pose"].tobytes()
    assert np.array_equal(dit.cpu().numpy(), h["iterations"]) and np.array_equal(dss.cpu().numpy(), h["status"])
    st = dst.cpu().numpy().view(h["stats"].dtype).reshape(B, ITERS)
    for b in range(B):
        n = h["iterations"][b]
        assert st[b, :n].tobytes() == h["stats"][b, :n].tobytes()


def _localizer_case(seed, n_mp=400, n_kf=600):
    """Map points of a pose problem, keyframe keypoints where they project (plus distractors), and a match table with
    unmatched rows, repeated map points and map points whose use flag is cleared."""
    rng = np.random.default_rng(seed)
    p = ps.make_problem(E=n_mp, seed=seed)
    kp = np.zeros(n_kf, KP_DTYPE)
    kp["x"] = rng.uniform(0, 640, n_kf); kp["y"] = rng.uniform(0, 480, n_kf)
    kp["octave"] = rng.integers(0, 8, n_kf); kp["class_id"] = -1
    slots = rng.permutation(n_kf)[:n_mp]
    kp["x"][slots] = p["uv"][:, 0]; kp["y"][slots] = p["uv"][:, 1]
    m = np.full(n_kf, -1, np.int32)
    m[slots] = np.arange(n_mp)
    m[slots[: n_mp // 3]] = -1                                   # unmatched
    dup = rng.choice(n_kf, 20, replace=False)
    m[dup] = rng.integers(0, n_mp, 20)                           # map points observed twice
    use = (rng.random(n_mp) > 0.1).astype(np.uint8)
    return p, kp, m, use


@pytest.mark.parametrize("seed", [1, 2])
def test_localizer_entry_matches_host_flattening(seed):
    p, kp, m, use = _localizer_case(40 + seed)
    xyz, uv, w = pba.localizer_edges(kp, m, p["xyz"], use, ps.INV_SIGMA2)
    assert (w == ps.INV_SIGMA2[kp["octave"][0]]).all()
    r = pba.localizerBA(kp, m, p["xyz"], use, ps.INV_SIGMA2, p["Tcw"], prm(), min_edges=30)
    assert r["n_edges"] == len(xyz) > 30
    h = pba.poseOnlyBA(p["Tcw"][None], [0, len(xyz)], xyz, uv, w, prm())
    assert r["Tcw"].tobytes() == h["Tcw"][0].tobytes() and r["pose"].tobytes() == h["pose"][0].tobytes()
    assert r["iterations"] == h["iterations"][0] and r["stats"].tobytes() == h["stats"][0][:r["iterations"]].tobytes()
    o = pypose.run(p["Tcw"], xyz, uv, w, ps.FX, ps.CX, ps.CY, ps.Tbc_f32(), DELTA, iterations=ITERS)
    assert np.abs(r["Tcw"] - o["Tcw"]).max() <= 1e-5 * max(1.0, np.abs(o["Tcw"]).max())
    # the gate: no more edges than min_edges leaves the pose and reports GATED
    g = pba.localizerBA(kp, m, p["xyz"], use, ps.INV_SIGMA2, p["Tcw"], prm(), min_edges=len(xyz))
    assert g["status"] == pba.GATED and g["n_edges"] == len(xyz) and g["Tcw"].tobytes() == p["Tcw"].tobytes()


@pytest.mark.parametrize("seed", [3, 4])
def test_localizer_entry_across_keypoint_rounds(seed):
    """~3 000 keypoints, so the edge scan walks several rounds of 1 024 keypoints. A map point matched by two keypoints
    takes the higher index's position: 1 024 apart (one thread, two rounds), 1 023 apart (neighbouring threads of two
    warps, two rounds, no barrier between them) and 600 apart (two warps of one round). Match indices >= n_mp are
    ignored, and kp[0] on the top octave sets every edge's information (the reference's octave quirk). Checked against
    the host flattening and the oracle."""
    p, kp, m, use = _localizer_case(50 + seed, n_mp=400, n_kf=3000)
    n_mp = len(use)
    pairs = {int(j): (lo, hi) for j, (lo, hi) in zip(np.flatnonzero(use)[seed:seed + 3],
                                                    [(700 + seed, 1724 + seed), (1600, 2623), (1030, 1630)])}
    for j, (lo, hi) in pairs.items():
        m[m == j] = -1
        m[[lo, hi]] = j
        kp["x"][lo], kp["y"][lo] = p["uv"][j] + np.float32(40)
        kp["x"][hi], kp["y"][hi] = p["uv"][j] + np.float32(0.5)
    m[[5, 1500, 2999]] = [n_mp, n_mp + 7, 2 ** 30]
    kp["octave"][0] = len(ps.INV_SIGMA2) - 1
    xyz, uv, w = pba.localizer_edges(kp, m, p["xyz"], use, ps.INV_SIGMA2)
    js = np.flatnonzero(use != 0)
    for j, (lo, hi) in pairs.items():
        e = int(np.searchsorted(js[np.isin(js, m)], j))
        assert uv[e].tolist() == [kp["x"][hi], kp["y"][hi]], (lo, hi)
    assert (w == ps.INV_SIGMA2[-1]).all() and len(xyz) > 30
    r = pba.localizerBA(kp, m, p["xyz"], use, ps.INV_SIGMA2, p["Tcw"], prm(), min_edges=30)
    assert r["n_edges"] == len(xyz)
    h = pba.poseOnlyBA(p["Tcw"][None], [0, len(xyz)], xyz, uv, w, prm())
    assert r["Tcw"].tobytes() == h["Tcw"][0].tobytes() and r["pose"].tobytes() == h["pose"][0].tobytes()
    o = pypose.run(p["Tcw"], xyz, uv, w, ps.FX, ps.CX, ps.CY, ps.Tbc_f32(), DELTA, iterations=ITERS)
    assert np.abs(r["Tcw"] - o["Tcw"]).max() <= 1e-5 * max(1.0, np.abs(o["Tcw"]).max())
    assert r["status"] == o["status"]


def test_device_chain_from_match_by_projection():
    """se2gpu_match_by_projection_device -> se2gpu_localizer_ba_device without leaving the device, against the host
    flattening of the same matches into the oracle."""
    import torch
    from se2lam_b200.matcher import FrameView, ORBmatcher
    rng = np.random.default_rng(7)
    n_mp, n_kf = 300, 500
    p = ps.make_problem(E=n_mp, seed=77)
    kp = np.zeros(n_kf, KP_DTYPE)
    kp["x"] = rng.uniform(0, 640, n_kf); kp["y"] = rng.uniform(0, 480, n_kf)
    kp["octave"] = rng.integers(0, 4, n_kf); kp["class_id"] = -1; kp["size"] = 31
    slots = rng.permutation(n_kf)[:n_mp]
    kp["x"][slots] = p["uv"][:, 0]; kp["y"][slots] = p["uv"][:, 1]
    desc = rng.integers(0, 256, (n_kf, 32), dtype=np.uint8)
    mp_desc = desc[slots].copy()
    mp_uv = np.stack([kp["x"][slots], kp["y"][slots]], 1).astype(np.float32)
    mp_oct = kp["octave"][slots].astype(np.int32)
    mp_valid = (rng.random(n_mp) > 0.05).astype(np.uint8)
    use = (rng.random(n_mp) > 0.1).astype(np.uint8)
    dev = lambda a: torch.from_numpy(np.ascontiguousarray(a).view(np.uint8) if np.asarray(a).dtype == KP_DTYPE else np.ascontiguousarray(a)).cuda()
    d_kp, d_desc = dev(kp), dev(desc)
    d_m = torch.full((n_kf,), 7, dtype=torch.int32, device="cuda"); d_nm = torch.zeros(1, dtype=torch.int32, device="cuda")
    mt = ORBmatcher(0.9, max_queries=n_mp, max_db=n_kf)
    s = torch.cuda.current_stream().cuda_stream
    mt.MatchByProjectionDevice(d_kp, d_desc, n_kf, dev(np.zeros(n_kf, np.uint8)), dev(mp_valid), dev(mp_uv), n_mp, dev(mp_oct), dev(mp_desc),
                               FrameView(None, None).grid(), 15, 2, d_m, d_nm, stream=s)
    d_T = dev(p["Tcw"].reshape(16).copy()); d_ne = torch.zeros(1, dtype=torch.int32, device="cuda")
    d_it = torch.zeros(1, dtype=torch.int32, device="cuda"); d_st = torch.full((1,), 9, dtype=torch.int32, device="cuda")
    loc = pba.Localizer(n_mp)
    loc.localizerBA(d_kp, n_kf, d_m, n_mp, dev(p["xyz"]), dev(use), dev(ps.INV_SIGMA2), 8, d_T, prm(), 30, d_n_edges=d_ne, d_iterations=d_it,
                    d_status=d_st, stream=s)
    torch.cuda.synchronize()
    m = d_m.cpu().numpy()
    assert int(d_nm.item()) > 0.8 * n_mp
    xyz, uv, w = pba.localizer_edges(kp, m, p["xyz"], use, ps.INV_SIGMA2)
    assert int(d_ne.item()) == len(xyz) > 30 and int(d_st.item()) == pba.OK
    o = pypose.run(p["Tcw"], xyz, uv, w, ps.FX, ps.CX, ps.CY, ps.Tbc_f32(), DELTA, iterations=ITERS)
    Tg = d_T.cpu().numpy().reshape(4, 4)
    assert np.abs(Tg - o["Tcw"]).max() <= 1e-5 * max(1.0, np.abs(o["Tcw"]).max())
    h = pba.poseOnlyBA(p["Tcw"][None], [0, len(xyz)], xyz, uv, w, prm())
    assert Tg.tobytes() == h["Tcw"][0].tobytes() and int(d_it.item()) == h["iterations"][0]
