"""Track::removeOutliers on the GPU against the oracle, bit for bit (test_fundam_gpu._check: nInlier, matches12, the bytes of
F and the hypothesis count), on the scene families of tests/fundam_scenes.py: zero motion, keypoint lattices up to the
8192-pair capacity and getSubset give-ups. Also the device entry's documented edges (NULL counts, counts outside
[0, cap], match indices past the frame-2 count, a side stream) and the device chain extract -> MatchByWindow ->
removeOutliers -> doTriangulate of INTEGRATION.md section 1, batched over eight frame pairs."""
import ctypes as C

import numpy as np
import pytest

from oracle import pyfundam, pygeom
from tests import fundam_scenes as fs
from tests.test_fundam_gpu import _check

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")
if not torch.cuda.is_available():
    pytest.skip("no CUDA device", allow_module_level=True)

from se2lam_b200 import _capi  # noqa: E402
from se2lam_b200._capi import KP_DTYPE, ptr  # noqa: E402
from se2lam_b200.geometry import removeOutliers  # noqa: E402
from tests.test_geom_gpu import same  # noqa: E402  (NaN positions compare as one canonical NaN)

SENTINEL = 77


@pytest.fixture(scope="module")
def cases():
    out = []
    for s in fs.all_scenes():
        kp1, kp2, m = s.keypoints(KP_DTYPE)
        out.append((s, kp1, kp2, m, pyfundam.remove_outliers(kp1, kp2, m)))
    return out


def _small(cases, k, lo=8, hi=400):
    return [c for c in cases if lo <= c[0].n <= hi][:k]


def _batch(sel):
    return removeOutliers([c[1] for c in sel], [c[2] for c in sel], [c[3] for c in sel], return_details=True)


def test_batches_of_64_with_mixed_n(cases):
    order = np.random.default_rng(5).permutation(len(cases))
    for a in range(0, len(order), 64):
        chunk = [cases[i] for i in order[a:a + 64]]
        for c, r in zip(chunk, _batch(chunk)):
            _check(r, c[4], repr(c[0]))


def test_pair_by_pair(cases):
    for c in cases:
        _check(removeOutliers(c[1], c[2], c[3], return_details=True), c[4], repr(c[0]))


def test_full_capacity_every_keypoint_matched(cases):
    full = [c for c in cases if len(c[1]) == fs.MAX_PAIRS and (c[3] >= 0).all()]
    assert {c[0].family for c in full} == {"static", "lattice"}
    for c, r in zip(full, _batch(full)):
        _check(r, c[4], repr(c[0]))


def test_capacity_set_by_one_sparse_pair(cases):
    """One pair of 8192 keypoints with 20 matched sets cap1 for 63 small ones."""
    kp1, kp2, m = fs.sparse_capacity_pair()
    want = pyfundam.remove_outliers(kp1, kp2, m)
    _check(removeOutliers(kp1, kp2, m, return_details=True), want, "sparse alone")
    # 63 small pairs: the small scenes, each with a few interleavings of unmatched keypoints
    small = [c[0] for c in _small(cases, 64)]
    sel = [(s, *s.keypoints(KP_DTYPE, variant=v)) for v in range(4) for s in small][:63]
    assert len(sel) == 63
    K1 = [c[1] for c in sel]; K2 = [c[2] for c in sel]; M = [c[3] for c in sel]
    res = removeOutliers(K1[:31] + [kp1] + K1[31:], K2[:31] + [kp2] + K2[31:], M[:31] + [m] + M[31:], return_details=True)
    assert len(res) == 64
    _check(res[31], want, "sparse in a batch")
    for c, r in zip(sel, res[:31] + res[32:]):
        _check(r, pyfundam.remove_outliers(*c[1:]), repr(c[0]))


# ------------------------------------------------------------------------------------------ device entry
def _tensor(a):
    return torch.from_numpy(np.ascontiguousarray(a).view(np.uint8) if a.dtype == KP_DTYPE else np.ascontiguousarray(a)).cuda()


def _pack(pairs, cap1, cap2):
    """pairs of (kp1, kp2, matches12) into [B, cap] arrays; matches12 past each pair's kp1 is SENTINEL."""
    B = len(pairs)
    k1 = np.zeros((B, cap1), KP_DTYPE); k2 = np.zeros((B, cap2), KP_DTYPE); m = np.full((B, cap1), SENTINEL, np.int32)
    for b, (a1, a2, mm) in enumerate(pairs):
        k1[b, :len(a1)] = a1; k2[b, :len(a2)] = a2; m[b, :len(mm)] = mm
    return k1, k2, m


def _device(k1, n1, cap1, k2, n2, cap2, m, stream=None):
    """se2gpu_remove_outliers_device on [B, cap] host arrays; n1 / n2 None pass NULL. Returns (nin, m, F, iters) per pair
    over the whole capacity row."""
    B = len(k1)
    dk1, dk2, dm = _tensor(k1), _tensor(k2), _tensor(m)
    dn1 = None if n1 is None else _tensor(np.asarray(n1, np.int32))
    dn2 = None if n2 is None else _tensor(np.asarray(n2, np.int32))
    dnin = torch.full((B,), -9, dtype=torch.int32, device="cuda")
    dF = torch.full((B * 9,), 5.0, dtype=torch.float64, device="cuda")
    dit = torch.full((B,), -9, dtype=torch.int32, device="cuda")
    s = stream if stream is not None else torch.cuda.current_stream()
    s.wait_stream(torch.cuda.current_stream())
    rc = _capi.lib().se2gpu_remove_outliers_device(B, ptr(dk1), ptr(dn1), cap1, ptr(dk2), ptr(dn2), cap2, ptr(dm), ptr(dnin), ptr(dF),
                                                    ptr(dit), C.c_void_p(s.cuda_stream))
    _capi.check(rc, "se2gpu_remove_outliers_device")
    s.synchronize()
    mm, nin, F, it = dm.cpu().numpy(), dnin.cpu().numpy(), dF.cpu().numpy().reshape(B, 3, 3), dit.cpu().numpy()
    return [(int(nin[b]), mm[b], F[b], int(it[b])) for b in range(B)]


def test_null_counts_mean_full_capacity(cases):
    """d_n1 = d_n2 = NULL: every row is its capacity, so the frames are padded with unmatched keypoints up to it."""
    sel = _small(cases, 24, 7, 1000)
    cap1 = max(len(c[1]) for c in sel) + 3; cap2 = max(len(c[2]) for c in sel) + 2
    rng = np.random.default_rng(9)
    pairs = []
    for c in sel:
        k1 = np.zeros(cap1, KP_DTYPE); k2 = np.zeros(cap2, KP_DTYPE); m = np.full(cap1, -1, np.int32)
        for k, src in ((k1, c[1]), (k2, c[2])):
            k["x"] = rng.uniform(0, 640, len(k)); k["y"] = rng.uniform(0, 480, len(k))
            k[:len(src)] = src
        m[:len(c[3])] = c[3]
        pairs.append((k1, k2, m))
    k1, k2, m = _pack(pairs, cap1, cap2)
    got = _device(k1, None, cap1, k2, None, cap2, m)
    for c, (a1, a2, mm), r in zip(sel, pairs, got):
        want = pyfundam.remove_outliers(a1, a2, mm)
        _check(r, want, repr(c[0]))
        _check(r, c[4][:1] + (np.r_[c[4][1], np.full(cap1 - len(c[3]), -1, np.int32)],) + c[4][2:], repr(c[0]))


def test_counts_outside_the_capacity_are_clamped(cases):
    """n < 0 counts as 0 and n > cap as cap (the oracle runs on the clamped count); matches12 past n1 is not touched."""
    base = [c for c in cases if c[0].family == "lattice" and 100 <= c[0].n <= 1000][:2] + _small(cases, 1, 20, 100)
    cap1 = max(len(c[1]) for c in base); cap2 = max(len(c[2]) for c in base)
    rows, n1, n2, wants = [], [], [], []
    for c in base:
        for a, b in ((-3, len(c[2])), (len(c[1]), -3), (-3, -3), (cap1 + 5, cap2 + 5), (len(c[1]), len(c[2]))):
            # a count past the capacity reads the whole row: pad it with unmatched keypoints
            k1 = np.zeros(cap1, KP_DTYPE); k2 = np.zeros(cap2, KP_DTYPE); m = np.full(cap1, SENTINEL, np.int32)
            k1[:len(c[1])] = c[1]; k2[:len(c[2])] = c[2]; m[:len(c[3])] = c[3]
            if a > cap1:
                m[len(c[3]):] = -1
            c1, c2 = min(max(a, 0), cap1), min(max(b, 0), cap2)
            mm = np.where(m[:c1] < c2, m[:c1], -1)
            rows.append((k1, k2, m)); n1.append(a); n2.append(b)
            wants.append((c1, pyfundam.remove_outliers(k1[:c1], k2[:max(c2, 1)], mm), m))
    k1, k2, m = _pack(rows, cap1, cap2)
    got = _device(k1, n1, cap1, k2, n2, cap2, m)
    for (c1, want, m0), r, a, b in zip(wants, got, n1, n2):
        nin, mm, F, it = r
        _check((nin, mm[:c1], F, it), want, (a, b))
        assert np.array_equal(mm[c1:], m0[c1:]), (a, b)
        if a <= 0 or b <= 0:
            assert nin == 0 and it == 0 and not F.any()


def test_match_indices_past_the_frame2_count(cases):
    """Matches in [n2, cap2) count as unmatched: the result is the oracle's with them set to -1, and they are left as
    they were unless the 10-inlier rule clears every match."""
    sel = [c for c in cases if c[0].expect == "ransac" and c[0].n >= 200][:2] + \
          [c for c in cases if c[0].expect == "static-none"][:1] + [c for c in cases if c[0].family == "lattice" and c[0].n == 16]
    rng = np.random.default_rng(11)
    cap1 = max(len(c[1]) for c in sel); cap2 = max(len(c[2]) for c in sel) + 8
    rows, n2, wants, stale = [], [], [], []
    for c in sel:
        k1, k2, m = c[1], c[2], c[3].copy()
        free = np.flatnonzero(m < 0)
        hit = np.sort(rng.choice(np.flatnonzero(m >= 0), 3, replace=False))
        m[hit] = len(k2) + rng.integers(0, cap2 - len(k2), 3)       # three matched entries point past n2
        if len(free):
            m[free[:2]] = len(k2) + 1
        past = m >= len(k2)
        want = pyfundam.remove_outliers(k1, k2, np.where(past, -1, m))
        rows.append((k1, k2, m)); n2.append(len(k2)); wants.append((want, m, past)); stale.append(past.sum())
    k1, k2, m = _pack(rows, cap1, cap2)
    n1 = [len(c[1]) for c in sel]
    got = _device(k1, n1, cap1, k2, n2, cap2, m)
    fired = []
    for c, (want, m0, past), r, a in zip(sel, wants, got, n1):
        nin, mm, F, it = r
        expect = np.where(past, m0 if want[0] >= 10 else -1, want[1])
        _check((nin, mm[:a], F, it), (want[0], expect, want[2], want[3]), repr(c[0]))
        assert (mm[a:] == SENTINEL).all()
        fired.append(want[0] < 10)
    assert any(fired) and not all(fired)


def test_side_stream_and_alternating_capacity(cases):
    """Calls on a non-default stream, alternating between cap1 = 8192 and small capacities (the launch's dynamic shared
    memory follows cap1)."""
    big = [c for c in cases if len(c[1]) == fs.MAX_PAIRS]
    small = _small(cases, 16)
    sparse = fs.sparse_capacity_pair()
    sparse_want = pyfundam.remove_outliers(*sparse)
    s = torch.cuda.Stream()
    for step in range(4):
        if step % 2 == 0:
            sel = [big[step // 2 % len(big)]]
            pairs = [sel[0][1:4], sparse]
            wants = [sel[0][4], sparse_want]
        else:
            sel = small[step // 2 * 8:step // 2 * 8 + 8]
            pairs = [c[1:4] for c in sel]
            wants = [c[4] for c in sel]
        cap1 = max(len(p[0]) for p in pairs); cap2 = max(len(p[1]) for p in pairs)
        k1, k2, m = _pack(pairs, cap1, cap2)
        got = _device(k1, [len(p[0]) for p in pairs], cap1, k2, [len(p[1]) for p in pairs], cap2, m, stream=s)
        for p, w, r in zip(pairs, wants, got):
            nin, mm, F, it = r
            _check((nin, mm[:len(p[0])], F, it), w, (step, cap1))


# ------------------------------------------------------------------------------------------ the device chain
def _warp(img, deg, tx, ty, scale=1.0):
    """Nearest-neighbour rotation by deg about the centre, scaling and a shift."""
    h, w = img.shape
    y, x = np.mgrid[0:h, 0:w].astype(np.float64)
    c, s = np.cos(np.radians(deg)) / scale, np.sin(np.radians(deg)) / scale
    cx, cy = (w - 1) / 2, (h - 1) / 2
    xs = c * (x - cx - tx) + s * (y - cy - ty) + cx
    ys = -s * (x - cx - tx) + c * (y - cy - ty) + cy
    return img[np.clip(np.rint(ys), 0, h - 1).astype(np.int64), np.clip(np.rint(xs), 0, w - 1).astype(np.int64)]


def _chain_frames(W, H):
    from tools import synth
    f = [synth.orb_frame(2000, W, H)]
    f.append(np.roll(f[-1], (2, 3), axis=(0, 1)))
    f.append(_warp(f[-1], 1.5, 1, -1))
    f.append(f[-1].copy())                                    # a repeated frame: zero motion
    f.append(np.roll(f[-1], (-3, 1), axis=(0, 1)))
    f.append(_warp(f[-1], -2.0, 2, 2, 1.03))
    f.append(np.roll(f[-1], (0, 45), axis=(0, 1)))            # past the 20 px window: almost nothing matches
    f.append(np.roll(f[-1], (1, -2), axis=(0, 1)))
    f.append(_warp(f[-1], 1.0, -2, 1, 0.98))
    return np.stack(f)


def test_device_chain_extract_match_remove_outliers_triangulate():
    from oracle import pyoracle
    from se2lam_b200.matcher import ORBmatcher
    from se2lam_b200.orb import ORBextractor
    from tools import geom_scenes as gs
    W, H, NF = 320, 240, 500
    frames = _chain_frames(W, H)
    B = len(frames) - 1
    f32 = np.float32
    grid = _capi.GridParams(f32(0), f32(0), f32(f32(64) / f32(W)), f32(f32(48) / f32(H)))
    sc = gs.track_scene(NF, seed=21)
    Kc = np.array([[200, 0, W / 2], [0, 200, H / 2], [0, 0, 1]], np.float32)
    ext = ORBextractor(NF, 1.2, 6, fastTh=20, max_width=W, max_height=H, max_batch=B + 1, device=0)
    m = ORBmatcher(0.9, max_queries=NF, max_db=NF)
    lib = _capi.lib()
    KB, DB = NF * KP_DTYPE.itemsize, NF * 32
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        d_img = torch.from_numpy(frames).to("cuda", non_blocking=False)
        d_kps = torch.zeros((B + 1) * KB, dtype=torch.uint8, device="cuda")
        d_desc = torch.zeros((B + 1) * DB, dtype=torch.uint8, device="cuda")
        d_cnt = torch.zeros(B + 1, dtype=torch.int32, device="cuda")
        d_prev = torch.zeros((B, NF * 2), dtype=torch.float32, device="cuda")
        d_m12 = torch.full((B, NF), -1, dtype=torch.int32, device="cuda")
        d_nm = torch.zeros(B, dtype=torch.int32, device="cuda")
        d_nin = torch.full((B,), -9, dtype=torch.int32, device="cuda")
        d_F = torch.zeros(B * 9, dtype=torch.float64, device="cuda")
        d_it = torch.full((B,), -9, dtype=torch.int32, device="cuda")
        d_obs, d_vm, d_T, d_K = [_tensor(a) for a in (sc["kf_observed"], sc["kf_view_mp"], sc["Tcr"], Kc)]
        d_lm = _tensor(np.tile(sc["local_mps"], (B, 1, 1)))
        d_good = torch.zeros((B, NF), dtype=torch.uint8, device="cuda")
        d_counts = torch.zeros((B, 2), dtype=torch.int32, device="cuda")
        st = C.c_void_p(s.cuda_stream)
        kp = lambda f: C.c_void_p(d_kps.data_ptr() + f * KB)       # noqa: E731
        desc = lambda f: C.c_void_p(d_desc.data_ptr() + f * DB)    # noqa: E731
        cnt = lambda f: C.c_void_p(d_cnt.data_ptr() + 4 * f)       # noqa: E731
        assert lib.se2gpu_orb_extract_device(ext.h, ptr(d_img), B + 1, W, H, W, W * H, ptr(d_kps), ptr(d_desc), ptr(d_cnt), st) == 0
        for b in range(B):
            assert lib.se2gpu_keypoints_to_points_device(kp(b), NF, cnt(b), ptr(d_prev[b]), st) == 0
            assert lib.se2gpu_match_by_window_device(m.h, kp(b), desc(b), NF, cnt(b), kp(b + 1), desc(b + 1), NF, cnt(b + 1),
                                                     ptr(d_prev[b]), grid, 20, 1, 0, 8, 0.9, ptr(d_m12[b]), ptr(d_nm[b:b + 1]),
                                                     st) == 0
        matched = d_m12.clone()
        # every pair (b, b + 1) in one call: frame b's keypoints as kp1, frame b + 1's (one capacity further) as kp2
        assert lib.se2gpu_remove_outliers_device(B, kp(0), cnt(0), NF, kp(1), cnt(1), NF, ptr(d_m12), ptr(d_nin), ptr(d_F),
                                                 ptr(d_it), st) == 0
        filtered = d_m12.clone()
        for b in range(B):
            assert lib.se2gpu_track_triangulate_device(kp(b), NF, cnt(b), kp(b + 1), ptr(d_m12[b]), ptr(d_obs), ptr(d_vm), ptr(d_T),
                                                       ptr(d_K), 0.1, 10.0, 2, ptr(d_lm[b]), ptr(d_good[b]), ptr(d_counts[b]),
                                                       st) == 0
    s.synchronize()

    g_cnt = d_cnt.cpu().numpy()
    g_kps = d_kps.cpu().numpy().view(KP_DTYPE).reshape(B + 1, NF); g_desc = d_desc.cpu().numpy().reshape(B + 1, NF, 32)
    g_matched, g_filtered, g_final = matched.cpu().numpy(), filtered.cpu().numpy(), d_m12.cpu().numpy()
    g_nin, g_F, g_it = d_nin.cpu().numpy(), d_F.cpu().numpy().reshape(B, 3, 3), d_it.cpu().numpy()
    g_lm = d_lm.cpu().numpy().view(np.float32).reshape(B, NF, 3)
    g_good, g_counts = d_good.cpu().numpy(), d_counts.cpu().numpy()

    ex = [pyoracle.OrbOracle(NF, 1.2, 6, 20).extract(f) for f in frames]
    for f, (k, d) in enumerate(ex):
        assert g_cnt[f] == len(k) and g_kps[f, :len(k)].tobytes() == k.tobytes() and g_desc[f, :len(k)].tobytes() == d.tobytes(), f
    ransac_kept = fired = 0
    for b in range(B):
        (k1, d1), (k2, d2) = ex[b], ex[b + 1]
        n1 = len(k1)
        prev = np.stack([k1["x"], k1["y"]], 1).astype(f32)
        _, m_o, _ = pyoracle.match_by_window(k1, d1, k2, d2, prev, (f32(0), f32(0), grid.inv_w, grid.inv_h), 20, 1, 0, 8, 0.9)
        assert np.array_equal(g_matched[b, :n1], m_o), b
        want = pyfundam.remove_outliers(k1, k2, m_o)
        _check((int(g_nin[b]), g_filtered[b, :n1], g_F[b], int(g_it[b])), want, b)
        mt, lmt, goodt, counts = pygeom.track_triangulate(k1, k2, want[1], sc["kf_observed"][:n1], sc["kf_view_mp"][:n1], sc["Tcr"], Kc,
                                                          0.1, 10.0, 2, sc["local_mps"][:n1])
        assert tuple(g_counts[b]) == counts and np.array_equal(g_final[b, :n1], mt), b
        assert same(g_lm[b, :n1], lmt) and np.array_equal(g_good[b, :n1], goodt), b
        npairs = int((m_o >= 0).sum())
        ransac_kept += npairs >= 15 and want[0] >= 10 and (mt >= 0).any()
        fired += npairs > 0 and want[0] == 0
    assert ransac_kept >= 1 and fired >= 1
    m.close()
