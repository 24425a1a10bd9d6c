"""GPU parity of the HARRIS_SCORE extractor (scoreType = HARRIS_SCORE, reference src/ORBextractor.cpp:85-126, :625-629)
against the CPU oracle and the committed golden vectors: counts, all 28 keypoint bytes (response included) and the
32-byte descriptors, bit for bit."""
import os
import struct
import subprocess

import numpy as np
import pytest

from oracle import pyharris, pyoracle
from se2lam_b200 import _capi, build
from se2lam_b200.orb import FAST_SCORE, HARRIS_SCORE, ORBextractor
from tools import synth

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = np.load(os.path.join(ROOT, "tests", "golden", "orb_harris_golden.npz"))
CASES = {
    "synth1000": lambda: synth.orb_frame(1000), "synth1001": lambda: synth.orb_frame(1001),
    "constant": lambda: synth.orb_adversarial("constant"), "noise": lambda: synth.orb_adversarial("noise"),
    "lowcontrast": lambda: synth.orb_adversarial("lowcontrast"), "gradient": lambda: synth.orb_adversarial("gradient"),
    "small_320x240": lambda: synth.orb_frame(5, 320, 240), "odd_501x377": lambda: synth.orb_frame(6, 501, 377),
}


def assert_same(kg, dg, ko, do_, what=""):
    assert len(kg) == len(ko), f"{what}: {len(kg)} vs {len(ko)} keypoints"
    for field in ("octave", "x", "y", "response", "angle", "size", "class_id"):
        bad = np.flatnonzero(kg[field].view(np.int32) != ko[field].view(np.int32))
        assert bad.size == 0, f"{what}: {field} differs at {bad[:5]} ({kg[field][bad[:5]]} vs {ko[field][bad[:5]]})"
    bad = np.flatnonzero((dg != do_).any(axis=1))
    assert bad.size == 0, f"{what}: {bad.size} descriptors differ, first at {bad[:5]}"


def oracle(nf=1000, sf=1.2, nl=8, th=20):
    return pyharris.HarrisOrbOracle(nf, sf, nl, th)


@pytest.fixture(scope="module")
def ext():
    return ORBextractor(1000, 1.2, 8, HARRIS_SCORE, 20, max_width=640, max_height=480, max_batch=8)


@pytest.mark.parametrize("name", sorted(CASES))
def test_matches_golden_vectors(ext, name):
    kps, desc = ext(CASES[name]())
    assert_same(kps, desc, GOLD[name + "_kps"], GOLD[name + "_desc"], name)


def test_golden_frames_as_one_batch(ext):
    names = [n for n in sorted(CASES) if CASES[n]().shape == (480, 640)]
    imgs = np.stack([CASES[n]() for n in names])
    kps, desc, counts = ext.extract_batch(imgs)
    for i, n in enumerate(names):
        assert_same(kps[i, :counts[i]], desc[i, :counts[i]], GOLD[n + "_kps"], GOLD[n + "_desc"], f"batch {n}")


@pytest.mark.parametrize("nf,sf,nl,th", [(300, 1.2, 8, 20), (2000, 1.15, 6, 20), (1000, 1.3, 4, 7), (1000, 1.2, 8, 60),
                                         (2000, 1.3, 6, 60), (300, 1.15, 4, 7)])
def test_other_parameters(nf, sf, nl, th):
    img = synth.orb_frame(77)
    kg, dg = ORBextractor(nf, sf, nl, HARRIS_SCORE, th)(img)
    ko, do_ = oracle(nf, sf, nl, th).extract(img)
    assert_same(kg, dg, ko, do_, f"{nf} {sf} {nl} {th}")


def test_large_frames_take_the_other_fast_kernels():
    """1280x720 (orb_fast_cells<false>) and 1920x1080 (orb_fast_cells_big) with 1000 features."""
    for seed, w, h in ((4244, 1280, 720), (4242, 1920, 1080)):
        img = synth.orb_frame(seed, w, h)
        kg, dg = ORBextractor(1000, 1.2, 8, HARRIS_SCORE, 20, max_width=w, max_height=h)(img)
        ko, do_ = oracle().extract(img)
        assert_same(kg, dg, ko, do_, f"{w}x{h}")


def test_candidate_totals_beyond_the_selection_stage():
    """Noise at fastTh 7: level 0 has far more FAST candidates than the 6144 64-bit records orb_select<true> stages in
    shared memory, so its cells are selected in place in the 64-bit candidate buffer."""
    img = np.random.default_rng(99).integers(0, 256, (480, 640), dtype=np.uint8)
    kg, dg = ORBextractor(2000, 1.2, 8, HARRIS_SCORE, 7)(img)
    ko, do_ = oracle(2000, 1.2, 8, 7).extract(img)
    assert_same(kg, dg, ko, do_, "noise fastTh 7")


def periodic(period, seed, w=640, h=480):
    tile = np.random.default_rng(seed).integers(0, 256, (period, period), dtype=np.uint8)
    return np.ascontiguousarray(np.tile(tile, (h // period + 1, w // period + 1))[:h, :w])


@pytest.mark.parametrize("period,seed", [(8, 1), (12, 2), (16, 3), (5, 4)])
def test_periodic_textures_with_tied_responses(period, seed):
    """Identical windows inside and across cells: equal Harris responses everywhere, so the introselect permutation alone
    decides which keypoints survive and in which order."""
    img = periodic(period, seed)
    kg, dg = ORBextractor(1000, 1.2, 8, HARRIS_SCORE, 20)(img)
    ko, do_ = oracle().extract(img)
    r0 = ko[ko["octave"] == 0]["response"]
    assert len(r0) > len(np.unique(r0))                           # ties are really there
    assert_same(kg, dg, ko, do_, f"period {period}")


def test_undistort_submit_wait_and_device_entry():
    import torch
    K = np.array([[520.9, 0, 325.1], [0, 521.0, 249.7], [0, 0, 1]], np.float32)
    D = np.array([0.2312, -0.7849, -0.0033, -0.0001, 0.9172], np.float32)
    orc = oracle()
    n = 4
    e = ORBextractor(1000, 1.2, 8, HARRIS_SCORE, 20, max_batch=n)
    # set_undistort
    raw = synth.orb_frame(1000)
    e.set_undistort(K, D)
    kg, dg = e(raw)
    ko, do_ = orc.extract(pyoracle.undistort(raw, K, D))
    assert_same(kg, dg, ko, do_, "undistort")
    e.set_undistort(None)
    # submit / wait (the twin context inherits the score type)
    batches = [synth.orb_batch(n, first_seed=5000 + 10 * k) for k in range(3)]
    outs = [(np.zeros((n, 1000), pyoracle.KP_DTYPE), np.zeros((n, 1000, 32), np.uint8), np.zeros(n, np.int32)) for _ in range(2)]
    got = []
    for k, b in enumerate(batches):
        e.submit(b, *outs[k & 1])
        if k >= 1:
            e.wait()
            got.append(tuple(a.copy() for a in outs[(k - 1) & 1]))
    e.wait()
    got.append(tuple(a.copy() for a in outs[(len(batches) - 1) & 1]))
    for b, (kps, desc, counts) in zip(batches, got):
        for i in range(n):
            ko, do_ = orc.extract(b[i])
            assert_same(kps[i, :counts[i]], desc[i, :counts[i]], ko, do_, f"submit frame {i}")
    # extract_device on a torch stream
    imgs = synth.orb_batch(n, first_seed=6000)
    d_img = torch.from_numpy(imgs).cuda()
    d_kps = torch.zeros((n, 1000 * 28), dtype=torch.uint8, device="cuda")
    d_desc = torch.zeros((n, 1000, 32), dtype=torch.uint8, device="cuda")
    d_counts = torch.zeros(n, dtype=torch.int32, device="cuda")
    st = torch.cuda.Stream()
    with torch.cuda.stream(st):
        e.extract_device(d_img, n, 480, 640, d_kps, d_desc, d_counts, stream=st.cuda_stream)
    st.synchronize()
    kps = d_kps.cpu().numpy().view(pyoracle.KP_DTYPE).reshape(n, 1000)
    desc, counts = d_desc.cpu().numpy(), d_counts.cpu().numpy()
    for i in range(n):
        ko, do_ = orc.extract(imgs[i])
        assert_same(kps[i, :counts[i]], desc[i, :counts[i]], ko, do_, f"device frame {i}")


def test_fast_and_harris_handles_alternate():
    fast = ORBextractor(1000, 1.2, 8, FAST_SCORE, 20)
    harris = ORBextractor(1000, 1.2, 8, HARRIS_SCORE, 20)
    of, oh = pyoracle.OrbOracle(), oracle()
    for seed in (11, 12, 13):
        img = synth.orb_frame(seed)
        for e, o, what in ((fast, of, "fast"), (harris, oh, "harris"), (fast, of, "fast again")):
            kg, dg = e(img)
            ko, do_ = o.extract(img)
            assert_same(kg, dg, ko, do_, f"{what} {seed}")


def test_warp_nth_element_f32_matches_std_nth_element():
    rng = np.random.default_rng(8)
    lists, nths = [], []
    for case in range(2000):
        kind = case % 5
        n = int(rng.integers(1, 40)) if kind == 0 else int(rng.integers(40, 3000))
        if kind == 1:
            v = rng.integers(-1, 2, n).astype(np.float32) * np.float32(0.25)    # almost everything tied, +-0 included
            v[rng.random(n) < 0.3] = np.float32(-0.0)
        elif kind == 2:
            v = np.sort(rng.normal(size=n).astype(np.float32))[::-1]
        elif kind == 3:
            v = np.sort(rng.integers(-50, 50, n)).astype(np.float32) * np.float32(1e-3)
        else:
            v = rng.integers(-int(rng.integers(1, 300)), 300, n).astype(np.float32) * np.float32(3.7e-4)
        lists.append(np.ascontiguousarray(v, np.float32))
        nths.append(int(rng.integers(0, n)))
    for n in (64, 257, 1024, 2048):                                    # organ pipe: heap-select fallback
        half = (np.arange(n // 2) % 251).astype(np.float32) - 125
        lists.append(np.concatenate([half, half[::-1]])); nths.append(n // 2)
    offs = np.zeros(len(lists) + 1, np.int32)
    offs[1:] = np.cumsum([len(x) for x in lists])
    vals = np.concatenate(lists).astype(np.float32)
    nth = np.asarray(nths, np.int32)
    perm = np.zeros(len(vals), np.int32)
    _capi.check(_capi.lib().se2gpu_orb_debug_nth_element_f32(vals.ctypes.data, offs.ctypes.data, nth.ctypes.data, len(lists),
                                                             perm.ctypes.data, 0), "nth f32")
    for k, v in enumerate(lists):
        want = pyoracle.nth_element(v, nths[k])
        assert np.array_equal(perm[offs[k]:offs[k + 1]], want), f"list {k} (n={len(v)}, nth={nths[k]})"


def test_cpp_drop_in_header_with_harris_score(tmp_path):
    build.build_lib()
    exe = str(tmp_path / "orb_harris_demo")
    libdir = os.path.dirname(build.LIB_PATH)
    res = subprocess.run(["g++", "-O1", "-std=c++14", "-Wall", "-I", os.path.join(ROOT, "include"),
                          os.path.join(ROOT, "tests", "native", "orb_harris_demo.cpp"), "-o", exe, "-L", libdir, "-lse2gpu",
                          f"-Wl,-rpath,{libdir}"], capture_output=True, text=True)
    assert res.returncode == 0, res.stderr
    img = synth.orb_frame(1006)
    fin, fout = str(tmp_path / "in.bin"), str(tmp_path / "out.bin")
    with open(fin, "wb") as f:
        f.write(struct.pack("ii", 640, 480)); f.write(img.tobytes())
    res = subprocess.run([exe, fin, fout], capture_output=True, text=True)
    assert res.returncode == 0, res.stderr
    buf = open(fout, "rb").read()
    (N,) = struct.unpack_from("i", buf, 0)
    kps = np.frombuffer(buf, pyoracle.KP_DTYPE, N, 4)
    desc = np.frombuffer(buf, np.uint8, 32 * N, 4 + 28 * N).reshape(N, 32)
    ko, do_ = oracle().extract(img)
    assert_same(kps, desc, ko, do_, "drop-in header")
