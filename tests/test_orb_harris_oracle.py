"""CPU: the HARRIS_SCORE ORB oracle (oracle/orb_harris_oracle.cpp) reproduces its golden vectors (pinned against cv2 4.13 by
oracle/pin_orb_harris_against_cv2.py), its HarrisResponses matches a numpy float32 restatement, and the host builds of
the Harris selection's order key (resp_key.h) and 64-bit introselect match the float order and std::nth_element."""
import os
import subprocess

import numpy as np
import pytest

from oracle import pyharris, pyoracle
from tools import synth

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = np.load(os.path.join(ROOT, "tests", "golden", "orb_harris_golden.npz"))
CASES = {
    "synth1000": lambda: synth.orb_frame(1000), "synth1001": lambda: synth.orb_frame(1001),
    "constant": lambda: synth.orb_adversarial("constant"), "noise": lambda: synth.orb_adversarial("noise"),
    "lowcontrast": lambda: synth.orb_adversarial("lowcontrast"), "gradient": lambda: synth.orb_adversarial("gradient"),
    "small_320x240": lambda: synth.orb_frame(5, 320, 240), "odd_501x377": lambda: synth.orb_frame(6, 501, 377),
}
f32 = np.float32


def harris_np(img, x, y):
    """HarrisResponses (reference src/ORBextractor.cpp:85-126) in numpy float32 scalars, C++ evaluation order, no contraction."""
    P = img[y - 4:y + 5, x - 4:x + 5].astype(np.int64)
    Ix = (P[1:-1, 2:] - P[1:-1, :-2]) * 2 + (P[:-2, 2:] - P[:-2, :-2]) + (P[2:, 2:] - P[2:, :-2])
    Iy = (P[2:, 1:-1] - P[:-2, 1:-1]) * 2 + (P[2:, :-2] - P[:-2, :-2]) + (P[2:, 2:] - P[:-2, 2:])
    a, b, c = f32(int((Ix * Ix).sum())), f32(int((Iy * Iy).sum())), f32(int((Ix * Iy).sum()))
    s = f32(1) / f32(7140)
    s4 = ((s * s) * s) * s
    return f32(f32(f32(a * b) - f32(c * c)) - f32(f32(f32(0.04) * f32(a + b)) * f32(a + b))) * s4


@pytest.mark.parametrize("name", sorted(CASES))
def test_oracle_matches_golden(name):
    kps, desc = pyharris.HarrisOrbOracle().extract(CASES[name]())
    assert kps.tobytes() == GOLD[name + "_kps"].tobytes()
    assert desc.tobytes() == GOLD[name + "_desc"].tobytes()


def test_harris_responses_are_not_fast_scores():
    k_h, _ = pyharris.HarrisOrbOracle().extract(synth.orb_frame(1000))
    k_f, _ = pyoracle.OrbOracle().extract(synth.orb_frame(1000))
    assert len(k_h) == len(k_f) == 1000
    assert not np.array_equal(k_h["response"], np.round(k_h["response"]))      # float responses, not integer scores
    assert np.all(np.diff(k_h["octave"]) >= 0) and np.all(k_h["class_id"] == -1)


def windows():
    rng = np.random.default_rng(21)
    out = []
    for _ in range(300):                                          # random content
        out.append(rng.integers(0, 256, (9, 9), dtype=np.uint8))
    for v in (0, 17, 255):                                        # flat: response 0
        out.append(np.full((9, 9), v, np.uint8))
    yy, xx = np.mgrid[0:9, 0:9]
    for p in (1, 2, 3):                                           # checkerboards / stripes: large a, b (float(a) rounds)
        out.append((((xx // p) + (yy // p)) % 2 * 255).astype(np.uint8))
        out.append(((xx // p) % 2 * 255).astype(np.uint8))
    for t in (-2, 0, 3):                                          # diagonal edges: negative c
        out.append(((xx + yy > 8 + t) * 255).astype(np.uint8))
        out.append(((xx - yy > t) * 200 + 20).astype(np.uint8))
    for _ in range(100):                                          # saturated random blocks
        out.append(np.kron(rng.integers(0, 2, (5, 5)), np.ones((2, 2), int))[:9, :9].astype(np.uint8) * 255)
    return out


def test_oracle_harris_matches_numpy_restatement():
    ws = windows()
    img = np.zeros((11, 11 * len(ws)), np.uint8)
    for i, w in enumerate(ws):
        img[1:10, 11 * i + 1:11 * i + 10] = w
    xs = np.array([11 * i + 5 for i in range(len(ws))], np.float32)
    ys = np.full(len(ws), 5, np.float32)
    got = pyharris.harris(img, xs, ys)
    want = np.array([harris_np(img, int(x), 5) for x in xs], np.float32)
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32))
    assert got[300] == 0 and got[301] == 0 and got[302] == 0          # flat windows
    assert (got < 0).any() and (got > 0).any()


def run_native(tmp_path, name, expect):
    exe = tmp_path / name
    subprocess.run(["g++", "-O2", "-std=c++17", "-o", str(exe), os.path.join(ROOT, "tests", "native", name + ".cpp")], check=True)
    out = subprocess.run([str(exe)], capture_output=True, text=True)
    assert out.returncode == 0, out.stderr
    assert expect in out.stdout


def test_resp_key_is_order_preserving(tmp_path):
    """se2lam_b200/csrc/resp_key.h (host build): +-0, denormals, +-FLT_MAX, neighbouring floats across signs."""
    run_native(tmp_path, "resp_key_host", "order-preserving")


def test_introselect64_matches_std_nth_element(tmp_path):
    """The 64-bit instantiation of introselect.h against std::nth_element with a float comparator on tie-heavy lists."""
    run_native(tmp_path, "introselect64_check", "identical")


def test_create_scored_rejects_unknown_score_type():
    from se2lam_b200 import _capi
    L = _capi.lib()
    for bad in (2, -1, 7):
        assert not L.se2gpu_orb_create_scored(1000, 1.2, 8, bad, 20, 640, 480, 1, 0)
        assert "score type" in _capi.last_error()
