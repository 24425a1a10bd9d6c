"""include/se2lam/local_se3_ba.h compiles and links against libse2gpu.so, shapes removeOutlierChi2's vnOutlierIdxAll from
the per-edge flags (CPU), and on a GPU returns what se2lam_b200.se3ba returns for the same window
(tests/native/local_se3_ba_demo.cpp)."""
import ctypes as C
import os
import struct
import subprocess

import numpy as np
import pytest

from se2lam_b200 import build

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def compile_demo(tmp_path):
    build.build_lib()
    exe = str(tmp_path / "local_se3_ba_demo")
    libdir = os.path.dirname(build.LIB_PATH)
    cmd = ["g++", "-O1", "-std=c++14", "-Wall", "-I", os.path.join(ROOT, "include"),
           os.path.join(ROOT, "tests", "native", "local_se3_ba_demo.cpp"), "-o", exe, "-L", libdir, "-lse2gpu", f"-Wl,-rpath,{libdir}"]
    res = subprocess.run(cmd, capture_output=True, text=True)
    assert res.returncode == 0, res.stderr
    return exe


def read_lists(raw, off):
    (L,) = struct.unpack_from("i", raw, off); off += 4
    lists = []
    for _ in range(L):
        (n,) = struct.unpack_from("i", raw, off); off += 4
        lists.append(list(struct.unpack_from(f"{n}i", raw, off))); off += 4 * n
    return lists


def test_outlier_lists_have_the_shape_of_vnOutlierIdxAll(tmp_path):
    from se2lam_b200.se3ba import Window, outlier_lists
    exe = compile_demo(tmp_path)
    rng = np.random.default_rng(0)
    L, E = 7, 40
    pt = rng.integers(0, L - 1, E).astype(np.int32)  # the last point has no edge
    kf = rng.integers(0, 9, E).astype(np.int32)
    out = (rng.random(E) < 0.4).astype(np.uint8)
    blob = struct.pack("ii", L, E) + b"".join(struct.pack("iiB", int(p), int(k), int(o)) for p, k, o in zip(pt, kf, out))
    fin, fout = tmp_path / "in.bin", tmp_path / "out.bin"
    fin.write_bytes(blob)
    res = subprocess.run([exe, "lists", str(fin), str(fout)], capture_output=True, text=True)
    assert res.returncode == 0, res.stderr
    lists = read_lists(fout.read_bytes(), 0)
    assert len(lists) == L and lists[-1] == []
    for j in range(L):
        assert lists[j] == [int(k) for p, k, o in zip(pt, kf, out) if p == j and o]
    w = Window(np.tile(np.eye(4), (9, 1, 1)), np.zeros(9), np.zeros(9), np.zeros((L, 3)), pt, kf, np.zeros((E, 2)), np.ones(E))
    assert outlier_lists(w, out.astype(bool)) == lists


@pytest.mark.gpu
def test_header_matches_the_python_binding(tmp_path):
    from se2lam_b200 import se3ba
    from tools import se3_window_synth as S
    exe = compile_demo(tmp_path)
    prob, w = S.window(8, 400, seed=31, outlier_frac=0.2)
    prm = S.window_params(prob)
    N, O, L, E = w.sizes
    blob = struct.pack("iiii", N, O, L, E) + b"".join(a.tobytes() for a in (
        w.Tcw, w.fixed, w.prior, w.odo_from, w.odo_to, w.odo_measure, w.odo_info, w.xyz, w.edge_point, w.edge_kf, w.uv,
        w.inv_sigma2)) + C.string_at(C.addressof(prm), C.sizeof(prm))
    fin, fout = tmp_path / "in.bin", tmp_path / "out.bin"
    fin.write_bytes(blob)
    res = subprocess.run([exe, "run", str(fin), str(fout)], capture_output=True, text=True)
    assert res.returncode == 0, res.stderr
    raw = fout.read_bytes()
    rc, status, iters = struct.unpack_from("iii", raw, 0)
    ref = se3ba.local_se3_ba(w, prm)
    assert (rc, status, iters) == (0, ref["status"], ref["iterations"])
    assert raw[12:12 + 8 * E] == ref["chi2"].tobytes()
    assert raw[12 + 8 * E:12 + 9 * E] == ref["outlier"].astype(np.uint8).tobytes()
    assert read_lists(raw, 12 + 9 * E) == se3ba.outlier_lists(w, ref["outlier"])
    assert any(read_lists(raw, 12 + 9 * E))
