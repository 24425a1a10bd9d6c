"""include/se2lam/global_ba.h compiles against cv_compat.h, links against libse2gpu.so and, on a GPU, returns what
se2lam_b200.globalba returns for the same graph and map points (tests/native/global_ba_demo.cpp)."""
import os
import struct
import subprocess

import numpy as np
import pytest

from se2lam_b200 import build
from tools import posegraph_synth as S

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def compile_demo(tmp_path):
    build.build_lib()
    exe = str(tmp_path / "global_ba_demo")
    libdir = os.path.dirname(build.LIB_PATH)
    cmd = ["g++", "-O1", "-std=c++14", "-Wall", "-I", os.path.join(ROOT, "include"), os.path.join(ROOT, "tests", "native", "global_ba_demo.cpp"),
           "-o", exe, "-L", libdir, "-lse2gpu", f"-Wl,-rpath,{libdir}"]
    res = subprocess.run(cmd, capture_output=True, text=True)
    assert res.returncode == 0, res.stderr
    return exe


def test_global_ba_header_compiles_and_links(tmp_path):
    compile_demo(tmp_path)


@pytest.mark.gpu
@pytest.mark.parametrize("kind,N", [("loop", 80), ("chain", 1)])
def test_global_ba_header_matches_the_python_binding(tmp_path, kind, N):
    from se2lam_b200 import globalba
    exe = compile_demo(tmp_path)
    g = S.graph(seed=N, N=N, kind=kind)
    kf, view = S.map_points(N + 1, g, 300)
    blob = struct.pack("i", N) + g["Tbc"].astype(np.float32).tobytes() + g["Tcw"].astype(np.float32).tobytes()
    blob += g["fixed"].astype(np.uint8).tobytes() + struct.pack("i", len(g["edges"]))
    for i, j, Z, O in g["edges"]:
        blob += struct.pack("ii", i, j) + np.asarray(Z, np.float32).tobytes() + np.asarray(O, np.float32).tobytes()
    blob += struct.pack("i", len(kf))
    for m in range(len(kf)):
        blob += struct.pack("i", int(kf[m])) + view[m].astype(np.float32).tobytes()
    fin, fout = tmp_path / "in.bin", tmp_path / "out.bin"
    fin.write_bytes(blob)
    res = subprocess.run([exe, str(fin), str(fout)], capture_output=True, text=True)
    assert res.returncode == 0, res.stderr
    raw = fout.read_bytes()
    ref = globalba.GlobalBA(g["Tcw"], g["fixed"], g["edges"], globalba.params(g["Tbc"]))
    status, iters = struct.unpack_from("ii", raw, 0)
    assert (status, iters) == (ref["status"], ref["iterations"])
    assert raw[8:8 + 64 * N] == ref["Tcw"].tobytes()
    assert raw[8 + 64 * N:] == globalba.update_map_points(kf, view, ref["Tcw"]).tobytes()
