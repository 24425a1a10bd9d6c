"""include/se2lam/feat_edge.h compiles against cv_compat.h, links against libse2gpu.so and, on a GPU, returns what
se2lam_b200.featgraph returns for the same pairs (tests/native/feat_edge_demo.cpp)."""
import os
import struct
import subprocess

import numpy as np
import pytest

from se2lam_b200 import build
from tools import featgraph_synth as S

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def compile_demo(tmp_path):
    build.build_lib()
    exe = str(tmp_path / "feat_edge_demo")
    libdir = os.path.dirname(build.LIB_PATH)
    cmd = ["g++", "-O1", "-std=c++14", "-Wall", "-I", os.path.join(ROOT, "include"), os.path.join(ROOT, "tests", "native", "feat_edge_demo.cpp"),
           "-o", exe, "-L", libdir, "-lse2gpu", f"-Wl,-rpath,{libdir}"]
    res = subprocess.run(cmd, capture_output=True, text=True)
    assert res.returncode == 0, res.stderr
    return exe


def test_feat_edge_header_compiles_and_links(tmp_path):
    compile_demo(tmp_path)


@pytest.mark.gpu
@pytest.mark.parametrize("matched", [0, 1])
def test_feat_edge_header_matches_the_python_binding(tmp_path, matched):
    from se2lam_b200 import featgraph
    exe = compile_demo(tmp_path)
    pairs = [S.scene(300 + b, n, noise=0.3, outlier_share=0.1 * matched, outlier_size=(0.2, 0.4)) for b, n in enumerate((40, 2, 9, 120, 300))]
    blob = struct.pack("ii", matched, len(pairs)) + pairs[0]["Tbc"].astype(np.float32).tobytes()
    for p in pairs:
        blob += p["Tcw0"].tobytes() + p["Tcw1"].tobytes() + struct.pack("i", len(p["xyz"]))
        for j in range(len(p["xyz"])):
            blob += p["xyz"][j].tobytes() + p["z0"][j].tobytes() + p["z1"][j].tobytes() + p["info0"][j].tobytes() + p["info1"][j].tobytes()
    fin, fout = tmp_path / "in.bin", tmp_path / "out.bin"
    fin.write_bytes(blob)
    res = subprocess.run([exe, str(fin), str(fout)], capture_output=True, text=True)
    assert res.returncode == 0, res.stderr
    raw = fout.read_bytes()
    ref = featgraph.UpdateFeatGraph(pairs, featgraph.params(pairs[0]["Tbc"]), mode=matched)
    off = 0
    for p, r in zip(pairs, ref):
        ret, status, iters = struct.unpack_from("iii", raw, off); off += 12
        measure = raw[off:off + 64]; off += 64
        info = raw[off:off + 144]; off += 144
        outlier = raw[off:off + len(p["xyz"])]; off += len(p["xyz"])
        assert status == r["status"] and iters == r["iterations"] and ret == (1 if status == featgraph.TOO_FEW else 0)
        assert outlier == r["outlier"].tobytes()
        if ret == 0:
            assert measure == r["measure"].tobytes() and info == r["info"].tobytes()
    assert off == len(raw)
