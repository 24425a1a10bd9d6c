"""se2lam_b200/csrc/fast_screen.h — the source passes C and E of orb_fast_cells are compiled from — checked on the host with the
packed-SIMD instructions emulated (tests/native/fast_nms_host.cpp): for every cell of 1..70 x 1..40 pixels in the TMA and the
plain-load layout, and random and adversarial score planes, the whole-word non-maximum suppression equals the scalar strict 3x3
maximum, and a simulated CTA's scan and emission give the scalar count and raster order. The GPU tests
(tests/test_orb_fast_cells_gpu.py, tests/test_orb_gpu.py) then pin the kernel bit for bit."""
import os
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_fast_nms_and_emission_on_the_host(tmp_path):
    exe = str(tmp_path / "fast_nms_host")
    res = subprocess.run(["g++", "-O2", "-std=c++14", "-Wall", "-Werror", os.path.join(ROOT, "tests", "native", "fast_nms_host.cpp"), "-o", exe],
                         capture_output=True, text=True)
    assert res.returncode == 0, res.stderr
    res = subprocess.run([exe], capture_output=True, text=True)
    assert res.returncode == 0, res.stdout + res.stderr
    assert res.stdout.startswith("OK ")
