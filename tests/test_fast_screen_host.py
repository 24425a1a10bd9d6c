"""se2lam_b200/csrc/fast_screen.h — the source pass A of orb_fast_cells is compiled from — checked on the host with the packed-SIMD
instructions emulated (tests/native/fast_screen_host.cpp): the screen equals the scalar FAST-9-16 quick reject pixel by pixel, never
rejects a true corner, and a simulated CTA, in the TMA and the plain-load patch layout, screens every interior pixel of a cell exactly
once into a candidate list bounded by the cell's pixel count. The GPU parity tests (tests/test_orb_gpu.py) then pin the kernels bit
for bit."""
import os
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_fast_screen_and_pass_a_on_the_host(tmp_path):
    exe = str(tmp_path / "fast_screen_host")
    res = subprocess.run(["g++", "-O1", "-std=c++14", "-Wall", "-Werror", os.path.join(ROOT, "tests", "native", "fast_screen_host.cpp"), "-o", exe],
                         capture_output=True, text=True)
    assert res.returncode == 0, res.stderr
    res = subprocess.run([exe], capture_output=True, text=True)
    assert res.returncode == 0, res.stdout + res.stderr
    assert res.stdout.startswith("OK ")
