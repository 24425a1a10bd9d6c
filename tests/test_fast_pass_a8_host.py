"""Pass A of orb_fast_cells as the kernel splits it — 8-pixel items of two patch words, two fastpx::screen4 calls on 16 shared
words, one shared atomicAdd per lane — simulated on the host (tests/native/fast_pass_a8_host.cpp) from se2lam_b200/csrc/fast_screen.h,
in the TMA and the plain-load patch layout: every interior pixel is screened exactly once, the candidates equal the scalar quick
reject, the list stays within the cell's pixel count, and no read goes more than one word past the patch."""
import os
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_pass_a_8_pixel_items_on_the_host(tmp_path):
    exe = str(tmp_path / "fast_pass_a8_host")
    res = subprocess.run(["g++", "-O1", "-std=c++14", "-Wall", "-Werror", os.path.join(ROOT, "tests", "native", "fast_pass_a8_host.cpp"), "-o", exe],
                         capture_output=True, text=True)
    assert res.returncode == 0, res.stderr
    res = subprocess.run([exe], capture_output=True, text=True)
    assert res.returncode == 0, res.stdout + res.stderr
    assert res.stdout.startswith("OK ")
