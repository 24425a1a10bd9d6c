"""se2lam_b200/csrc/blur_px.h — the byte <-> float32 conversions orb_blur uses instead of I2F / F2I — checked on the host with PRMT
emulated (tests/native/blur_px_host.cpp): byte -> float is exact for all 256 bytes, and the magic-add rounding equals lrintf, ties
included, for every float32 in [0, 256], with the saturation at 255. The GPU tests (tests/test_orb_gpu.py,
tests/test_orb_blur_gpu.py) then pin the kernel's planes bit for bit."""
import os
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_blur_conversions_on_the_host(tmp_path):
    exe = str(tmp_path / "blur_px_host")
    res = subprocess.run(["g++", "-O2", "-std=c++14", "-Wall", "-Werror", os.path.join(ROOT, "tests", "native", "blur_px_host.cpp"), "-o", exe],
                         capture_output=True, text=True)
    assert res.returncode == 0, res.stderr
    res = subprocess.run([exe], capture_output=True, text=True)
    assert res.returncode == 0, res.stdout + res.stderr
    assert res.stdout.startswith("OK ")
