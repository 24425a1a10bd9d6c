"""se2lam_b200/csrc/lm.h, the Levenberg-Marquardt control of the windowed, pose-only, feature-edge and global BA kernels,
compiled on the host with g++ (tests/native/lm_host.cpp): lambda_0 and nu at the first iteration, both clamps of the accept
factor, nu doubling over rejections, a failed solve, ten failed trials ending in terminate and NOT_PD, rho == 0 and a NaN
trial chi2. The decisions are compared exactly, and lambda exactly where the factor is a clamp. The GPU tests then hold
each kernel's per-iteration statistics to the oracles'."""
import os
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_lm_control_on_the_host(tmp_path):
    exe = str(tmp_path / "lm_host")
    res = subprocess.run(["g++", "-O1", "-std=c++17", "-Wall", "-Werror", os.path.join(ROOT, "tests", "native", "lm_host.cpp"), "-o", exe],
                         capture_output=True, text=True)
    assert res.returncode == 0, res.stderr
    res = subprocess.run([exe], capture_output=True, text=True)
    assert res.returncode == 0, res.stdout + res.stderr
    assert res.stdout.startswith("OK ")
