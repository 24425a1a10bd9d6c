"""orb_harris evaluates the reference's Harris expression with every float operation rounded on its own: its SASS has no
fused multiply-add (the x86-64 reference build contracts nothing), only the three int-to-float conversions, the five
multiplications and the three additions / subtractions of `((float)a*b - (float)c*c - k*((float)a+b)*((float)a+b)) * s`."""
import os
import re
import shutil
import subprocess
from collections import Counter

import pytest

from se2lam_b200 import build

SRC = os.path.join(build.CSRC, "orb.cu")


def _tool(name):
    for cand in (shutil.which(name), os.path.join("/usr/local/cuda/bin", name)):
        if cand and os.path.exists(cand):
            return cand
    pytest.skip(f"{name} not found")


def test_orb_harris_float_ops_are_unfused(tmp_path):
    cubin = str(tmp_path / "orb.cubin")
    flags = [f for f in build.NVCC_FLAGS if f not in ("-shared", "-Xcompiler", "-fPIC", "-cudart", "static")]
    subprocess.run([_tool("nvcc"), *flags, "-cubin", "-o", cubin, SRC], check=True, capture_output=True)
    sass = subprocess.run([_tool("cuobjdump"), "-sass", cubin], check=True, capture_output=True, text=True).stdout
    body, cur = [], None
    for row in sass.splitlines():
        m = re.search(r"Function : (\S+)", row)
        if m:
            cur = m.group(1); continue
        if cur and re.search(r"10orb_harrisE", cur):
            m = re.match(r"\s*/\*[0-9a-f]{4}\*/\s+(?:@!?U?P\w+\s+)?([A-Z][A-Z0-9_.]*)", row)
            if m:
                body.append(m.group(1))
    assert body, "orb_harris not found in the SASS"
    ops = Counter(op.split(".")[0] for op in body)
    assert ops["FFMA"] == 0 and ops["DFMA"] == 0, ops     # (HFMA2.MMA appears only as a constant-move idiom)
    assert (ops["I2FP"] + ops["I2F"], ops["FMUL"], ops["FADD"]) == (3, 5, 3), ops
