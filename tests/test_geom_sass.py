"""The fused multiply-adds in the geometry kernels' SASS are only those the host path has.

The reference's arithmetic has one fused form on an x86-64 AVX2 host: the rows of A in cvu::triangulate (cv::addWeighted's
dispatched kernel, pinned by oracle/pin_geom_against_cv2.py). Every other operation in geom.cu is an explicitly rounded
intrinsic that nvcc never contracts. The remaining FFMA / DFMA in the SASS belong to the correctly rounded division and
square root sequences (__fdiv_rn, __ddiv_rn, __fsqrt_rn, __dsqrt_rn and their out-of-line slow paths) and to sincos.
This test compiles geom.cu with line information, disassembles it, and checks each FFMA / DFMA against that list.
"""
import os
import re
import shutil
import subprocess

import pytest

from se2lam_b200 import build

SRC = os.path.join(build.CSRC, "geom.cu")
KERNELS = ("k_triangulate", "k_track_triangulate", "k_xyz_info", "k_projection_observations", "k_debug_svd4")
# source tokens whose expansion legitimately contains FFMA / DFMA
EXPANDING = ("__fdiv_rn", "__ddiv_rn", "__fsqrt_rn", "__dsqrt_rn", "sincos(")


def _tool(name):
    for cand in (shutil.which(name), os.path.join("/usr/local/cuda/bin", name)):
        if cand and os.path.exists(cand):
            return cand
    pytest.skip(f"{name} not found")


@pytest.fixture(scope="module")
def fma_sites(tmp_path_factory):
    out = tmp_path_factory.mktemp("sass")
    cubin = str(out / "geom.cubin")
    flags = [f for f in build.NVCC_FLAGS if f not in ("-shared", "-Xcompiler", "-fPIC", "-cudart", "static")]
    subprocess.run([_tool("nvcc"), *flags, "-cubin", "-o", cubin, SRC], check=True, capture_output=True)
    dis = subprocess.run([_tool("nvdisasm"), "-g", "-c", cubin], check=True, capture_output=True, text=True).stdout
    sites = []                     # (kernel, in_subroutine, op, source line number)
    kernel, label, line = None, "", 0
    for row in dis.splitlines():
        m = re.search(r"\.text\.(\S+):", row)
        if m:
            # mangled names carry the identifier's length: ..._geom_cu_<hash><len>k_nameE...
            names = [k for k in KERNELS if re.search(rf"{len(k)}{k}E", m.group(1))]
            kernel = names[0] if names else m.group(1); label = ""; continue
        m = re.match(r"\s*(\S+):\s*$", row)
        if m:
            # the out-of-line slow paths ($__internal_*) follow the kernel body; everything after the first one is theirs
            label = label if "__internal" in label else m.group(1); continue
        m = re.search(r'//## File "([^"]+)", line (\d+)', row)
        if m:
            line = int(m.group(2)) if m.group(1).endswith("geom.cu") else -1; continue
        m = re.search(r"\b(FFMA|DFMA)\b", row)
        if m:
            sites.append((kernel, "__internal" in label, m.group(1), line))
    return sites


def test_every_kernel_was_disassembled(fma_sites):
    assert {k for k, *_ in fma_sites} >= set(KERNELS)


def test_fmas_come_only_from_the_a_rows_and_rounded_sequences(fma_sites):
    src = open(SRC).read().splitlines()
    bad = []
    for kernel, in_sub, op, line in fma_sites:
        if in_sub or line < 0:
            continue               # out-of-line slow path of a rounded division / square root, or a CUDA header
        text = src[line - 1]
        if op == "FFMA" and "__fmaf_rn" in text:
            continue
        if any(t in text for t in EXPANDING):
            continue
        bad.append((kernel, op, line, text.strip()))
    assert not bad, bad


def test_explicit_fmas_are_the_sixteen_a_row_fmas(fma_sites):
    src = open(SRC).read().splitlines()
    fma_lines = {i + 1 for i, t in enumerate(src) if "__fmaf_rn" in t}
    assert len(fma_lines) == 4 and all(re.search(r"A\[(\d+ \+ )?k\] = __fmaf_rn", src[i - 1]) for i in fma_lines)
    for kernel in ("k_triangulate", "k_track_triangulate", "k_projection_observations"):
        n = sum(1 for k, in_sub, op, line in fma_sites if k == kernel and not in_sub and op == "FFMA" and line in fma_lines)
        assert n == 16, (kernel, n)
    assert not any(k in ("k_xyz_info", "k_debug_svd4") and line in fma_lines for k, _, _, line in fma_sites)
