"""The fused multiply-adds in fundam.cu's SASS come only from correctly rounded divisions and square roots.

OpenCV's fundam.cpp is built without FMA on an x86-64 host, so the kernel fuses nothing: every operation is an explicitly
rounded intrinsic that nvcc never contracts. The FFMA / DFMA left belong to the __ddiv_rn / __dsqrt_rn sequences and their
out-of-line slow paths. Same method as tests/test_geom_sass.py.
"""
import os
import re
import shutil
import subprocess

import pytest

from se2lam_b200 import build

SRC = os.path.join(build.CSRC, "fundam.cu")
KERNELS = ("k_remove_outliers", "k_debug_niters")
EXPANDING = ("__ddiv_rn", "__dsqrt_rn")


def _tool(name):
    for cand in (shutil.which(name), os.path.join("/usr/local/cuda/bin", name)):
        if cand and os.path.exists(cand):
            return cand
    pytest.skip(f"{name} not found")


@pytest.fixture(scope="module")
def fma_sites(tmp_path_factory):
    out = tmp_path_factory.mktemp("sass")
    cubin = str(out / "fundam.cubin")
    flags = [f for f in build.NVCC_FLAGS if f not in ("-shared", "-Xcompiler", "-fPIC", "-cudart", "static")]
    subprocess.run([_tool("nvcc"), *flags, "-cubin", "-o", cubin, SRC], check=True, capture_output=True)
    dis = subprocess.run([_tool("nvdisasm"), "-g", "-c", cubin], check=True, capture_output=True, text=True).stdout
    sites, kernels = [], set()
    kernel, label, line = None, "", 0
    for row in dis.splitlines():
        m = re.search(r"\.text\.(\S+):", row)
        if m:
            names = [k for k in KERNELS if re.search(rf"{len(k)}{k}E", m.group(1))]
            kernel = names[0] if names else m.group(1); label = ""; kernels.add(kernel); continue
        m = re.match(r"\s*(\S+):\s*$", row)
        if m:
            label = label if "__internal" in label else m.group(1); continue
        m = re.search(r'//## File "([^"]+)", line (\d+)', row)
        if m:
            line = int(m.group(2)) if m.group(1).endswith("fundam.cu") else -1; continue
        m = re.search(r"\b(FFMA|DFMA)\b", row)
        if m:
            sites.append((kernel, "__internal" in label, m.group(1), line))
    return kernels, sites


def test_every_kernel_was_disassembled(fma_sites):
    assert fma_sites[0] >= set(KERNELS)


def test_fmas_come_only_from_rounded_divisions_and_square_roots(fma_sites):
    src = open(SRC).read().splitlines()
    bad = []
    for kernel, in_sub, op, line in fma_sites[1]:
        if in_sub or line < 0:
            continue
        text = src[line - 1]
        if any(t in text for t in EXPANDING):
            continue
        bad.append((kernel, op, line, text.strip()))
    assert not bad, bad


def test_source_has_no_explicit_fma():
    txt = open(SRC).read()
    assert not re.search(r"__fma[f]?_r[nzdu]|\bfmaf?\(", txt)
