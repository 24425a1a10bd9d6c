"""The batched local BA's cluster kernel synchronises with the cluster barrier, and the persistent kernel it shares its body
with keeps the registers and spills it had before the body became a template over the team of CTAs.

ba_persistent_cluster must end its phases with barrier.cluster (UCGABAR_ARV / UCGABAR_WAIT in sm_90a SASS); ba_persistent
synchronises its cooperative grid and has neither. The budget of ba_persistent is what ptxas (CUDA 12.9, sm_90a) reported for
it before the team template: 128 registers, 356 bytes of spill stores and 428 bytes of spill loads.
"""
import os
import re
import shutil
import subprocess

import pytest

from se2lam_b200 import build

SRC = os.path.join(build.CSRC, "ba.cu")
BUDGET = {"registers": 128, "spill_stores": 356, "spill_loads": 428}


def _tool(name):
    for cand in (shutil.which(name), os.path.join("/usr/local/cuda/bin", name)):
        if cand and os.path.exists(cand):
            return cand
    pytest.skip(f"{name} not found")


@pytest.fixture(scope="module")
def compiled(tmp_path_factory):
    out = tmp_path_factory.mktemp("ba_sass")
    cubin = str(out / "ba.cubin")
    flags = [f for f in build.NVCC_FLAGS if f not in ("-shared", "-Xcompiler", "-fPIC", "-cudart", "static")]
    res = subprocess.run([_tool("nvcc"), *flags, "-Xptxas", "-v", "-cubin", "-o", cubin, SRC], check=True, capture_output=True, text=True)
    sass = subprocess.run([_tool("cuobjdump"), "-sass", cubin], check=True, capture_output=True, text=True).stdout
    return res.stderr, sass


def _kernel_sass(sass, name):
    parts = re.split(r"\n\s*Function : ", sass)
    hits = [p for p in parts if re.match(rf"\S*{len(name)}{name}E", p)]
    assert len(hits) == 1, name
    return hits[0]


def _resources(log, name):
    m = re.search(rf"Function properties for \S*{len(name)}{name}E\S*\n\s*(\d+) bytes stack frame, (\d+) bytes spill stores, "
                  rf"(\d+) bytes spill loads\n.*?Used (\d+) registers", log)
    assert m, name
    return {"spill_stores": int(m.group(2)), "spill_loads": int(m.group(3)), "registers": int(m.group(4))}


def test_cluster_kernel_uses_the_cluster_barrier(compiled):
    _, sass = compiled
    cluster = _kernel_sass(sass, "ba_persistent_cluster")
    grid = _kernel_sass(sass, "ba_persistent")
    assert "UCGABAR_ARV" in cluster and "UCGABAR_WAIT" in cluster
    assert "UCGABAR_ARV" not in grid and "UCGABAR_WAIT" not in grid


def test_persistent_kernel_keeps_its_register_budget(compiled):
    log, _ = compiled
    got = _resources(log, "ba_persistent")
    assert all(got[k] <= BUDGET[k] for k in BUDGET), got



def test_both_instantiations_contract_the_same_fmas(compiled):
    """The cluster kernel spells out edge_xyz's contraction (ClusterTeam::kExplicitFma): it fuses exactly what ba_persistent fuses."""
    _, sass = compiled
    cluster = _kernel_sass(sass, "ba_persistent_cluster")
    grid = _kernel_sass(sass, "ba_persistent")
    assert len(re.findall(r"\bDFMA\b", cluster)) == len(re.findall(r"\bDFMA\b", grid))
