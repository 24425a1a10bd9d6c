"""Builds se2lam_b200/lib/libse2gpu.so (hand-written sm_90a CUDA + the C ABI) in-tree with nvcc."""
from __future__ import annotations

import os
import shutil
import subprocess

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB_DIR = os.path.join(HERE, "lib")
LIB_PATH = os.path.join(LIB_DIR, "libse2gpu.so")
SOURCES = ["common.cu", "ba.cu", "ba_band.cu", "ba_loader.cu", "orb.cu", "matcher.cu", "bow.cu", "geom.cu", "fundam.cu", "pose_ba.cu", "feat_edge.cu", "global_ba.cu", "se3_ba.cu", "track.cu", "loc.cu", "loop.cu"]
GENCODE = ["-gencode", "arch=compute_90a,code=sm_90a"]     # H100 (Hopper)
NVCC_FLAGS = ["-O3", "-std=c++17", *GENCODE, "-lineinfo",
              "-Xcompiler", "-fPIC", "-shared", "-cudart", "static"]
# the flags of the last build: objects or a library built with other flags (another GPU architecture) are stale
FLAGS_STAMP = os.path.join(LIB_DIR, "nvcc_flags.txt")


def _nvcc() -> str:
    for cand in (shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and os.path.exists(cand):
            return cand
    raise RuntimeError("nvcc not found")


def sources():
    return [os.path.join(CSRC, s) for s in SOURCES if os.path.exists(os.path.join(CSRC, s))]


def _flags_changed() -> bool:
    try:
        return open(FLAGS_STAMP).read() != " ".join(NVCC_FLAGS)
    except OSError:
        return True


def is_stale() -> bool:
    if not os.path.exists(LIB_PATH) or _flags_changed():
        return True
    t = os.path.getmtime(LIB_PATH)
    deps = [os.path.join(CSRC, f) for f in os.listdir(CSRC)] + [os.path.join(HERE, "..", "include", "se2gpu.h")]
    return any(os.path.getmtime(d) > t for d in deps if os.path.isfile(d))


def build_lib(force: bool = False, verbose: bool = False) -> str:
    """One object per translation unit (compiled concurrently, re-used while its source and the shared headers are
    unchanged), then one link step. Objects live in se2lam_b200/lib/obj (git-ignored)."""
    if not force and not is_stale():
        return LIB_PATH
    force = force or _flags_changed()
    from concurrent.futures import ThreadPoolExecutor
    obj_dir = os.path.join(LIB_DIR, "obj")
    os.makedirs(obj_dir, exist_ok=True)
    env = dict(os.environ)
    env.pop("CXX", None); env.pop("CC", None)
    compile_flags = [f for f in NVCC_FLAGS if f not in ("-shared",)]
    headers = [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".h", ".inc", ".cuh"))] + \
              [os.path.join(HERE, "..", "include", "se2gpu.h")]
    hdr_time = max(os.path.getmtime(hh) for hh in headers if os.path.isfile(hh))

    def compile_one(src):
        obj = os.path.join(obj_dir, os.path.basename(src)[:-3] + ".o")
        if not force and os.path.exists(obj) and os.path.getmtime(obj) > max(os.path.getmtime(src), hdr_time):
            return obj, ""
        cmd = [_nvcc()] + compile_flags + (["-Xptxas", "-v"] if verbose else []) + ["-c", "-o", obj, src]
        res = subprocess.run(cmd, capture_output=True, text=True, env=env)
        if res.returncode != 0:
            raise RuntimeError("nvcc failed on " + src + ":\n" + res.stdout + res.stderr)
        return obj, res.stderr

    with ThreadPoolExecutor(max(len(SOURCES), 1)) as pool:
        results = list(pool.map(compile_one, sources()))
    if verbose:
        for _, log in results:
            print(log)
    link = [_nvcc(), "-shared", *GENCODE, "-cudart", "static", "-Xcompiler", "-fPIC",
            "-o", LIB_PATH] + [o for o, _ in results]
    res = subprocess.run(link, capture_output=True, text=True, env=env)
    if res.returncode != 0:
        raise RuntimeError("link failed:\n" + res.stdout + res.stderr)
    with open(FLAGS_STAMP, "w") as f:
        f.write(" ".join(NVCC_FLAGS))
    return LIB_PATH


if __name__ == "__main__":
    import sys
    print(build_lib(force="--force" in sys.argv, verbose="-v" in sys.argv))
