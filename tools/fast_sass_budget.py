#!/usr/bin/env python
"""SASS instruction budget of the FAST cell kernel's passes, from the sm_90a cross-compile (no GPU needed).

Compiles se2lam_b200/csrc/orb.cu for sm_90a with line information, disassembles both instantiations of orb_fast_cells, finds the
loops by their back-edges (a branch to a lower address) and assigns each loop to pass A, B or C by the source lines of its body:
the kernel opens each pass with a comment line `// pass A`, `// pass B`, `// pass C: ...`, `// pass E: ...`. A pass's loop is its
largest loop without a CTA barrier (the retry loop around the passes contains the barriers). Reports SASS instructions per loop
iteration and per unit (pass A: per pixel; pass B: per candidate; pass C: per 32-pixel bitmap word), the kernel's count of
BAR.SYNC and its registers per thread. Pass A stores each surviving pixel of its item with one predicated STS.U16 into the
candidate list, so the count of STS.U16 in its loop is the item's pixel count.

usage: python tools/fast_sass_budget.py [--json]
"""
from __future__ import annotations

import json
import os
import re
import shutil
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from se2lam_b200 import build  # noqa: E402

SRC = os.path.join(build.CSRC, "orb.cu")
KERNELS = {"tma": "orb_fast_cellsILb1E", "plain": "orb_fast_cellsILb0E"}
MARKER = re.compile(r"^\s*// pass ([ABCE])(:|$)")


def tool(name: str) -> str:
    for cand in (shutil.which(name), os.path.join("/usr/local/cuda/bin", name)):
        if cand and os.path.exists(cand):
            return cand
    raise FileNotFoundError(name)


def pass_regions() -> dict:
    """pass -> [first, last] source line of orb.cu, from the pass markers inside orb_fast_cells"""
    src = open(SRC).read().splitlines()
    start = next(i for i, t in enumerate(src) if re.search(r"__global__ .*\borb_fast_cells\(", t))
    end = next(i for i in range(start + 1, len(src)) if src[i].startswith("}"))
    marks = [(m.group(1), i + 1) for i in range(start, end) for m in [MARKER.match(src[i])] if m]
    if [name for name, _ in marks] != list("ABCE"):
        raise ValueError(f"orb_fast_cells must mark its passes A, B, C, E once each, in order; found {marks}")
    return {marks[k][0]: (marks[k][1], marks[k + 1][1] - 1) for k in range(len(marks) - 1)}


def compile_cubin(workdir: str) -> str:
    cubin = os.path.join(workdir, "orb.cubin")
    flags = [f for f in build.NVCC_FLAGS if f not in ("-shared", "-Xcompiler", "-fPIC", "-cudart", "static")]
    if "-lineinfo" not in flags:
        flags.append("-lineinfo")
    subprocess.run([tool("nvcc"), *flags, "-cubin", "-o", cubin, SRC], check=True, capture_output=True)
    return cubin


def registers(cubin: str) -> dict:
    """kernel key -> registers per thread"""
    out, cur = {}, None
    for row in subprocess.run([tool("cuobjdump"), "-res-usage", cubin], check=True, capture_output=True, text=True).stdout.splitlines():
        m = re.search(r"Function (\S+):", row)
        if m:
            keys = [k for k, v in KERNELS.items() if v in m.group(1)]
            cur = keys[0] if keys else None
            continue
        m = re.search(r"\bREG:(\d+)", row)
        if m and cur:
            out[cur] = int(m.group(1)); cur = None
    return out


def functions(dis: str) -> dict:
    """kernel key -> list of (address, opcode text, orb.cu line or -1) and {label: address}"""
    out = {}
    cur, line, pending = None, -1, []
    for row in dis.splitlines():
        m = re.match(r"\.text\.(\S+):", row)
        if m:
            keys = [k for k, v in KERNELS.items() if v in m.group(1)]
            cur = keys[0] if keys else None
            if cur:
                out[cur] = ([], {})
            pending = []; line = -1
            continue
        if cur is None:
            continue
        m = re.match(r"(\.L_x_\d+):", row)
        if m:
            pending.append(m.group(1)); continue
        m = re.search(r'//## File "([^"]+)", line (\d+)', row)
        if m:
            line = int(m.group(2)) if m.group(1).endswith("orb.cu") else -1; continue
        m = re.match(r"\s*/\*([0-9a-f]{4,})\*/\s+(.*?)\s*;?\s*$", row)
        if m:
            addr = int(m.group(1), 16)
            insts, labels = out[cur]
            for lab in pending:
                labels[lab] = addr
            pending = []
            insts.append((addr, m.group(2), line))
    return out


def loops(insts, labels):
    """(first index, back-edge index) of every loop"""
    index = {a: i for i, (a, _, _) in enumerate(insts)}
    res = []
    for i, (addr, text, _) in enumerate(insts):
        m = re.search(r"\bBRA\b.*`\((\.L_x_\d+)\)", text)
        if m and m.group(1) in labels and labels[m.group(1)] <= addr:
            res.append((index[labels[m.group(1)]], i))
    return res


def budget() -> dict:
    regions = pass_regions()
    with tempfile.TemporaryDirectory() as tmp:
        cubin = compile_cubin(tmp)
        funcs = functions(subprocess.run([tool("nvdisasm"), "-g", "-c", cubin], check=True, capture_output=True, text=True).stdout)
        regs = registers(cubin)
    result = {}
    for key in KERNELS:
        insts, labels = funcs[key]
        best, body_of = {}, {}
        for a, b in loops(insts, labels):
            body = insts[a:b + 1]
            if any("BAR.SYNC" in t for _, t, _ in body):
                continue
            votes = {}
            for _, _, ln in body:
                for name, (lo, hi) in regions.items():
                    if lo <= ln <= hi:
                        votes[name] = votes.get(name, 0) + 1
            if not votes:
                continue
            name = max(votes, key=votes.get)
            if len(body) > best.get(name, 0):
                best[name] = len(body); body_of[name] = body
        px = sum(1 for _, t, _ in body_of.get("A", ()) if re.search(r"\bSTS\.U16\b", t)) or None
        result[key] = {
            "pass_a_per_item": best.get("A"), "pass_a_px_per_item": px,
            "pass_a_per_px": best["A"] / px if "A" in best and px else None,
            "pass_b_per_candidate": best.get("B"), "pass_c_per_word": best.get("C"),
            "bar_sync": sum(1 for _, t, _ in insts if "BAR.SYNC" in t),
            "registers": regs.get(key),
        }
    return result


def main():
    res = budget()
    if "--json" in sys.argv:
        print(json.dumps(res, indent=1))
        return
    for key, r in res.items():
        print(f"orb_fast_cells<{'true' if key == 'tma' else 'false'}>: pass A {r['pass_a_per_item']} SASS per {r['pass_a_px_per_item']}-pixel item "
              f"({r['pass_a_per_px']:.1f} per pixel), pass B {r['pass_b_per_candidate']} per candidate, pass C {r['pass_c_per_word']} per word, "
              f"{r['bar_sync']} BAR.SYNC, {r['registers']} registers")


if __name__ == "__main__":
    main()
