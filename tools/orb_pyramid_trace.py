#!/usr/bin/env python
"""Kernel-by-kernel trace of the benchmark's ORB step: 64 frames of 640x480 (seeded as in bench.py), 1000 features, 8 levels,
scale 1.2, through se2gpu_orb_extract_device, under torch.profiler with CUDA activities.

usage: orb_pyramid_trace.py OUT_DIR [--steps K] [--warmup W]

Writes OUT_DIR/orb_trace.json (every kernel launch of the traced steps: name, start relative to the step's first kernel,
duration, in launch order) and OUT_DIR/orb_trace.txt (per kernel name: launches per step, mean duration, and the wall time from
the step's first pyramid kernel to the end of its last one; then the whole step: each launch's mean start and end, the gaps
across the chain's edges - last resize to FAST, FAST to the selection, selection to the descriptors; a negative gap is a
launch that began before its predecessor ended - and where the blur launches sit), and prints the text table."""
from __future__ import annotations

import argparse
import json
import os
import sys
from collections import OrderedDict

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

W, H, NFEAT, NLEV, BATCH = 640, 480, 1000, 8, 64
PYRAMID_KERNELS = ("orb_pyr0", "orb_resize")


def short_name(name: str) -> str:
    name = name.replace("(anonymous namespace)::", "").split("(")[0].replace("void ", "").strip()
    return name.split("::")[-1].split("<")[0]


def step_timeline(steps) -> list:
    """Per launch of a step (in launch order, repeated names numbered): mean start / end in us from the step's first kernel;
    then the mean gaps across the chain's edges and the step's span."""
    import numpy as np
    table, gaps = OrderedDict(), OrderedDict()
    for s in steps:
        t0 = s[0].time_range.start
        seen = {}
        for e in s:
            n = short_name(e.name)
            seen[n] = seen.get(n, 0) + 1
            key = f"{n} #{seen[n]}" if n.startswith(("orb_resize", "orb_blur")) else n
            table.setdefault(key, []).append((e.time_range.start - t0, e.time_range.end - t0))

        def first(prefix, last=False):
            m = [e for e in s if short_name(e.name).startswith(prefix)]
            return (m[-1] if last else m[0]) if m else None
        rz, fast, sel0, sel1, desc = (first("orb_resize", True), first("orb_fast_cells"), first("orb_select"),
                                      first("orb_select", True), first("orb_orient_describe"))
        for name, a, b in (("last resize end -> FAST start", rz, fast), ("FAST end -> selection start", fast, sel0),
                           ("selection end -> descriptors start", sel1, desc)):
            if a is not None and b is not None:
                gaps.setdefault(name, []).append(b.time_range.start - a.time_range.end)
        if sel0 is not None and sel1 is not sel0:
            gaps.setdefault("selection launch 1 end -> launch 2 start", []).append(sel1.time_range.start - sel0.time_range.end)
        gaps.setdefault("step span (first start..last end)", []).append(max(e.time_range.end for e in s) - t0)
    out = ["", "whole step, per launch (us from the step's first kernel start)", f"{'launch':32s} {'start':>9s} {'end':>9s}"]
    for k, v in table.items():
        a = np.array(v)
        out.append(f"{k:32s} {a[:, 0].mean():9.1f} {a[:, 1].mean():9.1f}")
    out += ["", f"{'edge':44s} {'mean us':>9s} {'min us':>9s} {'max us':>9s}"]
    for k, v in gaps.items():
        out.append(f"{k:44s} {np.mean(v):9.1f} {np.min(v):9.1f} {np.max(v):9.1f}")
    return out


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("out_dir")
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()

    import numpy as np
    import torch
    from torch.profiler import ProfilerActivity, profile

    from tools import synth
    from se2lam_b200.orb import ORBextractor

    if not torch.cuda.is_available():
        raise SystemExit("orb_pyramid_trace.py: no CUDA device")
    dev = torch.device("cuda", 0)
    imgs = torch.from_numpy(np.ascontiguousarray(synth.orb_batch(BATCH, first_seed=1000))).to(dev)
    ext = ORBextractor(NFEAT, 1.2, NLEV, fastTh=20, max_width=W, max_height=H, max_batch=BATCH, device=0)
    d_kps = torch.empty(BATCH * NFEAT * 28, dtype=torch.uint8, device=dev)
    d_desc = torch.empty(BATCH * NFEAT * 32, dtype=torch.uint8, device=dev)
    d_counts = torch.zeros(BATCH, dtype=torch.int32, device=dev)
    stream = torch.cuda.current_stream().cuda_stream

    def step():
        ext.extract_device(imgs, BATCH, H, W, d_kps, d_desc, d_counts, stream=stream)

    for _ in range(args.warmup):
        step()
    torch.cuda.synchronize()
    steps = []
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(args.steps):
            step()
            torch.cuda.synchronize()
    kernels = sorted((e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA and e.name and "memcpy" not in e.name.lower()
                      and "memset" not in e.name.lower()), key=lambda e: e.time_range.start)
    # split into steps: a step starts at its level-0 kernel (orb_pyr0 or orb_pyr0_undistort)
    for e in kernels:
        if short_name(e.name) in ("orb_pyr0", "orb_pyr0_undistort"):
            steps.append([])
        if steps:
            steps[-1].append(e)
    steps = [s for s in steps if s]
    os.makedirs(args.out_dir, exist_ok=True)
    rows = []
    for k, s in enumerate(steps):
        t0 = s[0].time_range.start
        for e in s:
            rows.append({"step": k, "name": short_name(e.name), "start_us": e.time_range.start - t0, "dur_us": e.time_range.elapsed_us()})
    per = OrderedDict()
    for k, s in enumerate(steps):
        resize_i = 0
        for e in s:
            n = short_name(e.name)
            if n.startswith("orb_resize"):
                resize_i += 1
                n = f"{n} (level {resize_i})"
            per.setdefault(n, []).append(e.time_range.elapsed_us())
    pyr_span = []
    for s in steps:
        pk = [e for e in s if short_name(e.name).startswith(PYRAMID_KERNELS)]
        if pk:
            pyr_span.append(max(e.time_range.end for e in pk) - pk[0].time_range.start)
    lines = [f"{torch.cuda.get_device_name(0)}; {len(steps)} traced steps of {BATCH} frames {W}x{H}, {NLEV} levels, scale 1.2",
             f"{'kernel':32s} {'launches/step':>13s} {'mean us':>9s} {'min us':>9s} {'max us':>9s}"]
    for n, v in per.items():
        lines.append(f"{n:32s} {len(v) / max(len(steps), 1):13.1f} {np.mean(v):9.1f} {np.min(v):9.1f} {np.max(v):9.1f}")
    if pyr_span:
        lines.append(f"{'pyramid span (first start..last end)':40s} mean {np.mean(pyr_span):7.1f} us, min {np.min(pyr_span):7.1f}, max {np.max(pyr_span):7.1f}")
    lines += step_timeline(steps)
    text = "\n".join(lines)
    with open(os.path.join(args.out_dir, "orb_trace.txt"), "w") as f:
        f.write(text + "\n")
    with open(os.path.join(args.out_dir, "orb_trace.json"), "w") as f:
        json.dump({"device": torch.cuda.get_device_name(0), "launches": rows}, f, indent=1)
    print(text)


if __name__ == "__main__":
    main()
