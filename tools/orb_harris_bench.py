"""Times the ORB extractor with HARRIS_SCORE against FAST_SCORE on device-resident batches (64 frames of 640x480, 1000
features, 8 levels; CUDA events on the launching stream), the orb_harris kernel alone (torch.profiler) and its share of
profile group 1 (FAST + orb_harris), and the oracle's Harris extraction on one host core. Prints one JSON line with the
card's name and power limit read in the same run; fails without a GPU.

    python tools/orb_harris_bench.py [--steps 50] [--warmup 5]
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

from oracle import pyharris  # noqa: E402
from se2lam_b200.orb import FAST_SCORE, HARRIS_SCORE, ORBextractor  # noqa: E402
from tools import synth  # noqa: E402

B, W, H, NF, NL = 64, 640, 480, 1000, 8


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs a GPU"
    imgs = synth.orb_batch(B)
    d_img = torch.from_numpy(imgs).cuda()
    d_kps = torch.empty((B, NF * 28), dtype=torch.uint8, device="cuda")
    d_desc = torch.empty((B, NF, 32), dtype=torch.uint8, device="cuda")
    d_counts = torch.empty(B, dtype=torch.int32, device="cuda")
    stream = torch.cuda.Stream()
    out = dict(tool="orb_harris_bench", frames_per_step=B, frame=f"{W}x{H}", nfeatures=NF, nlevels=NL, steps=args.steps)
    for name, st in (("fast", FAST_SCORE), ("harris", HARRIS_SCORE)):
        ext = ORBextractor(NF, 1.2, NL, st, 20, max_width=W, max_height=H, max_batch=B)

        def step():
            ext.extract_device(d_img, B, H, W, d_kps, d_desc, d_counts, stream=stream.cuda_stream)
        for _ in range(args.warmup):
            step()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        times = []
        for _ in range(args.steps):
            e0.record(stream); step(); e1.record(stream)
            e1.synchronize()
            times.append(e0.elapsed_time(e1))
        ms = float(np.median(times))
        kps = int(d_counts.sum().item())
        ext.profile(True)
        for _ in range(args.steps):
            step()
        torch.cuda.synchronize()
        prof = ext.profile_read()
        ext.profile(False)
        out[name] = dict(ms_per_step=round(ms, 4), keypoints_per_s=round(kps / (ms * 1e-3)),
                         profile_ms_per_step={g: round(v[0] / args.steps, 4) for g, v in prof.items()})
        if st == HARRIS_SCORE:
            with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as p:
                for _ in range(args.steps):
                    step()
                torch.cuda.synchronize()
            us = sum(e.device_time_total for e in p.key_averages() if "orb_harris" in e.key)
            hms = us / 1e3 / args.steps
            out["orb_harris_ms_per_step"] = round(hms, 4)
            out["orb_harris_share_of_group1"] = round(hms / (prof["orb_fast_cells"][0] / args.steps), 3)
        del ext
    o = pyharris.HarrisOrbOracle(NF, 1.2, NL, 20)
    t = []
    for i in range(5):
        t0 = time.perf_counter(); o.extract(imgs[i]); t.append((time.perf_counter() - t0) * 1e3)
    out["oracle_harris_ms_per_frame_one_core"] = round(float(np.median(t)), 2)
    out["harris_over_fast_step_time"] = round(out["harris"]["ms_per_step"] / out["fast"]["ms_per_step"], 4)
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    name, power = [x.strip() for x in smi.stdout.splitlines()[0].split(",")] if smi.returncode == 0 else (torch.cuda.get_device_name(0), "unknown")
    out.update(gpu=name, power_limit=power)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
