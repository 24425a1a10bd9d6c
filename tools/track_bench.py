"""Times se2lam_b200.track.Tracker steps on the GPU: B = 1 eager against B = 1 replayed, and B = 8 and 64 replayed, on
seeded 320x240 streams (tools/track_scenes.py) with the frames already in device memory. Prints one JSON line with the
card's name and power limit, the median step time over many steps after warm-up, frames per second and launches per
step. Writes nothing into the tree."""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
        return q.stdout.strip().splitlines()[0]
    except (OSError, IndexError):
        return "unknown"


def run(B, eager, steps, warmup):
    import torch
    from se2lam_b200 import _capi, track
    from tools import track_scenes as ts
    cfg = ts.config(nfeatures=500, max_frames=10 ** 6)    # keyframes by c4 only: a steady tracking load
    p = track.params(cfg["nfeatures"], cfg["scale_factor"], cfg["nlevels"], cfg["K"], cfg["grid"], cfg["lower_depth"],
                     cfg["upper_depth"], cfg["cTb"], cfg["bTc"], cfg["odo_noise"], cfg["max_frames"], cfg["min_frames"])
    T = 32
    streams = [ts.stream(b % 8, T, "normal", cfg) for b in range(B)]
    frames = torch.from_numpy(np.stack([np.stack([s[0][k] for s in streams]) for k in range(T)])).cuda()
    odom = np.stack([np.stack([s[1][k] for s in streams]) for k in range(T)])
    obs = torch.zeros(cfg["nfeatures"], dtype=torch.uint8, device="cuda")
    vmp = torch.full((cfg["nfeatures"], 3), -1.0, device="cuda")
    t = track.Tracker(B, ts.W, ts.H, p)
    t.set_eager(eager)
    t.first(frames[0], odom[0])
    t.reset(list(range(B)), [vmp] * B)
    kfo = odom[0].copy()
    times, launches = [], []
    L = _capi.lib()
    L.se2gpu_launch_count.restype = __import__("ctypes").c_ulonglong
    for i in range(warmup + steps):
        k = 1 + i % (T - 1)
        kf = [dict(observed=obs, view_mp=vmp, n_obs_mp=0, accept=True, odom=kfo[b]) for b in range(B)]
        l0 = L.se2gpu_launch_count()
        t0 = time.perf_counter()
        t.step(frames[k], odom[k], kf)          # synchronous: returns after the record is read back
        dt = time.perf_counter() - t0
        if i >= warmup:
            times.append(dt); launches.append(L.se2gpu_launch_count() - l0)
    kernels, nodes = t.graph_nodes()
    med = float(np.median(times))
    return dict(B=B, mode="eager" if eager else "graph", median_step_ms=med * 1e3, fps=B / med,
                launches_per_step=int(np.median(launches)), graph_kernels=kernels, graph_nodes=nodes)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    a = ap.parse_args()
    rows = [run(1, True, a.steps, a.warmup), run(1, False, a.steps, a.warmup), run(8, False, a.steps, a.warmup),
            run(64, False, a.steps, a.warmup)]
    print(json.dumps({"card": card(), "frame": "320x240", "nfeatures": 500, "rows": rows}))


if __name__ == "__main__":
    main()
