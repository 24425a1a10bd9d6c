"""Times se2lam_b200.loc.Localizer steps on the GPU over a seeded map of about 200 keyframes and 20 k map points
(tools/loc_scenes.py, keyframes extracted by the library's own extractor): B = 1 eager against B = 1 replayed, and B = 8
and 64 replayed, at 320x240 with 500 features and at 640x480 with 1000, every stream relocalized at its second frame
(the fraction of tracked stream-steps is reported) and its frames already in device memory. Also times the CPU oracle chain (oracle/pyloc.py) per frame on one core.
Prints one JSON line with the card's name and power limit, read in the same call. Writes nothing into the tree."""
from __future__ import annotations

import argparse
import ctypes
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

SIZES = {"320x240": (320, 240, 500), "640x480": (640, 480, 1000)}


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
        return q.stdout.strip().splitlines()[0]
    except (OSError, IndexError):
        return "unknown"


def scene(size, n_kf=200):
    from se2lam_b200.orb import ORBextractor
    from tools import loc_scenes as ls
    w, h, nf = SIZES[size]
    cfg = ls.config(nfeatures=nf, w=w, h=h, max_local_mps=4096)
    ext = ORBextractor(nf, cfg["scale_factor"], cfg["nlevels"], fastTh=cfg["fast_th"], max_width=w, max_height=h, max_batch=1, device=0)
    path = np.array([(0.012 * k - 1.2, 0.3 * np.sin(0.05 * k), 0.004 * k) for k in range(n_kf)], np.float32)
    m = ls.build_map(11, cfg, share=100.0 / nf, path=path, extract=lambda img: ext(img), min_shared=10)
    return cfg, m


def handle(cfg, m, B):
    from se2lam_b200 import loc
    from se2lam_b200.loc import MAP_FIELDS
    for cap in (4096, 2048):
        try:
            p = loc.params(cfg["nfeatures"], cfg["scale_factor"], cfg["nlevels"], cfg["K"], cfg["grid"], cfg["bounds"], cfg["cTb"],
                           cfg["bTc"], cfg["huber"], cap, cfg["fast_th"])
            return loc.Localizer(B, cfg["w"], cfg["h"], p, {k: m[k] for k in MAP_FIELDS}), cap
        except RuntimeError:
            continue
    raise RuntimeError("no capacity fits the matcher's shared-memory resolve")


def run(cfg, m, B, eager, steps, warmup, T=32):
    import torch
    from se2lam_b200 import _capi
    from tools import loc_scenes as ls
    streams = [ls.stream(1000 + b, m, cfg, T, "along") for b in range(B)]
    frames = torch.from_numpy(np.stack([np.stack([s[0][k] for s in streams]) for k in range(T)])).cuda()
    odom = np.stack([np.stack([s[1][k] for s in streams]) for k in range(T)])
    h, cap = handle(cfg, m, B)
    h.set_eager(eager)
    h.step(frames[0], odom[0])
    h.step(frames[1], odom[1])
    pairs = [ls.loop_matches(h.state(b)["kp"], None, m, streams[b][3]) for b in range(B)]
    h.relocalize(list(range(B)), [s[3] for s in streams], pairs)
    L = _capi.lib()
    L.se2gpu_launch_count.restype = ctypes.c_ulonglong
    times, launches, tracked, nmp = [], [], [], []
    k, d = 2, 1
    for i in range(warmup + steps):
        l0 = L.se2gpu_launch_count()
        t0 = time.perf_counter()
        r = h.step(frames[k], odom[k])          # synchronous: returns after the record is read back
        dt = time.perf_counter() - t0
        if i >= warmup:
            times.append(dt); launches.append(L.se2gpu_launch_count() - l0)
            tracked.append(float(r["tracked"].mean())); nmp.append(float(r["n_local_mps"].mean()))
        if not 1 <= k + d < T:                  # walk the frames forwards and back: the odometry stays consistent
            d = -d
        k += d
    kernels, nodes = h.graph_nodes()
    med = float(np.median(times))
    h.close()
    return dict(B=B, mode="eager" if eager else "graph", median_step_ms=med * 1e3, fps=B / med, launches_per_step=int(np.median(launches)),
                graph_kernels=kernels, graph_nodes=nodes, tracked_fraction=float(np.mean(tracked)), mean_local_mps=float(np.mean(nmp)),
                max_local_mps=cap)


def oracle_ms(cfg, m, frames=8):
    """the CPU oracle chain (oracle/pyloc.py: ORB, projection, MatchByProjection, pose BA, covisibility, local map) per
    tracked frame of one stream, single thread"""
    from oracle import pyloc
    from se2lam_b200.loc import inv_level_sigma2
    from tools import loc_scenes as ls
    s = ls.stream(1000, m, cfg, frames + 2, "along")
    o = pyloc.LocOracle(cfg, m, inv_level_sigma2(cfg["scale_factor"], cfg["nlevels"]))
    o.step(s[0][0], s[1][0]); o.step(s[0][1], s[1][1])
    o.relocalize(s[3], ls.loop_matches(o.kp, None, m, s[3]))
    t = []
    for k in range(2, frames + 2):
        t0 = time.perf_counter()
        o.step(s[0][k], s[1][k])
        t.append(time.perf_counter() - t0)
    return float(np.median(t)) * 1e3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--sizes", default="320x240,640x480")
    a = ap.parse_args()
    out = {"card": card(), "configs": []}
    for size in a.sizes.split(","):
        cfg, m = scene(size)
        rows = [run(cfg, m, 1, True, a.steps, a.warmup)] + [run(cfg, m, B, False, a.steps, a.warmup) for B in (1, 8, 64)]
        out["configs"].append(dict(frame=size, nfeatures=cfg["nfeatures"], keyframes=len(m["kf_kp_ptr"]) - 1,
                                   map_points=len(m["mp_null"]), rows=rows, cpu_oracle_ms_per_frame=oracle_ms(cfg, m)))
    print(json.dumps(out))


if __name__ == "__main__":
    main()
