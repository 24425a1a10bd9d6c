"""Timing of the map-point updates (se2gpu_mp_*_device) on the GPU, against the CPU oracle on one core.

Workloads: one keyframe's worth of addObservation (about 1 000 updates), 64 keyframes' worth in one call (64 000), and
updateMeasureInKFs over a local-BA window of 5 000 points (the C4 window's size). Each timed call starts from fresh copies
of the tables (copied on the device outside the timed window), timed by CUDA events over `--reps` calls after `--warmup`.
The card's name and power limit are read in the same run and printed with the numbers as one JSON line.

    python tools/mappoint_bench.py [--reps 50] [--warmup 5] [--out results/mappoint_bench.json]
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import pymappoint as pm  # noqa: E402
from tools import mappoint_scenes as ms  # noqa: E402


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    from se2lam_b200 import _capi, mappoint
    from se2lam_b200._capi import KP_DTYPE, ptr
    if not torch.cuda.is_available():
        sys.exit("no CUDA device: the timing needs the GPU")
    lib = _capi.lib()

    def dev(x):
        x = np.ascontiguousarray(x)
        return torch.from_numpy(x.view(np.uint8).reshape(len(x), -1) if x.dtype == KP_DTYPE else x).cuda()

    res = {"card": card()}
    cases = [("add_1k", ms.scene(1000, seed=11, n_upd=(0.0, 1.0, 0.0)), "add"),
             ("add_64k", ms.scene(64000, seed=12, n_upd=(0.0, 1.0, 0.0)), "add"),
             ("update_measure_5k", ms.scene(5000, seed=13), "measure")]
    for name, sc, kind in cases:
        pristine_kf = {k: dev(v) for k, v in sc["kf"].items()}
        pristine_mp = {k: dev(v) for k, v in sc["mp"].items()}
        kf = {k: v.clone() for k, v in pristine_kf.items()}
        mp = {k: v.clone() for k, v in pristine_mp.items()}
        M = len(sc["mp"]["obs_ptr"]) - 1
        up, pos = dev(sc["upd_ptr"]), dev(sc["upd_pos"])
        pts = dev(np.arange(M, dtype=np.int32))
        ab = torch.zeros(M, dtype=torch.uint8, device="cuda"); st = torch.zeros(1, dtype=torch.int32, device="cuda")
        prm = mappoint.params(**sc["params"])
        k_s, p_s = mappoint.keyframes(kf), mappoint.points(mp)
        s = torch.cuda.current_stream()

        def call():
            if kind == "add":
                return lib.se2gpu_mp_add_observations_device(C.byref(k_s), C.byref(p_s), ptr(up), ptr(pos), C.byref(prm), ptr(ab),
                                                             ptr(st), C.c_void_p(s.cuda_stream))
            return lib.se2gpu_mp_update_measure_device(C.byref(k_s), C.byref(p_s), M, ptr(pts), ptr(st), C.c_void_p(s.cuda_stream))

        times = []
        for r in range(a.warmup + a.reps):
            for k in kf:
                kf[k].copy_(pristine_kf[k])
            for k in mp:
                mp[k].copy_(pristine_mp[k])
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(s)
            assert call() == 0, _capi.last_error()
            e1.record(s)
            torch.cuda.synchronize()
            assert int(st.item()) == 0
            if r >= a.warmup:
                times.append(e0.elapsed_time(e1) * 1e3)
        # the oracle on one core, same tables
        okf, omp = ms.copy_tables(sc)
        t0 = time.perf_counter()
        if kind == "add":
            pm.add_observations(okf, omp, sc["upd_ptr"], sc["upd_pos"], sc["params"])
        else:
            pm.update_measure(okf, omp, np.arange(M, dtype=np.int32))
        cpu_us = (time.perf_counter() - t0) * 1e6
        res[name] = {"points": M, "updates": int(sc["upd_ptr"][-1]) if kind == "add" else M,
                     "gpu_us_median": float(np.median(times)), "gpu_us_min": float(np.min(times)), "oracle_1core_us": cpu_us}
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        open(a.out, "w").write(line + "\n")


if __name__ == "__main__":
    main()
