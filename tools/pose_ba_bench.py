"""Times the pose-only BA (Localizer::DoLocalBA): one problem of 300 and of 1000 edges and 64 such problems in one call,
30 LM iterations each, through the host entry (copies included, host clock around a synchronous call) and the device entry
(CUDA events around the launch on resident buffers), against the CPU oracle on one core.

    python tools/pose_ba_bench.py [--reps 50] [--json out.json] [--dump-outputs DIR]

--dump-outputs writes, per size, every output of the host entry (with the pose trace) and the device entry's poses.
"""
from __future__ import annotations

import argparse
import json
import math
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from oracle import pypose  # noqa: E402
from se2lam_b200 import pose as pba  # noqa: E402
from tools import dump  # noqa: E402
from tools import pose_synth as ps  # noqa: E402

DELTA = math.sqrt(5.991)


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        return out.splitlines()[0] if out else "unknown"
    except Exception as e:  # noqa: BLE001
        return f"unknown ({e})"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--json", default=None)
    ap.add_argument("--dump-outputs", metavar="DIR", help="write the outputs of the last run of each size as DIR/<tag>_<name>.npy")
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this benchmark measures the GPU and has no CPU fallback")
    prm = pba.params(ps.FX, ps.CX, ps.CY, ps.Tbc_f32(), DELTA, iterations=30)
    rows = []
    for E in (300, 1000):
        for B in (1, 64):
            probs = [ps.make_problem(E=E, seed=1000 + b, outliers=0.1) for b in range(B)]
            T, ptr, x, u, w = ps.batch(probs)
            for _ in range(3):
                g = pba.poseOnlyBA(T, ptr, x, u, w, prm)
            t0 = time.perf_counter()
            for _ in range(a.reps):
                g = pba.poseOnlyBA(T, ptr, x, u, w, prm)
            host_us = (time.perf_counter() - t0) / a.reps * 1e6
            dev = lambda arr: torch.from_numpy(np.ascontiguousarray(arr)).cuda()
            dT0, dp, dx, du, dw = dev(T), dev(ptr), dev(x), dev(u), dev(w)
            dT = dT0.clone()
            s = torch.cuda.current_stream()
            for _ in range(3):
                dT.copy_(dT0); pba.poseOnlyBADevice(B, dT, dp, dx, du, dw, prm, stream=s.cuda_stream)
            ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
            ms = 0.0
            for _ in range(a.reps):
                dT.copy_(dT0)
                ev[0].record(s); pba.poseOnlyBADevice(B, dT, dp, dx, du, dw, prm, stream=s.cuda_stream); ev[1].record(s)
                ev[1].synchronize()
                ms += ev[0].elapsed_time(ev[1])
            dev_us = ms / a.reps * 1e3
            if a.dump_outputs:
                tag = f"pose_E{E}_B{B}"
                dump.save(a.dump_outputs, tag, pba.poseOnlyBA(T, ptr, x, u, w, prm, trace=True))
                dump.save(a.dump_outputs, tag + "_device", dict(Tcw=dT.cpu().numpy()))
            n_cpu = max(1, min(B, 8))
            pypose.run(probs[0]["Tcw"], probs[0]["xyz"], probs[0]["uv"], probs[0]["info"], ps.FX, ps.CX, ps.CY, ps.Tbc_f32(), DELTA)
            cpu_reps = max(1, 16 // n_cpu)
            t0 = time.perf_counter()
            for _ in range(cpu_reps):
                for p in probs[:n_cpu]:
                    pypose.run(p["Tcw"], p["xyz"], p["uv"], p["info"], ps.FX, ps.CX, ps.CY, ps.Tbc_f32(), DELTA, iterations=30)
            cpu_us = (time.perf_counter() - t0) / (n_cpu * cpu_reps) * 1e6 * B
            its = float(np.mean(g["iterations"]))
            rows.append(dict(edges=E, batch=B, mean_iterations=its, host_entry_us=round(host_us, 1), device_entry_us=round(dev_us, 1),
                             device_us_per_problem=round(dev_us / B, 2), cpu_oracle_us=round(cpu_us, 1),
                             cpu_oracle_us_per_problem=round(cpu_us / B, 1)))
            print(json.dumps(rows[-1]), flush=True)
    res = dict(gpu=gpu_info(), cpu_oracle="one core, g++ -O2 -ffp-contract=off", iterations=30, rows=rows)
    print(json.dumps(res))
    if a.json:
        os.makedirs(os.path.dirname(os.path.abspath(a.json)), exist_ok=True)
        with open(a.json, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
