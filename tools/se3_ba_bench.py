"""Times the SE(3)-XYZ window BA (se2gpu_se3_ba, loadLocalGraphOnlyBa's graph) next to the SE(2)-XYZ local BA (se2gpu_ba) on
the same lifted window: the TIME_TO_LOG_LOCAL_BA comparison. Prints one JSON line per window, with the GPU name and power
limit: the median wall time over --runs calls (each ends in a synchronise) of the SE(3) host entry on one context and of
the SE(2) BA's set_problem + optimize, the SE(2) optimize alone, the k_se3_ba kernel's own time (torch.profiler, one
profiled call of its own, so the rest of the host entry is planning and copies), and the CPU oracle on one core."""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import numpy as np  # noqa: E402

from oracle import pyse3ba  # noqa: E402
from se2lam_b200 import se3ba  # noqa: E402
from se2lam_b200.ba import LocalBA  # noqa: E402
from tools import se3_window_synth as S  # noqa: E402

WINDOWS = {"20kf": (20, 2000), "C4": (50, 5000)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=10)
    ap.add_argument("--iterations", type=int, default=10)
    a = ap.parse_args()
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip()
    ctx = se3ba.Context()
    for name, (n_kf, n_lm) in WINDOWS.items():
        prob, w = S.window(n_kf, n_lm, seed=9, with_prior=False, odometry=False)
        prm = S.window_params(prob, iterations=a.iterations)
        ctx.run(w, prm)
        t3 = []
        for _ in range(a.runs):
            t = time.perf_counter(); r = ctx.run(w, prm); t3.append(time.perf_counter() - t)
        ba = LocalBA.from_problem(prob, device=0)
        ba.optimize(a.iterations)
        t2, t2o = [], []
        for _ in range(a.runs):
            t = time.perf_counter()
            ba = LocalBA.from_problem(prob, device=0)
            t1 = time.perf_counter(); ba.optimize(a.iterations); t2o.append(time.perf_counter() - t1); t2.append(time.perf_counter() - t)
        import torch
        from torch.profiler import ProfilerActivity, profile
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            ctx.run(w, prm)
            torch.cuda.synchronize()
        kern = sum(getattr(e, "device_time_total", None) or e.cuda_time_total for e in prof.key_averages() if "k_se3_ba" in e.key) / 1e3
        t = time.perf_counter(); pyse3ba.run(w, prm); cpu = time.perf_counter() - t
        print(json.dumps(dict(window=name, keyframes=n_kf, points=len(w.xyz), edges=len(w.edge_point), iterations=r["iterations"],
                              se3_host_entry_ms=1e3 * float(np.median(t3)), se3_kernel_ms=kern,
                              se2_set_problem_and_optimize_ms=1e3 * float(np.median(t2)), se2_optimize_ms=1e3 * float(np.median(t2o)),
                              cpu_oracle_ms=1e3 * cpu, gpu=gpu)))
    ctx.close()


if __name__ == "__main__":
    main()
