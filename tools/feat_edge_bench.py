"""Times the feature-graph constraint (GlobalMapper::CreateFeatEdge, se2gpu_feat_edge): one keyframe pair and 64 pairs in
one call, 50 and 300 points per pair, both modes, through the host entry (copies included, host clock around a synchronous
call) and the device entry (CUDA events around the launch on resident buffers), against the CPU oracle on one core.

    python tools/feat_edge_bench.py [--reps 50] [--json out.json] [--dump-outputs DIR]

--dump-outputs writes, per mode and size, every output of the host entry (with the pose trace) and of the device entry, and
the host entry's outputs for 256 pairs per mode whose start poses vary in yaw.
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

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from oracle import pyfeat  # noqa: E402
from se2lam_b200 import _capi, featgraph  # noqa: E402
from tools import dump  # noqa: E402
from tools import featgraph_synth as S  # noqa: E402


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
    L = _capi.lib()
    p = _capi.ptr
    rows = []
    for mode in (0, 1):
        for P in (50, 300):
            for B in (1, 64):
                pairs = [S.scene(2000 + b, P, noise=0.3 if mode else 1.0, outlier_share=0.1 if mode else 0.0, outlier_size=(0.2, 0.4))
                         for b in range(B)]
                prm = featgraph.params(pairs[0]["Tbc"])
                for _ in range(3):
                    g = featgraph.UpdateFeatGraph(pairs, prm, mode=mode)
                t0 = time.perf_counter()
                for _ in range(a.reps):
                    g = featgraph.UpdateFeatGraph(pairs, prm, mode=mode)
                host_us = (time.perf_counter() - t0) / a.reps * 1e6
                cat = lambda k, dt, w: torch.from_numpy(np.ascontiguousarray(np.concatenate([np.asarray(q[k], dt).reshape(-1, w) for q in pairs]))).cuda()
                T0, T1 = cat("Tcw0", np.float32, 16), cat("Tcw1", np.float32, 16)
                xyz, z0, z1 = cat("xyz", np.float32, 3), cat("z0", np.float32, 3), cat("z1", np.float32, 3)
                o0, o1 = cat("info0", np.float64, 9), cat("info1", np.float64, 9)
                pp = torch.arange(0, (B + 1) * P, P, dtype=torch.int32).cuda()
                meas = torch.zeros(B * 16, dtype=torch.float32).cuda(); info = torch.zeros(B * 36, dtype=torch.float32).cuda()
                pts = torch.zeros(B * P * 3, dtype=torch.float64).cuda(); work = torch.zeros_like(pts)
                st = torch.zeros(B, dtype=torch.int32).cuda()
                s = torch.cuda.current_stream()

                def launch():
                    rc = L.se2gpu_feat_edge_device(B, mode, p(T0), p(T1), p(pp), p(xyz), p(z0), p(z1), p(o0), p(o1), C.addressof(prm),
                                                   p(meas), p(info), p(st), None, None, None, None, p(pts), p(work), C.c_void_p(s.cuda_stream))
                    assert rc == 0, _capi.last_error()

                for _ in range(3):
                    launch()
                ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
                ms = 0.0
                for _ in range(a.reps):
                    ev[0].record(s); launch(); ev[1].record(s)
                    ev[1].synchronize()
                    ms += ev[0].elapsed_time(ev[1])
                dev_us = ms / a.reps * 1e3
                if a.dump_outputs:
                    tag = f"feat_m{mode}_P{P}_B{B}"
                    dump.save(a.dump_outputs, tag, featgraph.UpdateFeatGraph(pairs, prm, mode=mode, trace=True))
                    dump.save(a.dump_outputs, tag + "_device", dict(measure=meas.cpu().numpy(), info=info.cpu().numpy(),
                                                                    status=st.cpu().numpy(), points=pts.cpu().numpy()))
                assert meas.cpu().numpy().tobytes() == np.concatenate([r["measure"].ravel() for r in g]).tobytes()
                oprm = pyfeat.params(Tbc=pairs[0]["Tbc"])
                n_cpu = min(B, 8)
                run = lambda q: pyfeat.run(mode, q["Tcw0"], q["Tcw1"], q["xyz"], q["z0"], q["z1"], q["info0"], q["info1"], oprm)
                run(pairs[0])
                cpu_reps = max(1, 16 // n_cpu)
                t0 = time.perf_counter()
                for _ in range(cpu_reps):
                    for q in pairs[:n_cpu]:
                        run(q)
                cpu_us = (time.perf_counter() - t0) / (n_cpu * cpu_reps) * 1e6 * B
                rows.append(dict(mode=mode, points=P, batch=B, mean_iterations=float(np.mean([r["iterations"] for r in g])),
                                 mean_trials=float(np.mean([r["stats"]["trials"].sum() for r in g])),
                                 host_entry_us=round(host_us, 1), device_entry_us=round(dev_us, 1),
                                 device_us_per_pair=round(dev_us / B, 2), cpu_oracle_us=round(cpu_us, 1),
                                 cpu_oracle_us_per_pair=round(cpu_us / B, 1)))
                print(json.dumps(rows[-1]), flush=True)
    if a.dump_outputs:
        # 256 pairs per mode with start poses at every yaw, so the dump covers general start rotations, not one
        rng = np.random.default_rng(7)
        for mode in (0, 1):
            pairs = [S.scene(3000 + b, 60, start=(rng.uniform(-5, 5), rng.uniform(-5, 5), rng.uniform(-np.pi, np.pi)),
                             motion=(rng.uniform(0.1, 0.6), rng.uniform(-0.1, 0.1), rng.uniform(-0.3, 0.3)),
                             noise=0.3 if mode else 1.0, outlier_share=0.1 if mode else 0.0, outlier_size=(0.2, 0.4)) for b in range(256)]
            dump.save(a.dump_outputs, f"feat_m{mode}_varied", featgraph.UpdateFeatGraph(pairs, featgraph.params(pairs[0]["Tbc"]), mode=mode,
                                                                                          trace=True))
    res = dict(gpu=gpu_info(), cpu_oracle="one core, g++ -O2 -ffp-contract=off, ctypes call included", reps=a.reps, rows=rows)
    print(json.dumps(res))
    if a.json:
        os.makedirs(os.path.dirname(os.path.abspath(a.json)), exist_ok=True)
        with open(a.json, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
