"""Local-BA window load: host inputs through se2gpu_ba_set_problem against the same inputs already on the device through
se2gpu_ba_set_problem_device.

Each size slides a window along one seeded trajectory, so every load has a new topology (what LocalMapper::localBA does once
per keyframe). Per window: a host clock around each load (both end in a stream synchronise), around load + optimize(10),
and around the same-topology values-only refresh. The two paths alternate window by window in one process, after a warm-up.
Prints the card and its power limit first, then one JSON line per size. With --phases the device path runs again with
SE2GPU_BA_DEBUG=1 and its per-phase split goes to stderr.

    python tools/ba_load_bench.py [--windows 12] [--sizes small,c4,c5] [--phases]
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

from se2lam_b200.ba import LocalBA  # noqa: E402
from tools import synth  # noqa: E402

FIELDS = ("poses", "fixed", "points", "edge_pose", "edge_point", "uv", "info", "odo_i", "odo_j", "odo_meas", "odo_info")
DTYPES = (torch.float64, torch.uint8, torch.float64, torch.int32, torch.int32, torch.float64, torch.float64, torch.int32,
          torch.int32, torch.float64, torch.float64)
# (keyframes per window, landmarks per window, trajectory keyframes, trajectory landmarks): 6 observations per landmark
SIZES = {"small": (20, 1500), "c4": (50, 5000), "c5": (2000, 50000)}


def windows(size, count, seed=7):
    """`count` windows of `size` keyframes sliding along one trajectory, one keyframe apart, first keyframe fixed"""
    kf, lm = SIZES[size]
    step = 1
    traj = synth.ba_window(kf + step * count, int(lm * (kf + step * count) / kf), seed=seed,
                           layout="zigzag" if kf > 500 else "circle")
    from tests.test_ba_context_gpu import slide
    return [slide(traj, k * step, kf) for k in range(count)]


def on_device(prob):
    out = []
    for f, dt in zip(FIELDS, DTYPES):
        a = np.ascontiguousarray(getattr(prob, f)).reshape(-1)
        out.append((torch.from_numpy(a.copy()).to(dt) if a.size else torch.zeros(1, dtype=dt)).cuda())
    return out


def load_device(ba, prob, t):
    ba.set_problem_device(prob.P, prob.L, prob.E, prob.O, *t, prob.fx, prob.cx, prob.cy, prob.Tcb, prob.huber_delta)


def timed(fn):
    t0 = time.perf_counter()
    fn()
    return (time.perf_counter() - t0) * 1e3


def bench(size, count):
    ws = windows(size, count + 2)
    caps = (max(w.P for w in ws), max(w.L for w in ws), max(w.E for w in ws), max(w.O for w in ws))
    dev = [on_device(w) for w in ws]
    torch.cuda.synchronize()
    host_ba, dev_ba = LocalBA(*caps), LocalBA(*caps)
    for k in range(2):                                   # warm-up: both paths, every kernel shape once
        host_ba.set_problem(ws[k]); load_device(dev_ba, ws[k], dev[k])
        host_ba.optimize(10); dev_ba.optimize(10)
    r = {k: [] for k in ("host_load", "device_load", "host_load_opt", "device_load_opt", "host_refresh", "device_refresh")}
    for k in range(2, count + 2):
        w, t = ws[k], dev[k]
        order = (("host", lambda: host_ba.set_problem(w)), ("device", lambda: load_device(dev_ba, w, t)))
        for name, fn in (order if k % 2 else order[::-1]):
            r[name + "_load"].append(timed(fn))
        for name, fn, ba in (("host", lambda: host_ba.set_problem(w), host_ba), ("device", lambda: load_device(dev_ba, w, t), dev_ba)):
            r[name + "_refresh"].append(timed(fn))       # same topology as just loaded: values only
        for name, fn, ba in (("host", lambda: host_ba.set_problem(ws[k - 1]), host_ba),
                             ("device", lambda: load_device(dev_ba, ws[k - 1], dev[k - 1]), dev_ba)):
            r[name + "_load_opt"].append(timed(lambda: (fn(), ba.optimize(10))))
    w = ws[-1]
    blocks = dev_ba.debug_plan()["nblk"]
    out = {"size": size, "P": w.P, "L": w.L, "E": w.E, "O": w.O, "blocks": blocks,
           "pairs": int(len(dev_ba.debug_structure("pair_e1"))), "windows": count}
    for k, v in r.items():
        out[k + "_ms_median"] = round(float(np.median(v)), 3)
        out[k + "_ms_min"] = round(float(np.min(v)), 3)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--windows", type=int, default=12)
    ap.add_argument("--sizes", default="small,c4,c5")
    ap.add_argument("--phases", action="store_true", help="rerun the device path with SE2GPU_BA_DEBUG=1 (per-phase split on stderr)")
    ap.add_argument("--_phase_run", action="store_true", help=argparse.SUPPRESS)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("ba_load_bench needs a CUDA device")
    if a._phase_run:
        for size in a.sizes.split(","):
            ws = windows(size, 4)
            caps = (max(w.P for w in ws), max(w.L for w in ws), max(w.E for w in ws), max(w.O for w in ws))
            ba = LocalBA(*caps)
            for w in ws:
                load_device(ba, w, on_device(w))
        return
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    print(json.dumps({"gpu": torch.cuda.get_device_name(0), "nvidia_smi": smi}), flush=True)
    for size in a.sizes.split(","):
        print(json.dumps(bench(size, a.windows)), flush=True)
    if a.phases:
        env = dict(os.environ, SE2GPU_BA_DEBUG="1")
        subprocess.run([sys.executable, __file__, "--_phase_run", "--sizes", a.sizes], env=env, check=True)


if __name__ == "__main__":
    main()
