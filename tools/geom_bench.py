"""Times se2gpu_track_triangulate_device and se2gpu_projection_observations_device (CUDA events on the launching stream)
and the oracle port on one host core, for one frame of about 1000 matches and for 64 such frames in one call. Prints one
JSON line with the card's name and power limit read in the same run; fails without a GPU.

    python tools/geom_bench.py [--reps 200]
"""
from __future__ import annotations

import argparse
import ctypes
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

from oracle import pygeom  # noqa: E402
from se2lam_b200 import _capi  # noqa: E402
from se2lam_b200._capi import check, ptr  # noqa: E402
from tools import geom_scenes as gs  # noqa: E402


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a).view(np.uint8).reshape(-1).copy()).cuda()


def gpu_ms(fn, reps, stream):
    for _ in range(10):
        fn()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    times = []
    for _ in range(reps):
        a.record(stream); fn(); b.record(stream)
        b.synchronize()
        times.append(a.elapsed_time(b))
    return float(np.median(times))


def cpu_ms(fn, reps, reset=None):
    """Median wall time of fn() alone; reset() (restoring in-place outputs) runs outside the timed region."""
    times = []
    for _ in range(reps):
        if reset:
            reset()
        t = time.perf_counter(); fn(); times.append((time.perf_counter() - t) * 1e3)
    return float(np.median(times))


def oracle_calls(t, p):
    """The oracle's C++ loops called directly through ctypes on prepared buffers: no Python-side copies in the timed call."""
    L = pygeom.lib()
    c = np.ascontiguousarray
    P = lambda a: a.ctypes.data_as(ctypes.c_void_p)  # noqa: E731
    n = len(t["kp_kf"])
    kf, fr, obs, vm = c(t["kp_kf"]), c(t["kp_frame"]), c(t["kf_observed"], np.uint8), c(t["kf_view_mp"], np.float32)
    Tcr, K = c(t["Tcr"], np.float32), c(t["K"], np.float32)
    m0, lm0 = c(t["matches12"], np.int32), c(t["local_mps"], np.float32)
    m, lm, good, cnt = m0.copy(), lm0.copy(), np.zeros(n, np.uint8), np.zeros(2, np.int32)

    def track_reset():
        m[:] = m0; lm[:] = lm0

    def track():
        L.geom_oracle_track_triangulate(P(kf), n, P(fr), P(m), P(obs), P(vm), P(Tcr), P(K), 0.1, 10.0, 2, P(lm), P(good), P(cnt))
    mp = p["mp"]
    nk = len(p["kf_kp"])
    a = [c(p["kf_kp"]), c(p["matches_idx_mp"], np.int32), c(p["Tcw_new"], np.float32), c(mp["main_measure"], np.float32),
         c(mp["main_pose"], np.int32), c(mp["main_octave"], np.int32), c(mp["normal"], np.float32), c(mp["min_dist"], np.float32),
         c(mp["max_dist"], np.float32), c(p["Tcw_table"], np.float32), c(p["K"], np.float32)]
    acc, pos, info = np.zeros(nk, np.uint8), np.zeros((nk, 3), np.float32), np.zeros((nk, 3, 3))

    def proj():
        L.geom_oracle_projection_observations(nk, *[P(x) for x in a], 0.1, 10.0, float(p["fx"]), P(acc), P(pos), P(info))
    return track, track_reset, proj


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=200)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("geom_bench: no CUDA device")
    os.environ.setdefault("OMP_NUM_THREADS", "1")
    lib = _capi.lib()
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    name, power = [x.strip() for x in smi.stdout.splitlines()[0].split(",")] if smi.returncode == 0 else (torch.cuda.get_device_name(0), "unknown")
    s = torch.cuda.Stream()
    sp = s.cuda_stream
    out = dict(tool="geom_bench", gpu=name, power_limit=power, reps=args.reps)
    for label, n in (("1x1000", 1000), ("64x1000", 64000)):
        t = gs.track_scene(n, seed=1)
        d = {k: dev(t[k]) for k in ("kp_kf", "kp_frame", "kf_observed", "kf_view_mp", "Tcr", "K", "local_mps")}
        m0 = dev(t["matches12"])
        d_m = m0.clone(); d_good = torch.zeros(n, dtype=torch.uint8, device="cuda"); d_cnt = torch.zeros(2, dtype=torch.int32, device="cuda")

        def track():
            d_m.copy_(m0)
            check(lib.se2gpu_track_triangulate_device(ptr(d["kp_kf"]), n, None, ptr(d["kp_frame"]), ptr(d_m), ptr(d["kf_observed"]),
                                                      ptr(d["kf_view_mp"]), ptr(d["Tcr"]), ptr(d["K"]), 0.1, 10.0, 2, ptr(d["local_mps"]),
                                                      ptr(d_good), ptr(d_cnt), sp), "track_triangulate")
        with torch.cuda.stream(s):
            out[f"track_triangulate_{label}_gpu_ms"] = gpu_ms(track, args.reps, s)
        p = gs.projection_scene(n, n_mp=min(n, 4000), seed=2)
        mp = p["mp"]
        g = [dev(x) for x in (p["Tcw_new"], mp["main_measure"], mp["main_pose"], mp["main_octave"], mp["normal"], mp["min_dist"],
                              mp["max_dist"], p["Tcw_table"], p["K"])]
        d_kp, d_mi = dev(p["kf_kp"]), dev(p["matches_idx_mp"])
        d_acc = torch.zeros(n, dtype=torch.uint8, device="cuda"); d_pos = torch.zeros(3 * n, dtype=torch.float32, device="cuda")
        d_info = torch.zeros(9 * n, dtype=torch.float64, device="cuda")

        def proj():
            check(lib.se2gpu_projection_observations_device(ptr(d_kp), n, None, ptr(d_mi), *[ptr(x) for x in g], 0.1, 10.0, float(p["fx"]),
                                                            ptr(d_acc), ptr(d_pos), ptr(d_info), sp), "projection_observations")
        with torch.cuda.stream(s):
            out[f"projection_observations_{label}_gpu_ms"] = gpu_ms(proj, args.reps, s)
        torch.cuda.synchronize()
        creps = 20 if n <= 1000 else 3
        track_c, track_reset, proj_c = oracle_calls(t, p)
        out[f"track_triangulate_{label}_cpu1_ms"] = cpu_ms(track_c, creps, track_reset)
        out[f"projection_observations_{label}_cpu1_ms"] = cpu_ms(proj_c, creps)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
