"""Cost of GlobalMapper::GlobalBA on the GPU (se2gpu_global_ba) against the CPU oracle on one core.

Graphs: circles driven several times (tools/posegraph_synth.py), odometry plus feature edges 2..5 hops apart (about 4 per
keyframe) plus loop closures, 15 LM iterations. Per size: the host entry (uploads, plan, kernel, downloads), the device
entry on device-resident values (plan upload and kernel), launches per call, the kernel's time per phase
(se2gpu_global_ba_profile, in a separate run), and the CPU oracle. Prints one JSON line per
size with the card's name and power limit. --dump-outputs DIR writes, per size, every output of the host entry and the
device entry's poses."""
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

from oracle import pyglobal  # noqa: E402
from se2lam_b200 import _capi, globalba  # noqa: E402
from tools import dump  # noqa: E402
from tools import posegraph_synth as S  # noqa: E402


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return out.stdout.strip().splitlines()[0] if out.returncode == 0 else "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="100,500,2000,5000")
    ap.add_argument("--runs", type=int, default=10)
    ap.add_argument("--oracle-runs", type=int, default=1)
    ap.add_argument("--dump-outputs", metavar="DIR", help="write the outputs of the last run of each size as DIR/<tag>_<name>.npy")
    a = ap.parse_args()
    import torch
    name = card()
    ctx = globalba.Context(0)
    for N in [int(s) for s in a.sizes.split(",")]:
        g = S.graph(seed=N, N=N, kind="revisit", laps=max(1, N // 500))
        prm = globalba.params(g["Tbc"])
        ctx.run(g["Tcw"], g["fixed"], g["edges"], prm)  # warm-up: grows the context's buffers
        t = time.perf_counter()
        for _ in range(a.runs):
            r = ctx.run(g["Tcw"], g["fixed"], g["edges"], prm)
        host_ms = (time.perf_counter() - t) / a.runs * 1e3
        fr, to, me, inf = globalba.edge_arrays(g["edges"])
        dT = torch.from_numpy(np.ascontiguousarray(g["Tcw"].reshape(N, 16))).cuda()
        dm, di = torch.from_numpy(me).cuda(), torch.from_numpy(inf).cuda()
        out = torch.zeros((N, 16), dtype=torch.float32, device="cuda")
        fx = np.ascontiguousarray(g["fixed"], np.uint8)
        stream = torch.cuda.current_stream().cuda_stream
        L = _capi.lib()
        call = lambda: _capi.check(L.se2gpu_global_ba_device(ctx.h, N, _capi.ptr(dT), _capi.ptr(fx), len(fr), _capi.ptr(fr), _capi.ptr(to),
                                                             _capi.ptr(dm), _capi.ptr(di), None, C.addressof(prm), _capi.ptr(out), None,
                                                             None, None, None, stream), "se2gpu_global_ba_device")
        call(); torch.cuda.synchronize()
        l0 = L.se2gpu_launch_count()
        t = time.perf_counter()
        for _ in range(a.runs):
            call()
        torch.cuda.synchronize()
        dev_ms = (time.perf_counter() - t) / a.runs * 1e3
        launches = (L.se2gpu_launch_count() - l0) / a.runs
        if a.dump_outputs:
            dump.save(a.dump_outputs, f"global_N{N}", r)
            dump.save(a.dump_outputs, f"global_N{N}_device", dict(Tcw=out.cpu().numpy()))
        # the phase split, in a run of its own (the timer reads are not in the timed runs above)
        _capi.check(L.se2gpu_global_ba_profile(ctx.h, 1), "se2gpu_global_ba_profile")
        ctx.run(g["Tcw"], g["fixed"], g["edges"], prm)
        ms = (C.c_double * 7)()
        _capi.check(L.se2gpu_global_ba_profile_read(ctx.h, ms), "se2gpu_global_ba_profile_read")
        _capi.check(L.se2gpu_global_ba_profile(ctx.h, 0), "se2gpu_global_ba_profile")
        phases = dict(zip(("setup", "linearise", "gather", "damp", "factor", "substitute", "trial"), (round(v, 3) for v in ms)))
        t = time.perf_counter()
        for _ in range(a.oracle_runs):
            pyglobal.run(g, pyglobal.params(g["Tbc"]))
        cpu_ms = (time.perf_counter() - t) / a.oracle_runs * 1e3
        print(json.dumps(dict(card=name, N=N, E=len(g["edges"]), iterations=r["iterations"], host_entry_ms=round(host_ms, 3),
                              device_entry_ms=round(dev_ms, 3), launches_per_call=launches, phase_ms=phases, cpu_oracle_ms=round(cpu_ms, 1))), flush=True)
    ctx.close()


if __name__ == "__main__":
    main()
