"""Times Track::removeOutliers on the GPU (se2gpu_remove_outliers_device) and on one host core (the oracle).

For one frame pair of 1000 matches and for 64 such pairs in one call, at 10 %, 30 % and 50 % outliers: the median of
--runs launches, each timed with CUDA events on the launching stream (matches12 is restored before each launch, outside
the timed window), next to the oracle's median wall time per pair. Prints one JSON line with the GPU's name and power limit.

    python tools/fundam_bench.py [--runs 200]
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

from oracle import pin_fundam_against_cv2 as scenes_mod  # noqa: E402
from oracle import pyfundam  # noqa: E402
from se2lam_b200 import _capi  # noqa: E402
from se2lam_b200._capi import KP_DTYPE  # noqa: E402
from tests.fundam_cases import Scene  # noqa: E402


def frame_pairs(B, n, outliers, seed):
    rng = np.random.default_rng(seed)
    out = []
    for b in range(B):
        p = scenes_mod.two_view(rng, n, outliers)
        s = Scene(b, 0, p, True, None, None, 0)
        out.append(s.keypoints(KP_DTYPE, rng))
    return out


def gpu_case(torch, pairs, runs):
    B = len(pairs)
    cap1 = max(len(p[0]) for p in pairs); cap2 = max(len(p[1]) for p in pairs)
    k1 = np.zeros((B, cap1), KP_DTYPE); k2 = np.zeros((B, cap2), KP_DTYPE); m = np.full((B, cap1), -1, np.int32)
    n1 = np.array([len(p[0]) for p in pairs], np.int32); n2 = np.array([len(p[1]) for p in pairs], np.int32)
    for b, (a, c, mm) in enumerate(pairs):
        k1[b, :len(a)] = a; k2[b, :len(c)] = c; m[b, :len(mm)] = mm
    dev = torch.device("cuda:0")
    dk1 = torch.from_numpy(k1.view(np.uint8)).to(dev); dk2 = torch.from_numpy(k2.view(np.uint8)).to(dev)
    dn1 = torch.from_numpy(n1).to(dev); dn2 = torch.from_numpy(n2).to(dev)
    m0 = torch.from_numpy(m).to(dev); dm = m0.clone()
    dnin = torch.zeros(B, dtype=torch.int32, device=dev); dit = torch.zeros(B, dtype=torch.int32, device=dev)
    stream = torch.cuda.current_stream(dev)
    L, p = _capi.lib(), _capi.ptr

    def call():
        _capi.check(L.se2gpu_remove_outliers_device(B, p(dk1), p(dn1), cap1, p(dk2), p(dn2), cap2, p(dm), p(dnin), None, p(dit),
                                                    C.c_void_p(stream.cuda_stream)), "se2gpu_remove_outliers_device")
    for _ in range(5):
        dm.copy_(m0); call()
    times = []
    for _ in range(runs):
        dm.copy_(m0)
        e0 = torch.cuda.Event(enable_timing=True); e1 = torch.cuda.Event(enable_timing=True)
        e0.record(stream); call(); e1.record(stream)
        e1.synchronize()
        times.append(e0.elapsed_time(e1))
    it = dit.cpu().numpy()
    return float(np.median(times)), int(np.median(it)), int(it.max())


def oracle_case(pairs, runs):
    times = []
    for r in range(runs):
        k1, k2, m = pairs[r % len(pairs)]
        t0 = time.perf_counter(); pyfundam.remove_outliers(k1, k2, m); times.append((time.perf_counter() - t0) * 1e3)
    return float(np.median(times))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=200)
    ap.add_argument("--matches", type=int, default=1000)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this benchmark measures the GPU")
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    res = {"metric": "remove_outliers_ms", "gpu": q.stdout.strip(), "matches": args.matches, "runs": args.runs, "cases": []}
    for outl in (0.1, 0.3, 0.5):
        pairs = frame_pairs(64, args.matches, outl, seed=int(outl * 100))
        g1, it1, _ = gpu_case(torch, pairs[:1], args.runs)
        g64, it64, itmax = gpu_case(torch, pairs, args.runs)
        host = oracle_case(pairs, min(args.runs, 64))
        res["cases"].append({"outliers": outl, "gpu_1pair_ms": round(g1, 4), "gpu_64pairs_ms": round(g64, 4),
                             "oracle_1pair_ms_one_core": round(host, 4), "hypotheses_median": it64, "hypotheses_max": itmax,
                             "hypotheses_1pair": it1})
    print(json.dumps(res))


if __name__ == "__main__":
    main()
