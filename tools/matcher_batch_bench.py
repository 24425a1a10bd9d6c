"""Times MatchByWindow on B frame pairs: B single-pair calls (se2gpu_match_by_window_device) on one stream against one batched
call (se2gpu_match_by_window_batch_device), for B in 1, 8, 64.

The frames are bench.py's matcher workload (matcher_frames: 8 pairs of the ORB benchmark texture, 640x480, 1000 keypoints
per frame, extracted on the device); pair b of a batch is pair b % 8 of it. Every repetition restores vbPrevMatched outside
the timed window, and is timed with CUDA events on the launching stream; the result is the median of --runs repetitions
after --warmup untimed ones. The run also checks that both ways give the same bytes (matches, vbPrevMatched, match counts)
and counts the kernel launches per call. Prints one JSON line with the GPU's name and power limit. --profile DIR writes a
torch.profiler trace of one repetition of each way at the largest B (a separate run: tracing slows the host).

    python tools/matcher_batch_bench.py [--runs 50] [--warmup 5] [--batches 1 8 64] [--profile DIR]
"""
from __future__ import annotations

import argparse
import json
import os
import re
import subprocess
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from bench import NFEAT, H, W, matcher_frames  # noqa: E402
from se2lam_b200 import _capi  # noqa: E402
from se2lam_b200.matcher import FrameView, ORBmatcher  # noqa: E402
from se2lam_b200.orb import ORBextractor  # noqa: E402

WIN, RATIO = 20, 0.9


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--batches", type=int, nargs="+", default=[1, 8, 64])
    ap.add_argument("--profile", metavar="DIR")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this benchmark measures the GPU")
    dev = torch.device("cuda:0")
    stream = torch.cuda.current_stream(dev)
    sptr = stream.cuda_stream
    lib = _capi.lib()

    # bench.py's matcher frames, extracted on the device: frame 2p is pair p's reference frame, 2p + 1 its current frame
    imgs = matcher_frames()
    npair = len(imgs) // 2
    ext = ORBextractor(NFEAT, 1.2, 8, max_batch=len(imgs))
    d_imgs = torch.from_numpy(imgs).to(dev)
    kps = torch.zeros((len(imgs), NFEAT * 28), dtype=torch.uint8, device=dev)
    desc = torch.zeros((len(imgs), NFEAT * 32), dtype=torch.uint8, device=dev)
    counts = torch.zeros(len(imgs), dtype=torch.int32, device=dev)
    ext.extract_device(d_imgs, len(imgs), H, W, kps, desc, counts, stream=sptr)
    grid = FrameView(None, None).grid()
    Bmax = max(args.batches)
    single = ORBmatcher(RATIO, max_queries=NFEAT, max_db=NFEAT)
    batched = ORBmatcher(RATIO, max_queries=NFEAT, max_db=NFEAT, max_batch=Bmax)

    res = {"tool": "matcher_batch_bench", "gpu": gpu_info(), "workload": f"MatchByWindow, bench.py's {npair} frame pairs "
           f"(640x480, {NFEAT} keypoints per frame, window {WIN}, ratio {RATIO}), pair b = pair b % {npair}",
           "runs": args.runs, "warmup": args.warmup, "cases": []}
    for B in args.batches:
        ref, cur = torch.arange(B, device=dev) % npair * 2, torch.arange(B, device=dev) % npair * 2 + 1
        kp1, kp2, de1, de2 = kps[ref].contiguous(), kps[cur].contiguous(), desc[ref].contiguous(), desc[cur].contiguous()
        n1, n2 = counts[ref].contiguous(), counts[cur].contiguous()
        prev0 = kp1.view(torch.float32).view(B, NFEAT, 7)[:, :, :2].contiguous()
        out = {w: (prev0.clone(), torch.full((B, NFEAT), 7, dtype=torch.int32, device=dev), torch.zeros(B, dtype=torch.int32, device=dev))
               for w in ("single", "batch")}

        # device addresses resolved once, outside the timed window: the host work per call is the library's alone
        def addr(t, b, n):
            return t.data_ptr() + b * n * t.element_size()
        single_args = [(addr(kp1, b, NFEAT * 28), addr(de1, b, NFEAT * 32), addr(kp2, b, NFEAT * 28), addr(de2, b, NFEAT * 32),
                        addr(out["single"][0], b, NFEAT * 2), addr(out["single"][1], b, NFEAT), addr(out["single"][2], b, 1),
                        addr(n1, b, 1), addr(n2, b, 1)) for b in range(B)]
        batch_args = [t.data_ptr() for t in (kp1, de1, kp2, de2, *out["batch"], n1, n2)]

        def run_single():
            for k1, d1, k2, d2, prev, m, nm, c1, c2 in single_args:
                single.MatchByWindowDevice(k1, d1, NFEAT, k2, d2, NFEAT, prev, grid, WIN, m, nm, d_n1=c1, d_n2=c2, stream=sptr)

        def run_batch():
            k1, d1, k2, d2, prev, m, nm, c1, c2 = batch_args
            batched.MatchByWindowBatchDevice(B, k1, d1, NFEAT, k2, d2, NFEAT, prev, grid, WIN, m, nm, d_n1=c1, d_n2=c2, stream=sptr)

        case = {"B": B}
        for way, fn in (("single", run_single), ("batch", run_batch)):
            prev = out[way][0]
            for _ in range(args.warmup):
                prev.copy_(prev0); fn()
            torch.cuda.synchronize()
            times = []
            for r in range(args.runs):
                prev.copy_(prev0)
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record(stream)
                l0 = lib.se2gpu_launch_count()
                fn()
                launches = lib.se2gpu_launch_count() - l0
                e1.record(stream)
                e1.synchronize()
                times.append(e0.elapsed_time(e1))
            ms = float(np.median(times))
            case[way] = {"us_per_call": round(ms * 1e3, 2), "us_per_pair": round(ms * 1e3 / B, 2), "pairs_per_s": round(B / (ms * 1e-3)),
                         "launches_for_B_pairs": launches, "spread_us": [round(float(np.percentile(times, 10)) * 1e3, 2),
                                                                      round(float(np.percentile(times, 90)) * 1e3, 2)]}
        torch.cuda.synchronize()
        case["identical"] = all(out["single"][k].cpu().numpy().tobytes() == out["batch"][k].cpu().numpy().tobytes() for k in range(3))
        case["speedup_per_pair"] = round(case["single"]["us_per_pair"] / case["batch"]["us_per_pair"], 2)
        case["matches_per_pair"] = float(out["batch"][2].float().mean().item())
        res["cases"].append(case)

        if args.profile and B == Bmax:
            from torch.profiler import ProfilerActivity, profile
            os.makedirs(args.profile, exist_ok=True)
            for way, fn in (("single", run_single), ("batch", run_batch)):
                out[way][0].copy_(prev0)
                torch.cuda.synchronize()
                with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
                    fn()
                    torch.cuda.synchronize()
                prof.export_chrome_trace(os.path.join(args.profile, f"matcher_B{B}_{way}.pt.trace.json"))
                kern = {re.search(r"k_\w+(<\d>)?", e.key).group(0): round(e.device_time_total, 1)
                        for e in prof.key_averages() if re.search(r"k_\w+", e.key) and e.device_time_total > 0}
                case.setdefault("profile_device_us", {})[way] = kern
        if not case["identical"]:
            print(json.dumps(res))
            raise SystemExit(f"B = {B}: the batched call's outputs differ from the single calls'")
    print(json.dumps(res))


if __name__ == "__main__":
    main()
