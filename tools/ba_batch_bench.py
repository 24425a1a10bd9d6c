"""Batched local BA at every cluster size against sequential calls: B windows through se2gpu_ba_optimize_batch (one
thread-block cluster of C CTAs per window, C forced to 2, 4 and 8 with SE2GPU_BA_BATCH_CLUSTER) or through B
se2gpu_ba_optimize calls on one stream, the path a mapping process has without the batch.

    python tools/ba_batch_bench.py [--reps 20] [--warmup 3] [--iters 10] [--batches 1,8,32,64] [--out FILE]

Shapes: S (10 KF / 800 landmarks, nf = 9 < 16), C3 (20 KF / 2 000) and C4 (50 KF / 5 000), a distinct seed per window.
Per (shape, B) the sequential way and the three batched ways run alternating, each repetition timed with CUDA events on the
default stream (every call ends in a device synchronise): `reset` + `optimize(iters)` per window in turn, or `reset` x B +
`optimize_batch(iters)`. Reported: median, min and max ms per call, windows/s, LM iterations/s, launches per call, the
cluster size the library's rule picks for the shape, and whether every window of the B = 8 batch equals, byte for byte, a
single context run with SE2GPU_BA_PK_GRID = C. The card's name, power limit and SM clock are read in the same run.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

from se2lam_b200 import _capi  # noqa: E402
from se2lam_b200.ba import LocalBA  # noqa: E402
from tools import synth  # noqa: E402

SHAPES = {"S": dict(n_kf=10, n_lm=800), "C3": dict(n_kf=20, n_lm=2000), "C4": dict(n_kf=50, n_lm=5000)}
SIZES = (2, 4, 8)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def timed(fn):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    out = fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b), out


def context(prob, grid=None, cluster=None):
    """A context created under SE2GPU_BA_PK_GRID = grid and SE2GPU_BA_BATCH_CLUSTER = cluster (read at creation)."""
    for k, v in (("SE2GPU_BA_PK_GRID", grid), ("SE2GPU_BA_BATCH_CLUSTER", cluster)):
        if v is None:
            os.environ.pop(k, None)
        else:
            os.environ[k] = str(v)
    ba = LocalBA.from_problem(prob)
    os.environ.pop("SE2GPU_BA_PK_GRID", None)
    os.environ.pop("SE2GPU_BA_BATCH_CLUSTER", None)
    return ba


def result_bytes(ba, out):
    n, st = out
    p, l = ba.get()
    return n, st.tobytes(), p.tobytes(), l.tobytes()


def summary(ts, B, iters):
    ms = float(np.median(ts))
    return dict(ms=ms, ms_min=float(np.min(ts)), ms_max=float(np.max(ts)), windows_per_s=B / ms * 1e3, lm_iters_per_s=iters / ms * 1e3)


def run(args):
    lib = _capi.lib()
    rows = []
    for shape, kw in SHAPES.items():
        probs = [synth.ba_window(seed=1000 + k, **kw) for k in range(max(args.batches))]
        rule = context(probs[0]).batch_cluster()
        same = {}
        for C in SIZES:      # the B = 8 batch at size C against single contexts at grid C
            bas = [context(p, cluster=C) for p in probs[:8]]
            outs = LocalBA.optimize_batch(bas, args.iters)
            same[C] = all(result_bytes(b, o) == result_bytes(s, s.optimize(args.iters))
                          for b, o, s in zip(bas, outs, [context(p, grid=C) for p in probs[:8]]))
            del bas
        for B in args.batches:
            seq_bas = [context(p) for p in probs[:B]]
            bat_bas = {C: [context(p, cluster=C) for p in probs[:B]] for C in SIZES}
            seq, bat, n_seq, n_bat, launches = [], {C: [] for C in SIZES}, 0, {}, {}

            def sequential():
                n = 0
                for b in seq_bas:
                    b.reset()
                    n += b.optimize(args.iters)[0]
                return n

            def batched(C):
                for b in bat_bas[C]:
                    b.reset()
                n0 = lib.se2gpu_launch_count()
                out = LocalBA.optimize_batch(bat_bas[C], args.iters)
                return sum(o[0] for o in out), lib.se2gpu_launch_count() - n0

            for r in range(args.warmup + args.reps):
                t, n = timed(sequential)
                if r >= args.warmup:
                    seq.append(t); n_seq = n
                for C in SIZES:
                    t, (n, nl) = timed(lambda: batched(C))
                    if r >= args.warmup:
                        bat[C].append(t); n_bat[C] = n; launches[C] = nl
            row = dict(shape=shape, B=B, rule_cluster=rule, sequential=summary(seq, B, n_seq))
            for C in SIZES:
                row[f"C{C}"] = dict(summary(bat[C], B, n_bat[C]), launches_per_call=launches[C], bytes_equal_B8=same[C])
            rows.append(row)
            print(json.dumps(row), flush=True)
            del seq_bas, bat_bas
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--batches", default="1,8,32,64")
    ap.add_argument("--out", help="also write the rows as JSON to this file")
    args = ap.parse_args()
    args.batches = [int(b) for b in args.batches.split(",")]
    if not torch.cuda.is_available():
        sys.exit("ba_batch_bench: no GPU")
    info = card()
    print(json.dumps(dict(card=info)), flush=True)
    rows = run(args)
    if args.out:
        with open(args.out, "w") as f:
            json.dump(dict(card=info, rows=rows), f, indent=1)


if __name__ == "__main__":
    main()
