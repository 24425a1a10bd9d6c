"""Loop closure on the device: se2gpu_detect_loop_device for B queries against N keyframes and se2gpu_verify_loop_device for
B pairs, beside DBoW2's own L1Scoring on one CPU core.

    python tools/loop_bench.py [--reps 50] [--warmup 5] [--out FILE]

Vocabulary: tests/bow_cases.make_voc(10, 6), ORBvoc's shape (k = 10, L = 6), levelsup = 4. Keyframes: 1 000 features each
(64 distinct keyframes from tests/bow_cases.make_features, tiled for larger sets); BowVectors and FeatureVectors from
se2gpu_voc_compute_bow_device, built once. Query b is database keyframe 5 b with a few bits of every descriptor flipped.
  detect  B = 1, 8, 64 queries x N = 200, 2 000 keyframes, GlobalMapper parameters.
  verify  B = 1, 8, 64 pairs, query b against its own scene (keyPointsUn from two views of one 3D scene), GlobalMapper
          verdict.
  cpu     DetectLoopClose's loop as the reference runs it, on one core: every keyframe's BowVector copied
          (DBoW2::BowVector BowVec = pKF->mBowVec) and scored with DBoW2's L1Scoring::score from oracle/_ref/libdbow2_l1.so
          (built by oracle/dbow2_ref.mk from the reference tree; the column is absent without it), timed inside the
          library with std::chrono around the whole loop (dbow2_l1_detect_ms).
Every GPU repetition is timed with CUDA events on the current stream and ends in a device synchronise; reported are the
median, min and max over `reps` repetitions after `warmup` untimed ones. The card's name and power limit are read in the
same run.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

from oracle import pyloop  # noqa: E402
from se2lam_b200 import loop as gl  # noqa: E402
from se2lam_b200._capi import KP_DTYPE  # noqa: E402
from se2lam_b200.bow import Vocabulary  # noqa: E402
from se2lam_b200.matcher import ORBmatcher  # noqa: E402
from tests.bow_cases import make_features, make_voc  # noqa: E402

NF, LEVELSUP, DISTINCT = 1000, 4, 64


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def stats(fn, reps, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    t = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        t.append(a.elapsed_time(b))
    return dict(median_ms=float(np.median(t)), min_ms=float(np.min(t)), max_ms=float(np.max(t)))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("loop_bench needs a CUDA device")
    rows = [dict(card=card(), device=torch.cuda.get_device_name(0))]
    print(json.dumps(rows[0]), flush=True)
    s = torch.cuda.current_stream().cuda_stream
    voc = make_voc(10, 6, seed=6)
    v = Vocabulary(voc["desc"], voc["child_ptr"], voc["children"], voc["word_id"], voc["weight"], voc["levels"])
    rng = np.random.default_rng(7)
    d1 = np.stack([make_features(voc, NF, seed=1000 + b) for b in range(DISTINCT)])
    d2 = d1.copy()
    for b in range(DISTINCT):
        for i in range(NF):
            for bit in rng.integers(0, 256, int(rng.integers(0, 13))):
                d2[b, i, bit // 8] ^= np.uint8(1 << (bit % 8))

    def bow(desc):
        B = len(desc)
        z = lambda *sh, t=torch.int32: torch.zeros(sh, dtype=t, device="cuda:0")
        o = dict(word=z(B, NF), value=z(B, NF, t=torch.float64), nw=z(B), node=z(B, NF), ptr=z(B, NF + 1), feat=z(B, NF), nn=z(B))
        v.compute_bow_device(B, torch.from_numpy(np.ascontiguousarray(desc)).to("cuda:0"), NF, o["node"], o["ptr"], o["feat"], o["nn"],
                             o["word"], o["value"], o["nw"], levelsup=LEVELSUP, stream=s)
        return o

    Nmax, Bmax = 2000, 64
    db = bow(d1[np.arange(Nmax) % DISTINCT])
    qidx = (5 * np.arange(Bmax)) % DISTINCT
    qo = bow(d2[qidx])
    torch.cuda.synchronize()
    db_id = torch.arange(Nmax, dtype=torch.int32, device="cuda:0")
    q_id = torch.full((Bmax,), 10 ** 6, dtype=torch.int32, device="cuda:0")
    h = {k: t.cpu().numpy() for k, t in list(db.items()) + [("q" + k, t) for k, t in qo.items()]}
    ref = pyloop.make_ref()
    for N in (200, 2000):
        for B in (1, 8, 64):
            scores = torch.zeros(B * N, dtype=torch.float64, device="cuda:0")
            loop = torch.zeros(B, dtype=torch.int32, device="cuda:0"); best = torch.zeros(B, dtype=torch.float64, device="cuda:0")
            call = lambda: gl.detect_loop_device(B, qo["word"], qo["value"], qo["nw"], NF, N, db["word"], db["value"], db["nw"], NF,
                                                 scores, loop, best, d_q_id=q_id, d_db_id=db_id, params=gl.DETECT_GLOBAL_MAPPER,
                                                 stream=s)
            r = dict(leg="detect", B=B, N=N, words_per_keyframe_median=float(np.median(h["nw"][:N])), gpu=stats(call, args.reps, args.warmup))
            r["gpu_per_query_us"] = r["gpu"]["median_ms"] * 1e3 / B
            if ref and B == 1:
                n0 = h["qnw"][0]
                ms, best_c = pyloop.dbow2_detect_ms(h["qword"][0, :n0], h["qvalue"][0, :n0], h["word"][:N], h["value"][:N], h["nw"][:N])
                r["cpu_one_core_dbow2_ms_per_query"] = ms
                torch.cuda.synchronize()
                r["gpu_best_equals_cpu"] = bool(best.cpu().numpy()[0] == best_c)
            rows.append(r)
            print(json.dumps(r), flush=True)

    # verify: query b against its own scene
    P = np.stack([rng.uniform(-3, 3, NF), rng.uniform(-2, 2, NF), rng.uniform(3, 9, NF)], 1)
    proj = lambda X: np.stack([400 * X[:, 0] / X[:, 2] + 320, 400 * X[:, 1] / X[:, 2] + 240], 1)
    kp = np.zeros((2, Bmax, NF), KP_DTYPE)
    xy1, xy2 = proj(P), proj(P + np.array([0.4, 0.05, 0.1])) + rng.normal(0, 0.3, (NF, 2))
    kp["x"][0], kp["y"][0], kp["x"][1], kp["y"][1] = xy1[:, 0], xy1[:, 1], xy2[:, 0], xy2[:, 1]
    kp["angle"] = rng.uniform(0, 360, (2, Bmax, NF)).astype(np.float32)
    kp["angle"][1] = (kp["angle"][0] + rng.normal(0, 3, (Bmax, NF))) % 360
    mapo = bow(d1[qidx])
    torch.cuda.synchronize()
    t_kp = [torch.from_numpy(kp[k].view(np.uint8)).to("cuda:0") for k in range(2)]
    t_desc = [torch.from_numpy(np.ascontiguousarray(d)).to("cuda:0") for d in (d2[qidx], d1[qidx])]
    obs = [torch.from_numpy((rng.random((Bmax, NF)) < 0.7).astype(np.uint8)).to("cuda:0") for _ in range(2)]
    sides = [ORBmatcher.BowBatchSide(t_kp[1], t_desc[0], NF, qo["node"], qo["ptr"], qo["feat"], qo["nn"], has_mp=obs[0]),
             ORBmatcher.BowBatchSide(t_kp[0], t_desc[1], NF, mapo["node"], mapo["ptr"], mapo["feat"], mapo["nn"], has_mp=obs[1])]
    mt = ORBmatcher(0.6, True, max_queries=NF, max_db=NF, max_batch=Bmax)
    for B in (1, 8, 64):
        z = lambda *sh, t=torch.int32: torch.zeros(sh, dtype=t, device="cuda:0")
        o = dict(raw=z(B, NF), good=z(B, NF), mp=z(B, NF), counts=z(B, 3), verified=z(B, t=torch.uint8))
        loop = torch.arange(B, dtype=torch.int32, device="cuda:0")
        n_mps = torch.full((B,), 600, dtype=torch.int32, device="cuda:0")
        call = lambda: gl.verify_loop_device(mt, B, sides[0], sides[1], loop, o["raw"], o["good"], o["mp"], o["counts"], o["verified"],
                                             d_n_mps_cur=n_mps, stream=s)
        r = dict(leg="verify", B=B, gpu=stats(call, args.reps, args.warmup))
        c = o["counts"].cpu().numpy()
        r.update(raw_median=float(np.median(c[:, 0])), good_median=float(np.median(c[:, 1])), mp_median=float(np.median(c[:, 2])),
                 verified=int(o["verified"].cpu().numpy().sum()))
        rows.append(r)
        print(json.dumps(r), flush=True)
    rows.append(dict(card_after=card(), finished=time.strftime("%Y-%m-%dT%H:%M:%S")))
    print(json.dumps(rows[-1]), flush=True)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(rows, f, indent=1)


if __name__ == "__main__":
    main()
