"""Bag-of-words on the device: se2gpu_voc_compute_bow_device over B keyframes and se2gpu_search_by_bow_batch_device over B
keyframe pairs, against the host SearchByBoW entry called once per pair.

    python tools/bow_batch_bench.py [--reps 50] [--warmup 5] [--out FILE]

Vocabulary: tests/bow_cases.make_voc(10, 6), ORBvoc's shape (k = 10, L = 6, 1.1 M nodes), levelsup = 4 as
KeyFrame::ComputeBoW uses. Keyframes: 1 000 features each (64 distinct keyframes from tests/bow_cases.make_features, tiled
for larger batches; the side-2 keyframe of a pair is its side-1 keyframe with 0 to 12 bits of every descriptor flipped).
Every repetition is timed with CUDA events on the current stream and ends in a device synchronise; reported are the
median, min and max over `reps` repetitions after `warmup` untimed ones.
  compute_bow    B = 1, 64 and 2 000 keyframes (2 000: the ComputeBowVecAll case): the full call, the call without the
                 BowVector (no word sums, no ordered L1 norm) and the descent alone (se2gpu_voc_transform_device on the same
                 B x 1 000 descriptors); the assembly's share is the full call minus the descent.
  search_by_bow  B = 1, 8 and 64 pairs on FeatureVectors compute_bow_device wrote, mp_only = 1, orientation check on.
  host entry     se2gpu_matcher_search_by_bow once per pair for the same B pairs on FeatureVectors already assembled on
                 the host and descriptors in host memory: it uploads, runs and synchronises per pair. Building those
                 FeatureVectors on the host is NOT in this time.
The card's name, power limit and SM clocks are read in the same run.
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

from se2lam_b200._capi import KP_DTYPE, check, lib, ptr  # noqa: E402
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
        raise SystemExit("bow_batch_bench needs a CUDA device")
    rows = [dict(card=card(), device=torch.cuda.get_device_name(0))]
    print(json.dumps(rows[0]), flush=True)

    voc = make_voc(10, 6, seed=6)
    v = Vocabulary(voc["desc"], voc["child_ptr"], voc["children"], voc["word_id"], voc["weight"], voc["levels"])
    rng = np.random.default_rng(7)
    d1 = np.stack([make_features(voc, NF, seed=1000 + b) for b in range(DISTINCT)])
    d2 = d1.copy()
    for b in range(DISTINCT):                    # the same scene seen again: a few bits of every descriptor flipped
        for i in range(NF):
            for bit in rng.integers(0, 256, int(rng.integers(0, 13))):
                d2[b, i, bit // 8] ^= np.uint8(1 << (bit % 8))
    s = torch.cuda.current_stream().cuda_stream

    def outputs(B, bow=True):
        z = lambda *sh, t=torch.int32: torch.zeros(sh, dtype=t, device="cuda:0")
        o = dict(node=z(B, NF), ptr=z(B, NF + 1), feat=z(B, NF), nn=z(B))
        o.update(word=z(B, NF) if bow else None, value=z(B, NF, t=torch.float64) if bow else None, nw=z(B) if bow else None)
        return o

    def run_bow(B, d_desc, o):
        v.compute_bow_device(B, d_desc, NF, o["node"], o["ptr"], o["feat"], o["nn"], o["word"], o["value"], o["nw"], stream=s)

    for B in (1, 64, 2000):
        d_desc = torch.from_numpy(d1[np.arange(B) % DISTINCT]).to("cuda:0")
        full, fv = outputs(B), outputs(B, bow=False)
        word = torch.zeros(B * NF, dtype=torch.int32, device="cuda:0")
        weight = torch.zeros(B * NF, dtype=torch.float64, device="cuda:0")
        node = torch.zeros(B * NF, dtype=torch.int32, device="cuda:0")
        descent = lambda: check(lib().se2gpu_voc_transform_device(v.h, ptr(d_desc), B * NF, LEVELSUP, ptr(word), ptr(weight), ptr(node),
                                                                   ptr(s)), "se2gpu_voc_transform_device")
        r = dict(leg="compute_bow", B=B, features_per_keyframe=NF, full=stats(lambda: run_bow(B, d_desc, full), args.reps, args.warmup),
                 feature_vector_only=stats(lambda: run_bow(B, d_desc, fv), args.reps, args.warmup),
                 descent_only=stats(descent, args.reps, args.warmup))
        r["assembly_ms"] = r["full"]["median_ms"] - r["descent_only"]["median_ms"]
        r["keyframes_per_s"] = B / (r["full"]["median_ms"] * 1e-3)
        rows.append(r)
        print(json.dumps(r), flush=True)

    # pairs: keyframe b of side 1 against keyframe b of side 2, FeatureVectors from compute_bow_device
    Bmax = 64
    kp = np.zeros((2, Bmax, NF), KP_DTYPE)
    kp["angle"] = rng.uniform(0, 360, kp.shape[:2] + (NF,)).astype(np.float32)
    kp["angle"][1] = (kp["angle"][0] + rng.normal(0, 3, (Bmax, NF))) % 360
    has_mp = (rng.random((2, Bmax, NF)) < 0.8).astype(np.uint8)
    t_kp = [torch.from_numpy(kp[k].view(np.uint8)).to("cuda:0") for k in range(2)]
    t_desc = [torch.from_numpy(d[:Bmax]).to("cuda:0") for d in (d1, d2)]
    t_mp = [torch.from_numpy(has_mp[k]).to("cuda:0") for k in range(2)]
    fvs = [outputs(Bmax, bow=False) for _ in range(2)]
    for k in range(2):
        run_bow(Bmax, t_desc[k], fvs[k])
    torch.cuda.synchronize()
    sides = [ORBmatcher.BowBatchSide(t_kp[k], t_desc[k], NF, fvs[k]["node"], fvs[k]["ptr"], fvs[k]["feat"], fvs[k]["nn"],
                                     has_mp=t_mp[k]) for k in range(2)]
    mt = ORBmatcher(0.6, True, max_queries=NF, max_db=NF, max_batch=Bmax)
    host_mt = ORBmatcher(0.6, True, max_queries=NF, max_db=NF)
    h_fv = [{n: t.cpu().numpy() for n, t in fvs[k].items() if t is not None} for k in range(2)]

    def host_kf(k, b):
        K = int(h_fv[k]["nn"][b])
        p = h_fv[k]["ptr"][b, :K + 1]
        return dict(angle=kp["angle"][k, b], desc=(d1, d2)[k][b], has_mp=has_mp[k, b], node=h_fv[k]["node"][b, :K], ptr=p,
                    feat=h_fv[k]["feat"][b, :p[-1]])
    host_pairs = [(host_kf(0, b), host_kf(1, b)) for b in range(Bmax)]
    for B in (1, 8, 64):
        m = torch.zeros((B, NF), dtype=torch.int32, device="cuda:0")
        nm = torch.zeros(B, dtype=torch.int32, device="cuda:0")
        dev_call = lambda: mt.SearchByBoWBatchDevice(B, sides[0], sides[1], m, nm, stream=s)
        r = dict(leg="search_by_bow", B=B, features_per_keyframe=NF, batch_device=stats(dev_call, args.reps, args.warmup))
        host_res = [None] * B

        def host_calls():
            for b in range(B):
                host_res[b] = host_mt.SearchByBoW(*host_pairs[b], True)
        r["host_entry_per_pair_assembly_excluded"] = stats(host_calls, max(5, args.reps // 5), 2)
        torch.cuda.synchronize()
        nm_h, m_h = nm.cpu().numpy(), m.cpu().numpy()
        r["equal_to_host_entry"] = all(nm_h[b] == host_res[b][0] and np.array_equal(m_h[b], host_res[b][1]) for b in range(B))
        r["matches_per_pair_median"] = float(np.median(nm_h))
        r["speedup_vs_host_entry"] = r["host_entry_per_pair_assembly_excluded"]["median_ms"] / r["batch_device"]["median_ms"]
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
