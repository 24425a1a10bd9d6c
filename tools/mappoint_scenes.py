"""Seeded scenes for the map-point updates (tests/test_mappoint_*.py, tools/mappoint_bench.py): a chain of keyframes along
an SE(2) odometry path, map points each seen by a run of keyframes (1 to 40 observations, a few past the 32-entry
shared-memory list of the GPU kernels), and the tables of se2lam_b200.mappoint filled with plausible state.

Keyframe ids have gaps (so "within 6 ids" is not "within 6 keyframes"), a few keyframes are null, every observation owns
a keypoint slot of its keyframe, and each point's descriptors are one base descriptor with a few bits flipped per view.
"""
from __future__ import annotations

import copy

import numpy as np

from tools.geom_scenes import FX, K, KP_DTYPE, LOWER_DEPTH, UPPER_DEPTH, tcw_of_odom

NLEVELS = 8
SCALE_FACTORS = (np.float32(1.2) ** np.arange(NLEVELS, dtype=np.float32)).astype(np.float32)
LONG_LISTS = (33, 47, 64, 97)


def keyframe_chain(n_kf, rng, step=0.12, null_frac=0.03):
    Tcw = np.stack([tcw_of_odom(step * k, 0.05 * np.sin(0.2 * k), 0.03 * np.sin(0.15 * k)) for k in range(n_kf)])
    kf_id = (np.arange(n_kf) + np.arange(n_kf) // 9).astype(np.int32)        # an id gap every 9 keyframes
    kf_null = (rng.random(n_kf) < null_frac).astype(np.uint8)
    return Tcw.astype(np.float32), kf_id, kf_null


def scene(M, seed=0, n_kf=None, lengths=None, n_upd=(0.15, 0.65, 0.2), mode="add", good_frac=0.3, null_frac=0.02,
          updates=None, erase_main=False, kf_null_frac=0.03, nlevels=NLEVELS):
    """M points. lengths: the list length of every point (default 1..40 with a few LONG_LISTS). n_upd: probabilities of 0, 1
    and 2 updates per point. mode "add" picks update positions among the list, "erase" the same.
    updates=(lo, hi) draws lo..hi updates per point instead of n_upd. erase_main (mode "erase") makes every point erase its
    whole list, each time the entry of its current main keyframe. kf_null_frac is the share of null keyframes, nlevels the
    pyramid's level count (octaves and scale factors).
    Returns dict(kf, mp, upd_ptr, upd_pos, params) with params the arguments of mappoint.params."""
    rng = np.random.default_rng(seed)
    sf = SCALE_FACTORS if nlevels == NLEVELS else (np.float32(1.2) ** np.arange(nlevels, dtype=np.float32)).astype(np.float32)
    if lengths is None:
        lengths = np.minimum(rng.geometric(0.12, M), 40).astype(np.int64)
        long = rng.random(M) < 0.01
        lengths[long] = rng.choice(LONG_LISTS, int(long.sum()))
    lengths = np.asarray(lengths, np.int64)
    n_kf = n_kf or int(max(64, lengths.max() + 8))
    Tcw, kf_id, kf_null = keyframe_chain(n_kf, rng, null_frac=kf_null_frac)
    Twc = np.linalg.inv(Tcw.astype(np.float64))

    start = (rng.random(M) * (n_kf - lengths + 1)).astype(np.int64)
    obs_ptr = np.zeros(M + 1, np.int32); obs_ptr[1:] = np.cumsum(lengths)
    n_obs = int(obs_ptr[-1])
    owner = np.repeat(np.arange(M), lengths)
    rank = np.arange(n_obs) - np.repeat(obs_ptr[:-1], lengths)
    obs_kf = (start[owner] + rank).astype(np.int32)
    # mObservations iterates in shared_ptr address order: shuffle some lists
    shuffled = rng.random(M) < 0.3
    for m in np.nonzero(shuffled & (lengths > 1))[0]:
        s = slice(obs_ptr[m], obs_ptr[m + 1]); obs_kf[s] = rng.permutation(obs_kf[s])

    # one slot per observation, grouped by keyframe, plus a few unused slots per keyframe
    counts = np.bincount(obs_kf, minlength=n_kf) + 3
    kp_base = np.zeros(n_kf, np.int32); kp_base[1:] = np.cumsum(counts)[:-1]
    S = int(counts.sum())
    order = np.argsort(obs_kf, kind="stable")
    obs_idx = np.zeros(n_obs, np.int32)
    rank_in_kf = np.arange(n_obs) - np.searchsorted(obs_kf[order], obs_kf[order])
    obs_idx[order] = (rank_in_kf + 1).astype(np.int32)
    slot = kp_base[obs_kf] + obs_idx

    # world points in front of the middle observer
    mid = Twc[start + lengths // 2]
    depth = np.where(rng.random(M) < 0.05, rng.uniform(9.0, 40.0, M), rng.uniform(1.0, 7.0, M))
    lat = rng.uniform(-1.5, 1.5, (M, 2))
    Xc = np.stack([lat[:, 0] * depth / 3, lat[:, 1] * depth / 4, depth], 1)
    Xw = np.einsum("mij,mj->mi", mid[:, :3, :3], Xc) + mid[:, :3, 3]
    Xw[rng.random(M) < 0.02] *= -1.0                                          # some behind every camera
    T = Tcw[obs_kf].astype(np.float64)
    pc = np.einsum("nij,nj->ni", T[:, :3, :3], Xw[owner]) + T[:, :3, 3]
    uv = (K.astype(np.float64) @ pc.T).T
    uv = uv[:, :2] / uv[:, 2:3] + rng.normal(0, 0.7, (n_obs, 2))

    kp = np.zeros(S, KP_DTYPE)
    kp["x"] = rng.uniform(0, 640, S); kp["y"] = rng.uniform(0, 480, S)
    kp["octave"] = rng.integers(0, nlevels, S); kp["size"] = 31; kp["angle"] = -1; kp["class_id"] = -1
    kp["x"][slot] = uv[:, 0]; kp["y"][slot] = uv[:, 1]
    base = rng.integers(0, 256, (M, 32), dtype=np.uint8)
    desc = rng.integers(0, 256, (S, 32), dtype=np.uint8)
    flips = rng.random((n_obs, 256)) < rng.choice([0.02, 0.05, 0.1], n_obs)[:, None]
    desc[slot] = base[owner] ^ np.packbits(flips, axis=1)
    desc[slot[rng.random(n_obs) < 0.05]] = desc[slot[0]]                    # repeated descriptors: median ties
    view_mp = np.zeros((S, 3), np.float32)
    view_mp[slot] = (pc * (1 + rng.normal(0, 0.01, (n_obs, 1)))).astype(np.float32)
    view_info = np.zeros((S, 3, 3))
    d = rng.uniform(10, 1e4, (n_obs, 3))
    view_info[slot] = np.einsum("ni,ij->nij", d, np.eye(3))

    first = slot[obs_ptr[:-1].clip(max=n_obs - 1)]
    main_kf = np.where(rng.random(M) < 0.8, obs_kf[obs_ptr[:-1].clip(max=n_obs - 1)], -1).astype(np.int32)
    normal = Xw - Twc[start][:, :3, 3]
    normal /= np.linalg.norm(normal, axis=1, keepdims=True)
    main_octave = kp["octave"][first].astype(np.int32)
    level_scale = sf[main_octave]
    dist = np.linalg.norm(view_mp[first].astype(np.float64), axis=1).astype(np.float32)
    mp = dict(pos=(Xw + rng.normal(0, 0.02, (M, 3))).astype(np.float32),
              good_prl=(rng.random(M) < good_frac).astype(np.uint8), null=(rng.random(M) < null_frac).astype(np.uint8),
              main_kf=main_kf, main_desc=desc[first].copy(), main_octave=main_octave,
              main_measure=np.stack([kp["x"][first], kp["y"][first]], 1).astype(np.float32),
              level_scale=level_scale.astype(np.float32), normal=normal.astype(np.float32),
              min_dist=(dist * level_scale / sf[-1]).astype(np.float32), max_dist=(dist * level_scale).astype(np.float32),
              obs_ptr=obs_ptr, obs_kf=obs_kf, obs_idx=obs_idx)
    kf = dict(kf_id=kf_id, kf_null=kf_null, Tcw=Tcw, kp_base=kp_base, kp=kp, desc=desc, view_mp=view_mp, view_info=view_info)

    # updates: 0, 1 or 2 distinct list positions per point; adds favour the newest keyframes
    nu = np.minimum(rng.choice(3, M, p=n_upd) if updates is None else rng.integers(updates[0], updates[1] + 1, M), lengths)
    if erase_main:
        nu = lengths.copy()
    upd_ptr = np.zeros(M + 1, np.int32); upd_ptr[1:] = np.cumsum(nu)
    upd_pos = np.zeros(int(upd_ptr[-1]), np.int32)
    for m in np.nonzero(nu)[0]:
        L = int(lengths[m])
        if erase_main:
            pos = _main_first_order(kf_null[obs_kf[obs_ptr[m]:obs_ptr[m + 1]]], desc[slot[obs_ptr[m]:obs_ptr[m + 1]]],
                                    0 if main_kf[m] >= 0 else None)
        elif mode == "add" and rng.random() < 0.7:
            kfs = obs_kf[obs_ptr[m]:obs_ptr[m + 1]]
            pos = np.argsort(-kfs, kind="stable")[:nu[m]][::-1]            # the newest observers, oldest first
        else:
            pos = rng.choice(L, nu[m], replace=False)
        upd_pos[upd_ptr[m]:upd_ptr[m + 1]] = pos
    return dict(kf=kf, mp=mp, upd_ptr=upd_ptr, upd_pos=upd_pos,
                params=dict(K=K, lower_depth=LOWER_DEPTH, upper_depth=UPPER_DEPTH, fx=FX, scale_factors=sf))


def _main_first_order(kf_null, desc, main):
    """list positions in the order that erases the main keyframe's entry each time: `main` first (None: no main keyframe),
    then the entry updateMainKFandDescriptor picks among the rest (least median Hamming distance over the entries of
    non-null keyframes, first on ties), and any entry once only null keyframes remain"""
    left = list(range(len(kf_null)))
    order = []
    while left:
        valid = [j for j in left if not kf_null[j]]
        if main is None or main not in left:
            main = left[0]
            if valid:
                bits = np.unpackbits(desc[valid], axis=1).astype(np.int32)
                D = (bits[:, None, :] != bits[None, :, :]).sum(2)
                med = np.sort(D, axis=1)[:, int(0.5 * (len(valid) - 1))]
                main = valid[int(np.argmin(med))]
        order.append(main)
        left.remove(main)
    return np.array(order, np.int64)


def copy_tables(sc):
    """deep copies of the scene's kf / mp tables (every call updates them in place)"""
    return copy.deepcopy(sc["kf"]), copy.deepcopy(sc["mp"])
