"""Seeded static maps and camera streams for the localization handle (se2lam_b200.loc), built on the tracker's plane
renderer (tools/track_scenes.py). Keyframes are rendered along a path and extracted by the CPU ORB oracle; each keyframe
creates map points from a share of its keypoints, back-projected onto the plane, and neighbouring keyframes observe a
point when it projects within 2 px of one of their free keypoints. Some points are seeded null, some without good
parallax; covisibility links keyframes that share at least `min_shared` points.

Poses follow the Localizer's convention: Tcw(x, y, theta) = cTb * Se2(x, y, theta).inv().toCvSE3(), so a stream's first
frame (Tcw = cTb) sits at odometry (0, 0, 0) and UpdatePoseCurr chains the odometry from there.
"""
from __future__ import annotations

import numpy as np

from tools import track_scenes as ts

F32 = np.float32
DEPTH = 3.0


def config(nfeatures=500, w=ts.W, h=ts.H, max_local_mps=2048, **camera):
    """tools/track_scenes.config (camera: fx, dist, fast_th) plus the Localizer's image bounds, Huber width and local-map
    capacity"""
    c = ts.config(nfeatures=nfeatures, w=w, h=h, **camera)
    c.update(bounds=(0.0, float(w), 0.0, float(h)), huber=float(np.sqrt(5.991)), max_local_mps=max_local_mps, w=w, h=h)
    return c


def tcw(cfg, pose):
    x, y, th = (float(v) for v in pose)
    c, s = np.cos(th), np.sin(th)
    Twb = np.array([[c, -s, 0, x], [s, c, 0, y], [0, 0, 1, 0], [0, 0, 0, 1]], np.float64)
    return (cfg["cTb"].astype(np.float64) @ np.linalg.inv(Twb)).astype(np.float32)


def _project(K, T, P):
    pc = (T[:3, :3].astype(np.float64) @ P.T).T + T[:3, 3]
    return (K[0, 0] * pc[:, 0] / pc[:, 2] + K[0, 2]), (K[1, 1] * pc[:, 1] / pc[:, 2] + K[1, 2])


def build_map(seed, cfg, n_kf=8, step=0.08, share=0.6, p_null=0.05, p_bad=0.05, min_shared=15, path=None, extract=None):
    """the map dict of se2lam_b200.loc plus 'kf_pose' [K,3], 'tex', 'kf_kp' and 'kf_desc'. extract(img) -> (keypoints,
    descriptors) defaults to the CPU ORB oracle."""
    rng = np.random.default_rng(seed)
    tex = ts.texture(seed)
    K = np.asarray(cfg["K"], np.float32)
    w, h = cfg["w"], cfg["h"]
    if extract is None:
        from oracle import pyoracle
        extract = pyoracle.OrbOracle(cfg["nfeatures"], cfg["scale_factor"], cfg["nlevels"], cfg["fast_th"]).extract
    if path is None:
        path = np.array([(step * k, 0.02 * np.sin(k), 0.03 * k) for k in range(n_kf)], np.float32)
    kps, descs, Ts = [], [], []
    for pose in path:
        kp, d = extract(ts.render(tex, pose, K, DEPTH, w, h))
        kps.append(kp); descs.append(d); Ts.append(tcw(cfg, pose))
    kf_ptr = np.zeros(len(path) + 1, np.int32)
    for k, kp in enumerate(kps):
        kf_ptr[k + 1] = kf_ptr[k] + len(kp)
    slot = np.full(kf_ptr[-1], -1, np.int32)
    pos, desc, octv = [], [], []
    for k, kp in enumerate(kps):
        Tinv = np.linalg.inv(Ts[k].astype(np.float64))
        for i in np.flatnonzero(rng.random(len(kp)) < share):
            if slot[kf_ptr[k] + i] >= 0:
                continue
            pc = np.array([(kp["x"][i] - K[0, 2]) / K[0, 0] * DEPTH, (kp["y"][i] - K[1, 2]) / K[1, 1] * DEPTH, DEPTH, 1.0])
            P = (Tinv @ pc)[:3]
            j = len(pos)
            pos.append(P); desc.append(descs[k][i]); octv.append(int(kp["octave"][i]))
            slot[kf_ptr[k] + i] = j
            for q in (k - 2, k - 1, k + 1, k + 2):              # neighbours observe the point at a free keypoint nearby
                if q < 0 or q >= len(kps):
                    continue
                u, v = _project(K, Ts[q], P[None])
                d2 = (kps[q]["x"] - u[0]) ** 2 + (kps[q]["y"] - v[0]) ** 2
                c = int(np.argmin(d2)) if len(d2) else -1
                if c >= 0 and d2[c] < 4.0 and slot[kf_ptr[q] + c] < 0:
                    slot[kf_ptr[q] + c] = j
    M = len(pos)
    obs = [sorted(set(int(v) for v in slot[kf_ptr[k]:kf_ptr[k + 1]] if v >= 0)) for k in range(len(kps))]
    sets = [set(o) for o in obs]
    cov = [[q for q in range(len(kps)) if q != k and len(sets[k] & sets[q]) >= min_shared] for k in range(len(kps))]
    csr = lambda rows: (np.cumsum([0] + [len(r) for r in rows]).astype(np.int32),
                        np.array([v for r in rows for v in r], np.int32))
    obs_ptr, obs_idx = csr(obs)
    cov_ptr, cov_idx = csr(cov)
    null = (rng.random(M) < p_null).astype(np.uint8)
    good = (rng.random(M) >= p_bad).astype(np.uint8)
    return dict(kf_Tcw=np.stack(Ts), kf_kp_ptr=kf_ptr, kf_obs_mp=slot, kf_obs_ptr=obs_ptr, kf_obs=obs_idx, kf_cov_ptr=cov_ptr,
                kf_cov=cov_idx, mp_pos=np.array(pos, np.float32).reshape(M, 3), mp_null=null, mp_good_prl=good,
                mp_desc=np.array(desc, np.uint8).reshape(M, 32), mp_octave=np.array(octv, np.int32), kf_pose=path, tex=tex,
                kf_kp=kps, kf_desc=descs)


KINDS = ["along", "leave", "blank", "short"]


def stream(seed, m, cfg, frames=30, kind="along"):
    """(frames [T,H,W] u1, odom [T,3] f4, start pose [3]). The odometry is relative to the stream's start (its first frame
    is at odometry 0); the start sits on the map's path. along: follows the path; leave: walks off the textured map
    half-way; blank: featureless frames part of the way (few observations: the BA gate); short: stays near the start."""
    rng = np.random.default_rng(seed)
    path = m["kf_pose"]
    k0 = int(rng.integers(0, max(len(path) - 3, 1)))
    start = path[k0].astype(np.float64)
    od = np.zeros((frames, 3), np.float32)
    x = y = th = 0.0
    for t in range(1, frames):
        sp = {"along": 0.012, "leave": 0.012 if t < frames // 2 else 0.25, "blank": 0.01, "short": 0.002}[kind]
        th += 0.004 * (rng.random() - 0.3)
        x += sp * (0.8 + 0.4 * rng.random())
        od[t] = (x, y, th)
    imgs = []
    K = np.asarray(cfg["K"], np.float32)
    for t in range(frames):
        c, s = np.cos(start[2]), np.sin(start[2])
        wx = start[0] + c * od[t, 0] - s * od[t, 1]
        wy = start[1] + s * od[t, 0] + c * od[t, 1]
        img = ts.render(m["tex"], (wx, wy, start[2] + od[t, 2]), K, DEPTH, cfg["w"], cfg["h"])
        if kind == "blank" and frames // 3 <= t < frames // 3 + 4:
            img = np.full_like(img, 100)
            img[50:60, 50:60] = 200
        imgs.append(img)
    return np.stack(imgs), od, start.astype(np.float32), k0


def loop_matches(oracle_kp, oracle_desc, m, k, rng=None, extra_repeat=True):
    """a verified mapMatchGood stand-in between the stream's current keypoints and keyframe k: each current keypoint whose
    nearest keyframe keypoint (by image position, both views close) is within 3 px, ascending idxCurr; with extra_repeat,
    one idxLoop is used twice"""
    kk = m["kf_kp"][k]
    pairs = []
    for i in range(len(oracle_kp)):
        d2 = (kk["x"] - oracle_kp["x"][i]) ** 2 + (kk["y"] - oracle_kp["y"][i]) ** 2
        if len(d2) and d2.min() < 9.0:
            pairs.append((i, int(np.argmin(d2))))
    if extra_repeat and len(pairs) >= 2:
        pairs[1] = (pairs[1][0], pairs[0][1])
    return pairs
