"""Seeded camera streams for the tracker (se2lam_b200.track): frames rendered with numpy from a seeded texture on a plane
through the camera, so image motion follows the odometry, plus the configuration the tests and tools/track_bench.py use.
No OpenCV needed.

The camera looks along the body z axis at a plane `depth` metres away (cTb is a pure offset), so a body motion (x, y,
theta) moves the view of the plane by (x, y) and turns it by theta about the optical axis. The frames are rendered
without lens distortion whatever cfg["dist"] holds: the handles and the oracles undistort them alike.
"""
from __future__ import annotations

import numpy as np

W, H = 320, 240
F32 = np.float32


def config(nfeatures=500, max_frames=12, min_frames=8, w=W, h=H, fx=300.0, dist=(), fast_th=20):
    """the Config values of a w x h camera with focal length fx (principal point at the centre) and distortion
    coefficients dist (empty, or 4, 5, 8 or 12 of them)"""
    fx = fy = F32(fx)
    K = np.array([[fx, 0, w / 2], [0, fy, h / 2], [0, 0, 1]], np.float32)
    cTb = np.eye(4, dtype=np.float32); cTb[:3, 3] = (0.05, -0.02, 0.0)
    bTc = np.eye(4, dtype=np.float32); bTc[:3, 3] = -cTb[:3, 3]
    grid = (F32(0), F32(0), F32(F32(64) / F32(w)), F32(F32(48) / F32(h)))
    return dict(nfeatures=nfeatures, scale_factor=1.2, nlevels=6, fast_th=fast_th, K=K, dist=tuple(float(v) for v in dist),
                grid=grid, lower_depth=0.2, upper_depth=10.0, cTb=cTb, bTc=bTc, odo_noise=(0.01, 0.01, 0.002),
                min_frames=min_frames, max_frames=max_frames, w=w, h=h)


def texture(seed, size=1024):
    """seeded blob texture (values 0..255) on a size x size grid covering [-2, 2) m"""
    rng = np.random.default_rng(seed)
    t = np.zeros((size, size), np.float32)
    for scale in (8, 32, 64):
        c = rng.random((size // scale + 2, size // scale + 2)).astype(np.float32)
        idx = np.arange(size) / scale
        i0 = idx.astype(int); fr = (idx - i0).astype(np.float32)
        rows = c[i0] * (1 - fr)[:, None] + c[i0 + 1] * fr[:, None]
        t += rows[:, i0] * (1 - fr)[None, :] + rows[:, i0 + 1] * fr[None, :]
    t -= t.min(); t *= 255.0 / max(float(t.max()), 1e-6)
    return t


def render(tex, odom, K, depth=3.0, w=W, h=H, extent=4.0):
    """the view of the textured plane from body pose odom = (x, y, theta)"""
    x, y, th = (float(v) for v in odom)
    u, v = np.meshgrid(np.arange(w, dtype=np.float64), np.arange(h, dtype=np.float64))
    xc = (u - K[0, 2]) / K[0, 0] * depth; yc = (v - K[1, 2]) / K[1, 1] * depth
    c, s = np.cos(th), np.sin(th)
    X = c * xc - s * yc + x; Y = s * xc + c * yc + y
    n = tex.shape[0]
    px = np.clip(((X / extent + 0.5) * n).astype(int), 0, n - 1); py = np.clip(((Y / extent + 0.5) * n).astype(int), 0, n - 1)
    return np.ascontiguousarray(tex[py, px].astype(np.uint8))


def odometry(seed, frames, speed=0.02, turn=0.01, still=False):
    """a seeded smooth path; still=True stays put (odometry below both needNewKF thresholds)"""
    rng = np.random.default_rng(seed)
    od = np.zeros((frames, 3), np.float32)
    if still:
        return od
    th = x = y = 0.0
    for k in range(1, frames):
        th += turn * (0.5 + rng.random())
        step = speed * (0.5 + rng.random())
        x += step * np.cos(th); y += step * np.sin(th)
        od[k] = (x, y, np.arctan2(np.sin(th), np.cos(th)))
    return od


def stream(seed, frames=30, kind="normal", cfg=None):
    """(frames [T,h,w] u1 at cfg's size, odom [T,3] f4, kf side dict: observed [cap] u1, view_mp [cap,3] f4, n_obs_mp,
    accept [T]). kind: normal, lowtex_first (first frame <= 100 keypoints), blank (a constant frame mid-way), jump (an
    unrelated frame mid-way: fewer than 10 inliers), still (no motion), reject (acceptNewKF() false), prl (nothing
    observed: c1 && c2)"""
    cfg = cfg or config()
    cap, w, h = cfg["nfeatures"], cfg["w"], cfg["h"]
    rng = np.random.default_rng(seed + 1000)
    tex = texture(seed)
    od = odometry(seed, frames, still=(kind == "still"))
    imgs = np.stack([render(tex, o, cfg["K"], w=w, h=h) for o in od])
    if kind == "lowtex_first":
        imgs[0] = 128; imgs[0, 100:110, 150:160] = 255
    if kind == "blank":
        imgs[frames // 2] = 90
    if kind == "jump":
        imgs[frames // 2] = render(texture(seed + 7), od[frames // 2] + 0.5, cfg["K"], w=w, h=h)
    observed = (rng.random(cap) < (0.0 if kind == "prl" else 0.3)).astype(np.uint8)
    view_mp = rng.standard_normal((cap, 3)).astype(np.float32)
    accept = np.ones(frames, bool)
    if kind == "reject":
        accept[:] = False
    n_obs = int(observed.sum()) if kind != "prl" else 1000
    return imgs, od, dict(observed=observed, view_mp=view_mp, n_obs_mp=n_obs, accept=accept)


KINDS = ["normal", "lowtex_first", "blank", "jump", "still", "reject", "prl"]

# mild lens distortion of each length cv::undistort takes, in OpenCV's order (k1, k2, p1, p2[, k3[, k4, k5, k6[, s1, s2,
# s3, s4]]]): the rational (k4..k6) and thin-prism (s1..s4) terms are non-zero
DISTORTION = {
    4: (-0.06, 0.012, 0.0009, -0.0006),
    5: (-0.05, 0.01, 0.0008, -0.0005, 0.002),
    8: (-0.05, 0.01, 0.0008, -0.0005, 0.002, 0.01, -0.004, 0.002),
    12: (-0.05, 0.01, 0.0008, -0.0005, 0.002, 0.01, -0.004, 0.002, 0.001, -0.0004, 0.0007, -0.0003),
}
