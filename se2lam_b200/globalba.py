"""The global pose graph on the GPU: GlobalMapper::GlobalBA through se2gpu_global_ba, and its map-point write-back through
se2gpu_global_ba_update_points. numpy in, numpy out; there is no CPU fallback."""
from __future__ import annotations

import ctypes as C

import numpy as np

from ._capi import BA_STATS_DTYPE, GlobalBAParams, check, lib, ptr

OK, NOT_PD = 0, 2


def params(Tbc, xrot_info=1e6, yrot_info=1e6, z_info=1.0, iterations=15):
    """se2gpu_global_ba_params with the reference's values; Tbc = Config::bTc [4,4], iterations = Config::GLOBAL_ITER."""
    p = GlobalBAParams()
    p.Tbc[:] = [float(v) for v in np.asarray(Tbc, np.float32).reshape(16)]
    p.xrot_info, p.yrot_info, p.z_info, p.iterations = xrot_info, yrot_info, z_info, iterations
    return p


def edge_arrays(edges):
    """(from [E] int32, to [E] int32, measure [E,16] float32, info [E,36] float32) of a list of (from, to, measure, info)."""
    E = len(edges)
    fr = np.array([e[0] for e in edges], np.int32).reshape(E)
    to = np.array([e[1] for e in edges], np.int32).reshape(E)
    me = np.ascontiguousarray(np.array([np.asarray(e[2], np.float32).reshape(16) for e in edges], np.float32).reshape(E, 16))
    inf = np.ascontiguousarray(np.array([np.asarray(e[3], np.float32).reshape(36) for e in edges], np.float32).reshape(E, 36))
    return fr, to, me, inf


class Context:
    """se2gpu_global_ba_ctx: grow-only device buffers and a stream, reusable across graphs of any size."""

    def __init__(self, device=0):
        self.h = lib().se2gpu_global_ba_create(device)
        if not self.h:
            check(-1, "se2gpu_global_ba_create")

    def close(self):
        if self.h:
            lib().se2gpu_global_ba_destroy(self.h)
            self.h = None

    def __del__(self):
        self.close()

    def run(self, Tcw, fixed, edges, prm):
        """One GlobalBA. Tcw [N,4,4] (KeyFrame::Tcw), fixed [N] (mIdKF == 0), edges [(from, to, measure [4,4], info [6,6])],
        odometry and feature constraints alike. Returns dict(status, iterations, Tcw [N,4,4] float32 (what setPose
        receives), poses [N,7] (qx, qy, qz, qw, tx, ty, tz of each estimate, camera-to-world), stats)."""
        T = np.ascontiguousarray(Tcw, np.float32).reshape(-1, 16)
        N = len(T)
        fx = np.ascontiguousarray(fixed, np.uint8).reshape(N)
        fr, to, me, inf = edge_arrays(edges)
        out = np.zeros((N, 16), np.float32)
        poses = np.zeros((N, 7))
        status = np.zeros(1, np.int32); iters = np.zeros(1, np.int32)
        stats = np.zeros(max(prm.iterations, 1), BA_STATS_DTYPE)
        check(lib().se2gpu_global_ba(self.h, N, ptr(T), ptr(fx), len(edges), ptr(fr), ptr(to), ptr(me), ptr(inf),
                                     C.addressof(prm), ptr(out), ptr(status), ptr(iters), ptr(stats), ptr(poses)), "se2gpu_global_ba")
        n = int(iters[0])
        return dict(status=int(status[0]), iterations=n, Tcw=out.reshape(N, 4, 4), poses=poses, stats=stats[:n].copy())


def GlobalBA(Tcw, fixed, edges, prm, device=0):
    """GlobalMapper::GlobalBA on a fresh context; see Context.run. There is no per-iteration pose trace: the per-iteration
    record is `stats` (chi2 before / after, lambda, rho, trials, accepted, terminate), and the tests hold the final double
    estimates (`poses`) to the oracle."""
    ctx = Context(device)
    try:
        return ctx.run(Tcw, fixed, edges, prm)
    finally:
        ctx.close()


def update_map_points(kf_index, view_mp, Tcw, device=0):
    """GlobalBA's map-point write-back: kf_index [M] (the main keyframe of each point), view_mp [M,3] (its mViewMPs entry),
    Tcw [N,4,4] (the keyframes' new poses). Returns pos [M,3] float32."""
    kf = np.ascontiguousarray(kf_index, np.int32).reshape(-1)
    v = np.ascontiguousarray(view_mp, np.float32).reshape(-1, 3)
    T = np.ascontiguousarray(Tcw, np.float32).reshape(-1, 16)
    assert len(v) == len(kf)
    pos = np.zeros((max(len(kf), 1), 3), np.float32)
    check(lib().se2gpu_global_ba_update_points(len(kf), ptr(kf), ptr(v), len(T), ptr(T), ptr(pos), device),
          "se2gpu_global_ba_update_points")
    return pos[:len(kf)]
