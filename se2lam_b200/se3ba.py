"""The SE(3)-XYZ window BA on the GPU: the graph of Map::loadLocalGraph / loadLocalGraphOnlyBa under g2o's
Levenberg-Marquardt, with LocalMapper::removeOutlierChi2's per-edge chi2 cut, through se2gpu_se3_ba. numpy in, numpy out;
there is no CPU fallback."""
from __future__ import annotations

import ctypes as C

import numpy as np

from ._capi import BA_STATS_DTYPE, SE3BAParams, check, lib, ptr

OK, NOT_PD = 0, 2


def params(fx, cx, cy, Tbc, huber_delta, xrot_info=1e6, yrot_info=1e6, z_info=1.0, iterations=10, chi2_cut=25.0):
    """se2gpu_se3_ba_params: the camera (Config::Kcam), Config::bTc [4,4], Config::TH_HUBER, the PLANEMOTION_* informations,
    optimize(iterations) (10 in removeOutlierChi2) and the outlier cut (25 there)."""
    p = SE3BAParams()
    p.fx, p.cx, p.cy = fx, cx, cy
    p.Tbc[:] = [float(v) for v in np.asarray(Tbc, np.float32).reshape(16)]
    p.huber_delta, p.xrot_info, p.yrot_info, p.z_info = huber_delta, xrot_info, yrot_info, z_info
    p.iterations, p.chi2_cut = iterations, chi2_cut
    return p


class Window:
    """A flattened window. Tcw [N,4,4]; fixed [N]; prior [N] (the plane-motion prior; all zero for loadLocalGraphOnlyBa);
    odometry: odo_from / odo_to [O], odo_measure [O,4,4], odo_info [O,6,6] in KeyFrame's [trans rot] order; xyz [L,3];
    edges: edge_point / edge_kf [E], uv [E,2], inv_sigma2 [E]."""

    def __init__(self, Tcw, fixed, prior, xyz, edge_point, edge_kf, uv, inv_sigma2, odo_from=(), odo_to=(), odo_measure=None,
                 odo_info=None):
        self.Tcw = np.ascontiguousarray(Tcw, np.float32).reshape(-1, 16)
        N = len(self.Tcw)
        self.fixed = np.ascontiguousarray(fixed, np.uint8).reshape(N)
        self.prior = np.ascontiguousarray(prior, np.uint8).reshape(N)
        self.odo_from = np.ascontiguousarray(odo_from, np.int32).reshape(-1)
        self.odo_to = np.ascontiguousarray(odo_to, np.int32).reshape(-1)
        O = len(self.odo_from)
        self.odo_measure = np.ascontiguousarray(np.zeros((0, 16)) if odo_measure is None else odo_measure, np.float32).reshape(O, 16)
        self.odo_info = np.ascontiguousarray(np.zeros((0, 36)) if odo_info is None else odo_info, np.float32).reshape(O, 36)
        self.xyz = np.ascontiguousarray(xyz, np.float32).reshape(-1, 3)
        self.edge_point = np.ascontiguousarray(edge_point, np.int32).reshape(-1)
        self.edge_kf = np.ascontiguousarray(edge_kf, np.int32).reshape(-1)
        E = len(self.edge_point)
        self.uv = np.ascontiguousarray(uv, np.float32).reshape(E, 2)
        self.inv_sigma2 = np.ascontiguousarray(inv_sigma2, np.float32).reshape(E)

    @property
    def sizes(self):
        return len(self.Tcw), len(self.odo_from), len(self.xyz), len(self.edge_point)


class Context:
    """se2gpu_se3_ba_ctx: grow-only device buffers and a stream, reusable across windows of any size."""

    def __init__(self, device=0):
        self.h = lib().se2gpu_se3_ba_create(device)
        if not self.h:
            check(-1, "se2gpu_se3_ba_create")

    def close(self):
        if self.h:
            lib().se2gpu_se3_ba_destroy(self.h)
            self.h = None

    def __del__(self):
        self.close()

    def run(self, w: Window, prm, trace=False):
        """One optimize(prm.iterations) of the window. Returns dict(status, iterations, chi2 [E] (raw, at the final
        estimate), outlier [E] bool, poses [N,7] (qx, qy, qz, qw, tx, ty, tz), points [L,3] double, Tcw [N,4,4] float32,
        xyz [L,3] float32, stats, and with trace=True trace [iterations, N*7 + L*3] instead of Tcw / xyz)."""
        N, O, L, E = w.sizes
        chi2 = np.zeros(max(E, 1)); outl = np.zeros(max(E, 1), np.uint8)
        status = np.zeros(1, np.int32); iters = np.zeros(1, np.int32)
        stats = np.zeros(max(prm.iterations, 1), BA_STATS_DTYPE)
        poses = np.zeros((N, 7)); points = np.zeros((max(L, 1), 3))
        head = (self.h, N, ptr(w.Tcw), ptr(w.fixed), ptr(w.prior), O, ptr(w.odo_from), ptr(w.odo_to), ptr(w.odo_measure),
                ptr(w.odo_info), L, ptr(w.xyz), E, ptr(w.edge_point), ptr(w.edge_kf), ptr(w.uv), ptr(w.inv_sigma2),
                C.addressof(prm), ptr(chi2), ptr(outl), ptr(status), ptr(iters), ptr(stats), ptr(poses), ptr(points))
        out = {}
        if trace:
            tr = np.zeros((max(prm.iterations, 1), 7 * N + 3 * L))
            check(lib().se2gpu_se3_ba_debug_trace(*head, ptr(tr)), "se2gpu_se3_ba_debug_trace")
        else:
            T = np.zeros((N, 16), np.float32); X = np.zeros((max(L, 1), 3), np.float32)
            check(lib().se2gpu_se3_ba(*head, ptr(T), ptr(X)), "se2gpu_se3_ba")
            out.update(Tcw=T.reshape(N, 4, 4), xyz=X[:L])
        n = int(iters[0])
        out.update(status=int(status[0]), iterations=n, chi2=chi2[:E], outlier=outl[:E].astype(bool), poses=poses,
                   points=points[:L], stats=stats[:n].copy())
        if trace:
            out["trace"] = tr[:n]
        return out

    def run_device(self, w: Window, prm, stream=None):
        """The device entry on torch CUDA tensors of the window's values (topology stays on the host); returns the same
        dict as run() without Tcw / xyz / stats' padding, after a synchronise of the stream."""
        import torch
        N, O, L, E = w.sizes
        dev = torch.device("cuda")
        t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)  # noqa: E731
        dT, dm, di, dx, du, dw = t(w.Tcw), t(w.odo_measure), t(w.odo_info), t(w.xyz), t(w.uv), t(w.inv_sigma2)
        chi2 = torch.zeros(max(E, 1), dtype=torch.float64, device=dev)
        outl = torch.zeros(max(E, 1), dtype=torch.uint8, device=dev)
        status = torch.zeros(1, dtype=torch.int32, device=dev); iters = torch.zeros(1, dtype=torch.int32, device=dev)
        stats = torch.zeros(max(prm.iterations, 1) * BA_STATS_DTYPE.itemsize, dtype=torch.uint8, device=dev)
        poses = torch.zeros((N, 7), dtype=torch.float64, device=dev)
        points = torch.zeros((max(L, 1), 3), dtype=torch.float64, device=dev)
        T = torch.zeros((N, 16), dtype=torch.float32, device=dev); X = torch.zeros((max(L, 1), 3), dtype=torch.float32, device=dev)
        s = stream if stream is not None else torch.cuda.current_stream()
        check(lib().se2gpu_se3_ba_device(self.h, N, ptr(dT), ptr(w.fixed), ptr(w.prior), O, ptr(w.odo_from), ptr(w.odo_to), ptr(dm),
                                         ptr(di), L, ptr(dx), E, ptr(w.edge_point), ptr(w.edge_kf), ptr(du), ptr(dw),
                                         C.addressof(prm), ptr(chi2), ptr(outl), ptr(status), ptr(iters), ptr(stats), ptr(poses),
                                         ptr(points), ptr(T), ptr(X), C.c_void_p(s.cuda_stream)), "se2gpu_se3_ba_device")
        s.synchronize()
        n = int(iters.cpu()[0])
        st = np.frombuffer(stats.cpu().numpy().tobytes(), BA_STATS_DTYPE)
        return dict(status=int(status.cpu()[0]), iterations=n, chi2=chi2.cpu().numpy()[:E], outlier=outl.cpu().numpy()[:E].astype(bool),
                    poses=poses.cpu().numpy(), points=points.cpu().numpy()[:L], Tcw=T.cpu().numpy().reshape(N, 4, 4),
                    xyz=X.cpu().numpy()[:L], stats=st[:n].copy())


def local_se3_ba(w: Window, prm, device=0):
    """One call on a fresh context; see Context.run."""
    ctx = Context(device)
    try:
        return ctx.run(w, prm)
    finally:
        ctx.close()


def outlier_lists(w: Window, outlier):
    """removeOutlierChi2's vnOutlierIdxAll: for every point, the keyframes of its edges flagged as outliers, in edge order."""
    lists = [[] for _ in range(len(w.xyz))]
    for e in np.nonzero(np.asarray(outlier))[0]:
        lists[int(w.edge_point[e])].append(int(w.edge_kf[e]))
    return lists
