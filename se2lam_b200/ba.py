"""Host-side mirror of the reference's local-BA interface over the C ABI (se2gpu_ba_*).

Two layers:
* `LocalBA`          — thin object over se2gpu_ba_create/set_problem/optimize/get (SoA in, SoA out).
* `SlamOptimizer` +  — the subset of the g2o graph API that se2lam's local BA drives
  free functions       (reference include/se2lam/optimizer.h:77-110,140-141 and src/Map.cpp:891-1053,
                       src/LocalMapper.cpp:232-302): addCamPara, addVertexSE2, addEdgeSE2,
                       addVertexSBAXYZ, addEdgeSE2XYZ, initializeOptimization, optimize,
                       estimateVertexSE2, estimateVertexSBAXYZ — same names, argument order and meaning.
No CPU fallback: everything numerical happens in the CUDA library.
"""
from __future__ import annotations

import ctypes as C

import numpy as np

from . import _capi
from ._capi import BA_STATS_DTYPE, check, lib, ptr


class LocalBA:
    def __init__(self, max_poses, max_points, max_edges, max_odo, device=0):
        self.h = lib().se2gpu_ba_create(max_poses, max_points, max_edges, max(max_odo, 1), device)
        if not self.h:
            raise _capi.Se2GpuError("se2gpu_ba_create failed: " + _capi.last_error())
        self.P = self.L = self.E = self.O = 0
        self._cb = None

    def close(self):
        if getattr(self, "h", None):
            lib().se2gpu_ba_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:      # interpreter shutdown: module globals may already be gone
            pass

    @classmethod
    def from_problem(cls, prob, device=0, rank=0, world=1, allreduce=None, stream=None, mode=0):
        ba = cls(prob.P, max(prob.L, 1), max(prob.E, 1), max(prob.O, 1), device)
        ba.set_mode(mode)
        if stream is not None:
            ba.set_stream(stream)
        if world > 1:
            ba.set_shard(rank, world, allreduce)
        ba.set_problem(prob)
        return ba

    def set_stream(self, stream):
        check(lib().se2gpu_ba_set_stream(self.h, C.c_void_p(int(stream) if stream else 0)), "se2gpu_ba_set_stream")

    def set_shard(self, rank, world, allreduce):
        """allreduce(dev_ptr:int, count:int, op:int(0 sum,1 max), stream:int) -> None; must be ordered on `stream`."""
        def _cb(user, buf, count, op, stream):
            try:
                allreduce(int(buf), int(count), int(op), int(stream or 0))
                return 0
            except Exception as e:  # never let an exception cross the C boundary
                print("allreduce callback failed:", e)
                return 1
        self._cb = _capi.ALLREDUCE_FN(_cb)
        check(lib().se2gpu_ba_set_shard(self.h, rank, world, self._cb, None), "se2gpu_ba_set_shard")

    def enable_peer_exchange(self, all_gather):
        """Fused exchange of the reduced system over NVLink peer mappings (se2gpu_ba_peer_export/_import).
        all_gather(local: bytes) -> list[bytes] in rank order (e.g. torch.distributed.all_gather_object)."""
        n = _capi.PEER_HANDLE_BYTES
        mine = (C.c_uint8 * n)()
        check(lib().se2gpu_ba_peer_export(self.h, mine), "se2gpu_ba_peer_export")
        parts = all_gather(bytes(mine))
        blob = b"".join(parts)
        buf = (C.c_uint8 * len(blob)).from_buffer_copy(blob)
        check(lib().se2gpu_ba_peer_import(self.h, buf, len(parts)), "se2gpu_ba_peer_import")

    def set_problem(self, prob):
        c = np.ascontiguousarray
        a = [c(prob.poses, np.float64), c(prob.fixed, np.uint8), c(prob.points, np.float64), c(prob.edge_pose, np.int32),
             c(prob.edge_point, np.int32), c(prob.uv, np.float64), c(prob.info, np.float64), c(prob.odo_i, np.int32),
             c(prob.odo_j, np.int32), c(prob.odo_meas, np.float64), c(prob.odo_info, np.float64)]
        tcb = c(prob.Tcb, np.float64)
        self.P = self.L = self.E = self.O = 0          # a failed load leaves no window (se2gpu_ba_set_problem)
        check(lib().se2gpu_ba_set_problem(self.h, prob.P, prob.L, prob.E, prob.O, *[ptr(x) for x in a],
                                          float(prob.fx), float(prob.cx), float(prob.cy), ptr(tcb),
                                          float(prob.huber_delta)), "se2gpu_ba_set_problem")
        self.P, self.L, self.E, self.O = prob.P, prob.L, prob.E, prob.O

    def set_problem_device(self, P, L, E, O, poses, fixed, points, edge_pose, edge_point, uv, info, odo_i, odo_j, odo_meas,
                           odo_info, fx, cx, cy, Tcb, huber_delta):
        """set_problem from device memory (se2gpu_ba_set_problem_device): the same fields in the same order and layout, as
        torch CUDA tensors or raw device pointers (float64 / uint8 / int32 as in set_problem); Tcb [12] stays on the host.
        The structure is built on the device; the arrays are read on the context's stream (set_stream)."""
        tcb = np.ascontiguousarray(Tcb, np.float64)
        arrays = [poses, fixed, points, edge_pose, edge_point, uv, info, odo_i, odo_j, odo_meas, odo_info]
        self.P = self.L = self.E = self.O = 0          # a failed load leaves no window
        check(lib().se2gpu_ba_set_problem_device(self.h, int(P), int(L), int(E), int(O), *[ptr(x) for x in arrays], float(fx),
                                                 float(cx), float(cy), ptr(tcb), float(huber_delta)), "se2gpu_ba_set_problem_device")
        self.P, self.L, self.E, self.O = int(P), int(L), int(E), int(O)

    STRUCTURE_ARRAYS = ("hidx", "lm_ptr", "perm", "e_pose", "e_hidx", "pose_ptr", "pose_edges", "pose_odo_ptr", "pose_odo", "blk_a",
                        "blk_b", "blk_pair_ptr", "pair_e1", "pair_e2", "blk_odo_ptr", "blk_odo", "colmax", "tw_cmax1", "blk_order",
                        "env_idx", "odo_i", "odo_j", "e_u", "e_v", "e_w00", "e_w01", "e_w11", "odo_m", "odo_w")
    STRUCTURE_DOUBLES = ("e_u", "e_v", "e_w00", "e_w01", "e_w11", "odo_m", "odo_w")

    def debug_structure(self, which):
        """One device array of the loaded window (se2gpu_ba_debug_structure) by name; int32, or float64 for the values."""
        k = self.STRUCTURE_ARRAYS.index(which)
        n = check(lib().se2gpu_ba_debug_structure(self.h, k, None, 0), "se2gpu_ba_debug_structure")
        out = np.zeros(n, np.int32)
        check(lib().se2gpu_ba_debug_structure(self.h, k, ptr(out), n), "se2gpu_ba_debug_structure")
        return out.view(np.float64) if which in self.STRUCTURE_DOUBLES else out

    def optimize(self, iters, trace=False, stop_flag=None, first_iteration=0):
        """first_iteration > 0 continues the lambda / nu schedule of the previous call (g2o's solve(iteration) slices)."""
        st = np.zeros(max(iters, 1), BA_STATS_DTYPE)
        tp = np.zeros((max(iters, 1), self.P, 3)) if trace else None
        tl = np.zeros((max(iters, 1), self.L, 3)) if trace else None
        n = check(lib().se2gpu_ba_optimize_from(self.h, int(first_iteration), iters, ptr(stop_flag), ptr(st), ptr(tp), ptr(tl)),
                  "se2gpu_ba_optimize_from")
        return (n, st[:n], tp[:n], tl[:n]) if trace else (n, st[:n])

    @staticmethod
    def optimize_batch(bas, iters, trace=False, stop_flags=None):
        """Optimise the windows loaded in the contexts `bas` together (se2gpu_ba_optimize_batch): one thread-block cluster per
        window, one launch per cluster size. Returns, per window, what `optimize(iters, trace)` returns. stop_flags: None or
        one uint8 array of length 1 (or None) per window."""
        B = len(bas)
        arr = (C.c_void_p * B)(*[b.h if b is not None else None for b in bas])
        st = np.zeros((B, max(iters, 1)), BA_STATS_DTYPE)
        its = np.zeros(B, np.int32)
        flags = None if stop_flags is None else (C.c_void_p * B)(*[ptr(f) for f in stop_flags])
        tp = tl = tpa = tla = None
        if trace:          # a None context gets no trace buffer; the library refuses it and names the window
            tp = [np.zeros((max(iters, 1), b.P, 3)) if b is not None else None for b in bas]
            tl = [np.zeros((max(iters, 1), b.L, 3)) if b is not None else None for b in bas]
            tpa = (C.c_void_p * B)(*[ptr(x) for x in tp])
            tla = (C.c_void_p * B)(*[ptr(x) for x in tl])
        check(lib().se2gpu_ba_optimize_batch(arr, B, int(iters), flags, ptr(its), ptr(st), tpa, tla), "se2gpu_ba_optimize_batch")
        out = []
        for k in range(B):
            n = int(its[k])
            out.append((n, st[k, :n], tp[k][:n], tl[k][:n]) if trace else (n, st[k, :n]))
        return out

    def batch_cluster(self):
        """Cluster size (CTAs) optimize_batch runs the loaded window on (se2gpu_ba_batch_cluster)."""
        return check(lib().se2gpu_ba_batch_cluster(self.h), "se2gpu_ba_batch_cluster")

    @staticmethod
    def attach_local(bas):
        """Peer exchange between several contexts of THIS process (one per GPU, or several on one GPU): rank order."""
        arr = (C.c_void_p * len(bas))(*[b.h for b in bas])
        check(lib().se2gpu_ba_peer_attach_local(arr, len(bas)), "se2gpu_ba_peer_attach_local")

    def get_f32(self):
        """Estimates narrowed on the device like Map::optimizeLocalGraph's write-back (Map.cpp:768-779)."""
        poses = np.zeros((self.P, 3), np.float32); pts = np.zeros((self.L, 3), np.float32)
        check(lib().se2gpu_ba_get_f32(self.h, ptr(poses), ptr(pts)), "se2gpu_ba_get_f32")
        return poses, pts

    PROFILE_GROUPS = ("ba_linearize", "ba_pose_reduce", "ba_lm_prep", "ba_schur", "ba_chol_solve", "ba_backsub_update", "ba_lm_control",
                      "ba_persistent", "ba_stage_S")
    MODE_AUTO, MODE_MULTI_LAUNCH, MODE_PERSISTENT = 0, 1, 2

    def set_mode(self, mode):
        check(lib().se2gpu_ba_set_mode(self.h, int(mode)), "se2gpu_ba_set_mode")

    def reset(self):
        check(lib().se2gpu_ba_reset(self.h), "se2gpu_ba_reset")

    def profile(self, enable=True):
        check(lib().se2gpu_ba_profile(self.h, int(enable)), "se2gpu_ba_profile")

    def profile_read(self):
        ms = np.zeros(len(self.PROFILE_GROUPS)); n = np.zeros(len(self.PROFILE_GROUPS), np.int32)
        check(lib().se2gpu_ba_profile_read(self.h, ptr(ms), ptr(n)), "se2gpu_ba_profile_read")
        return {g: (float(ms[i]), int(n[i])) for i, g in enumerate(self.PROFILE_GROUPS)}

    def get(self):
        poses = np.zeros((self.P, 3)); pts = np.zeros((self.L, 3))
        check(lib().se2gpu_ba_get(self.h, ptr(poses), ptr(pts)), "se2gpu_ba_get")
        return poses, pts

    def debug_system(self, lam):
        out = {}
        chi = C.c_double()
        # first call to learn n
        n = check(lib().se2gpu_ba_debug_system(self.h, lam, C.byref(chi), *([None] * 9)), "se2gpu_ba_debug_system")
        out.update(Hpp=np.zeros((n, n)), bp=np.zeros(n), Hll=np.zeros((self.L, 3, 3)), bl=np.zeros((self.L, 3)),
                   Hpl=np.zeros((self.E, 3, 3)), S=np.zeros((n, n)), bs=np.zeros(n), dx_p=np.zeros(n), dx_l=np.zeros((self.L, 3)))
        check(lib().se2gpu_ba_debug_system(self.h, lam, C.byref(chi), ptr(out["Hpp"]), ptr(out["bp"]), ptr(out["Hll"]),
                                           ptr(out["bl"]), ptr(out["Hpl"]), ptr(out["S"]), ptr(out["bs"]), ptr(out["dx_p"]),
                                           ptr(out["dx_l"])), "se2gpu_ba_debug_system")
        out["chi2"] = chi.value
        out["n"] = n
        return out

    PLAN_FIELDS = ("nf", "n", "structure", "env_w", "solver", "tw_m0", "tw_w", "band_w", "band_p", "pk_grid", "workers",
                   "nblk", "max_own", "uncached")
    STRUCTURES = ("dense", "sorted", "device")
    SOLVERS = ("smem", "twisted", "band", "envelope")

    def debug_plan(self):
        """Host-side decisions of the last set_problem (se2gpu_ba_debug_plan): structure build, reduced solver and the
        persistent kernel's Schur work split. `structure` and `solver` are returned as names."""
        buf = np.zeros(len(self.PLAN_FIELDS), np.int32)
        nf = check(lib().se2gpu_ba_debug_plan(self.h, ptr(buf), len(buf)), "se2gpu_ba_debug_plan")
        if nf != len(buf):
            raise _capi.Se2GpuError(f"se2gpu_ba_debug_plan reports {nf} fields, the binding knows {len(buf)}")
        out = {k: int(v) for k, v in zip(self.PLAN_FIELDS, buf)}
        out["structure"] = self.STRUCTURES[out["structure"]]
        out["solver"] = self.SOLVERS[out["solver"]]
        return out


# ------------------------------------------------------------------------------------------------
# g2o-graph-style facade (the calls Map::loadLocalGraph / LocalMapper::localBA make)
# ------------------------------------------------------------------------------------------------
class CamPara:
    def __init__(self, fx, cx, cy):
        self.focal_length, self.principle_point = float(fx), (float(cx), float(cy))


class SlamOptimizer:
    """Collects an SE(2)-XYZ graph and runs it on the GPU. SE(3) vertex/edge types are out of scope."""

    def __init__(self, device=0):
        self.device = device
        self.clear()
        self._stop = None
        self._verbose = False
        self._ba = None

    # graph container -----------------------------------------------------------------------------
    def clear(self):
        self._vse2, self._vxyz, self._eodo, self._exyz = {}, {}, [], []
        self._cam = None
        self._ba = None
        self._maps = None

    def clearParameters(self):
        self._cam = None

    def setVerbose(self, v):
        self._verbose = bool(v)

    def setForceStopFlag(self, flag):
        """flag: numpy uint8 array of length 1 written by another thread (LocalMapper::mbAbortBA)."""
        self._stop = flag

    def setAlgorithm(self, _solver):  # the solver stack is fixed: LM + Schur + Cholesky on the GPU
        pass

    # optimisation --------------------------------------------------------------------------------
    def initializeOptimization(self, level=0):
        pose_ids = sorted(self._vse2)
        pt_ids = sorted(self._vxyz)
        pmap = {vid: k for k, vid in enumerate(pose_ids)}
        lmap = {vid: k for k, vid in enumerate(pt_ids)}
        from .problem import BAProblem
        cam = self._cam
        if cam is None:
            raise _capi.Se2GpuError("addCamPara was not called")
        Tcb = None
        ex = self._exyz
        if ex:
            Tcb = ex[0]["Tcb"]
            delta = ex[0]["delta"]
        else:
            Tcb = np.concatenate([np.eye(3).reshape(-1), np.zeros(3)]); delta = 1.0
        prob = BAProblem(
            poses=np.array([self._vse2[i]["est"] for i in pose_ids], np.float64).reshape(-1, 3),
            fixed=np.array([self._vse2[i]["fixed"] for i in pose_ids], np.uint8),
            points=np.array([self._vxyz[i]["est"] for i in pt_ids], np.float64).reshape(-1, 3),
            edge_pose=np.array([pmap[e["v0"]] for e in ex], np.int32), edge_point=np.array([lmap[e["v1"]] for e in ex], np.int32),
            uv=np.array([e["meas"] for e in ex], np.float64).reshape(-1, 2),
            info=np.array([(e["info"][0, 0], 0.5 * (e["info"][0, 1] + e["info"][1, 0]), e["info"][1, 1]) for e in ex], np.float64).reshape(-1, 3),
            odo_i=np.array([pmap[e["v0"]] for e in self._eodo], np.int32), odo_j=np.array([pmap[e["v1"]] for e in self._eodo], np.int32),
            odo_meas=np.array([e["meas"] for e in self._eodo], np.float64).reshape(-1, 3),
            odo_info=np.array([[e["info"][0, 0], e["info"][0, 1], e["info"][0, 2], e["info"][1, 1], e["info"][1, 2], e["info"][2, 2]]
                               for e in self._eodo], np.float64).reshape(-1, 6),
            fx=cam.focal_length, cx=cam.principle_point[0], cy=cam.principle_point[1], Tcb=np.asarray(Tcb, np.float64),
            huber_delta=float(delta))
        self._maps = (pose_ids, pt_ids)
        self._ba = LocalBA.from_problem(prob, device=self.device)
        self.stats = None
        return True

    def optimize(self, iterations):
        if self._ba is None:
            print("optimize: 0 vertices to optimize, maybe forgot to call initializeOptimization()")
            return -1
        n, st = self._ba.optimize(iterations, stop_flag=self._stop)
        self.stats = st
        if self._verbose:
            for k, s in enumerate(st):
                print(f"iteration= {k}\t chi2= {s['chi2_after']:.6f}\t lambda= {s['lambda']:.6f}\t levenbergIter= {s['trials']}")
        poses, pts = self._ba.get()
        pose_ids, pt_ids = self._maps
        for k, vid in enumerate(pose_ids):
            self._vse2[vid]["est"] = poses[k].copy()
        for k, vid in enumerate(pt_ids):
            self._vxyz[vid]["est"] = pts[k].copy()
        return n


def initOptimizer(opt: SlamOptimizer, verbose=False):                      # optimizer.cpp:199-205
    opt.setVerbose(verbose)


def addCamPara(opt: SlamOptimizer, K, id=0):                               # optimizer.cpp:207-215
    K = np.asarray(K, np.float32)
    opt._cam = CamPara(K[0, 0], K[0, 2], K[1, 2])
    return opt._cam


def addVertexSE2(opt: SlamOptimizer, pose, id, fixed=False):               # optimizer.cpp:34-43
    opt._vse2[int(id)] = dict(est=np.asarray(pose, np.float64).reshape(3).copy(), fixed=bool(fixed))


def estimateVertexSE2(opt: SlamOptimizer, id):                             # optimizer.cpp:45-50
    return opt._vse2[int(id)]["est"].copy()


def addEdgeSE2(opt: SlamOptimizer, meas, id0, id1, info):                  # optimizer.cpp:52-62 (PreEdgeSE2)
    opt._eodo.append(dict(meas=np.asarray(meas, np.float64).reshape(3), v0=int(id0), v1=int(id1),
                          info=np.asarray(info, np.float64).reshape(3, 3)))


def addVertexSBAXYZ(opt: SlamOptimizer, xyz, id, marginal=True, fixed=False):  # optimizer.cpp:316-324
    if not marginal or fixed:
        raise _capi.Se2GpuError("only marginalised, free VertexSBAPointXYZ are supported (as Map.cpp:988 creates them)")
    opt._vxyz[int(id)] = dict(est=np.asarray(xyz, np.float64).reshape(3).copy())


def estimateVertexSBAXYZ(opt: SlamOptimizer, id):                          # optimizer.cpp:549-554
    return opt._vxyz[int(id)]["est"].copy()


def addEdgeSE2XYZ(opt: SlamOptimizer, meas, id0, id1, campara, Tbc, info, thHuber):  # optimizer.cpp:17-32
    """Tbc = (Rbc 3x3, tbc 3) body<-camera extrinsic; the edge uses Tcb = Tbc^-1 (EdgeSE2XYZ.h:52)."""
    Rbc, tbc = Tbc
    Rbc = np.asarray(Rbc, np.float64).reshape(3, 3)
    Rcb = Rbc.T
    tcb = -Rcb @ np.asarray(tbc, np.float64).reshape(3)
    opt._exyz.append(dict(meas=np.asarray(meas, np.float64).reshape(2), v0=int(id0), v1=int(id1),
                          info=np.asarray(info, np.float64).reshape(2, 2), delta=float(thHuber),
                          Tcb=np.concatenate([Rcb.reshape(-1), tcb])))
