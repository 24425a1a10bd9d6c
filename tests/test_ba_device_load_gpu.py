"""se2gpu_ba_set_problem_device: a local-BA window loaded from device buffers, its structure built on the device.

The bar is identity with the host entry: after a device load the context holds the same device arrays, element for
element, as after se2gpu_ba_set_problem of the same window (se2gpu_ba_debug_structure), the same plan apart from the
`structure` field, the same reduced system at a fixed lambda, and byte-identical optimize() stats, traces and estimates.
The windows are those the host build's own tests use (tests/ba_cases.py, both structure builds, every reduced solver),
one context across sequences of windows with both entries mixed, sharded contexts, rejected windows, the context's
stream, and the device Omega of se2gpu_ba_build_information_device."""
import ctypes as C

import numpy as np
import pytest
import torch

from se2lam_b200 import _capi
from se2lam_b200.ba import LocalBA
from tests import ba_cases as bc
from tests.local_shards import pk_grid_share, run_local_shards
from tests.test_ba_context_gpu import new_values, slide
from tools import synth

pytestmark = pytest.mark.gpu

ERR_INVALID, ERR_CAPACITY = -3, -4          # SE2GPU_ERR_INVALID, SE2GPU_ERR_CAPACITY
DEV = torch.device("cuda", 0)
FIELDS = ("poses", "fixed", "points", "edge_pose", "edge_point", "uv", "info", "odo_i", "odo_j", "odo_meas", "odo_info")
DTYPES = (torch.float64, torch.uint8, torch.float64, torch.int32, torch.int32, torch.float64, torch.float64, torch.int32,
          torch.int32, torch.float64, torch.float64)


def on_device(prob):
    """the window's arrays as contiguous CUDA tensors (a 1-element tensor stands in for an empty array)"""
    out = []
    for f, dt in zip(FIELDS, DTYPES):
        a = np.ascontiguousarray(getattr(prob, f)).reshape(-1)
        t = torch.from_numpy(a.copy()).to(dt) if a.size else torch.zeros(1, dtype=dt)
        out.append(t.to(DEV))
    torch.cuda.synchronize()
    return out


def device_load(ba, prob, tensors=None):
    t = on_device(prob) if tensors is None else tensors
    ba.set_problem_device(prob.P, prob.L, prob.E, prob.O, *t, prob.fx, prob.cx, prob.cy, prob.Tcb, prob.huber_delta)


def caps_of(probs):
    return (max(p.P for p in probs), max(max(p.L for p in probs), 1), max(max(p.E for p in probs), 1), max(max(p.O for p in probs), 1))


def structure(ba):
    return {k: ba.debug_structure(k).tobytes() for k in LocalBA.STRUCTURE_ARRAYS}


def plan_but_structure(ba):
    p = ba.debug_plan()
    p.pop("structure")
    return p


def assert_same_structure(got, want, what=""):
    sg, sw = structure(got), structure(want)
    for k in LocalBA.STRUCTURE_ARRAYS:
        assert sg[k] == sw[k], f"{what}{k} differs from the host load's"
    assert plan_but_structure(got) == plan_but_structure(want), f"{what}plan differs"


def run(ba, iters):
    n, st, tp, tl = ba.optimize(iters, trace=True)
    p, l = ba.get()
    return n, st.tobytes(), tp.tobytes(), tl.tobytes(), p.tobytes(), l.tobytes()


def system_bytes(ba, lam):
    s = ba.debug_system(lam)
    return {k: (v.tobytes() if isinstance(v, np.ndarray) else v) for k, v in s.items()}


def pair(prob, mode=0, caps=None):
    """a host-loaded and a device-loaded context of the same window"""
    caps = caps or caps_of([prob])
    h, d = LocalBA(*caps), LocalBA(*caps)
    for ba in (h, d):
        ba.set_mode(mode)
    h.set_problem(prob)
    device_load(d, prob)
    return h, d


def assert_identical(prob, iters, modes=(0, 1, 2), system=True):
    h, d = pair(prob)
    assert d.debug_plan()["structure"] == "device"
    assert_same_structure(d, h)
    if system:
        lam = 1e-3
        assert system_bytes(d, lam) == system_bytes(h, lam), "debug_system differs"
    for mode in modes:
        h.set_mode(mode); d.set_mode(mode)
        h.reset(); d.reset()
        try:
            want = run(h, iters)
        except _capi.Se2GpuError:               # persistent mode unavailable for this window: the device load refuses too
            with pytest.raises(_capi.Se2GpuError):
                run(d, iters)
            continue
        assert run(d, iters) == want, f"mode {mode}: optimize differs"
    return h.debug_plan()


# ------------------------------------------------------------------------------------------------ 1. array for array
STRICT_NAMES = ["twist_w6", "twist_w16", "smem_w17", "chain_nf16", "smem_nf52", "large_nf53", "band_w1", "band_w6", "env_w11",
                "dense_nf29", "dense_arena", "tail_nf23", "tail_nf59", "broken_nf29", "reversed_nf28", "duplicated_nf28",
                "loop_nf39", "loop_nf79", "sparse_nf29"]


@pytest.mark.parametrize("name", STRICT_NAMES)
def test_reference_shaped_windows(name):
    prob, iters = bc.strict(name)
    assert_identical(prob, min(iters, 6))


@pytest.mark.parametrize("case", ["nonpd", "edge_permuted"])
def test_non_pd_and_permuted_edges(case):
    base = synth.ba_window(30, 1500, seed=3)
    prob = bc.nonpd(base) if case == "nonpd" else bc.edge_permuted(base, seed=4)
    assert_identical(prob, 6)


@pytest.mark.parametrize("cfg", ["C3", "C4"])
def test_c3_c4(cfg):
    assert_identical(synth.ba_config(cfg), 10)


def test_c5_like():
    plan = assert_identical(synth.ba_config("C5"), 2, modes=(0,), system=False)
    assert plan["structure"] == "dense" and plan["nf"] > 1000


def test_sorted_structure_window():
    """nf > 2048: the host takes its comparison-sorted build; the device build is the same for both"""
    prob, _ = bc.strict("sorted_w10")
    plan = assert_identical(prob, 2, modes=(0,), system=False)
    assert plan["structure"] == "sorted"


@pytest.mark.parametrize("env,name,solver", [("SE2GPU_BA_NO_TWIST", "twist_w10", "smem"), ("SE2GPU_BA_NO_BAND", "band_w4", "envelope")])
def test_switches_choose_the_same_solver(env, name, solver, monkeypatch):
    monkeypatch.setenv(env, "1")
    prob, iters = bc.strict(name)
    plan = assert_identical(prob, min(iters, 6))
    assert plan["solver"] == solver


# ------------------------------------------------------------------------------------------- 2. one context, many windows
def fresh_host(prob, caps, mode):
    ba = LocalBA(*caps)
    ba.set_mode(mode)
    ba.set_problem(prob)
    return ba


def check_step(ba, prob, caps, mode, iters=6):
    ref = fresh_host(prob, caps, mode)
    assert_same_structure(ba, ref)
    assert run(ba, iters) == run(ref, iters)
    ref.close()


@pytest.mark.parametrize("mode", [1, 2], ids=["multi-launch", "persistent"])
@pytest.mark.parametrize("mix", ["device", "alternating"])
def test_sliding_window_and_refresh(mode, mix):
    traj = synth.ba_window(40, 4000, seed=21)
    windows = [slide(traj, s, 14) for s in range(0, 20, 4)]
    windows.insert(2, new_values(windows[1], 5, camera=True))       # same topology: the values-only refresh
    drop = bc._copy(windows[3]); bc._keep_edges(drop, np.arange(drop.E) % 7 != 3)    # outlier edges removed, then reloaded
    windows[4:4] = [drop, windows[3]]
    caps = caps_of(windows)
    ba = LocalBA(*caps)
    ba.set_mode(mode)
    for k, w in enumerate(windows):
        if mix == "device" or k % 2 == 0:
            device_load(ba, w)
        else:
            ba.set_problem(w)
        check_step(ba, w, caps, mode)


@pytest.mark.parametrize("mode", [0, 1], ids=["auto", "multi-launch"])
def test_grow_shrink_and_degenerate_windows(mode):
    small = synth.ba_window(8, 400, seed=31)
    big = bc.strict("tail_nf59")[0]
    band = bc.strict("band_w3")[0]
    no_free = bc._copy(small); no_free.fixed[:] = 1
    no_edges = bc._copy(small); bc._keep_edges(no_edges, np.zeros(small.E, bool))
    no_odo = bc._copy(small); bc._keep_odo(no_odo, np.zeros(small.O, bool))
    orphans = bc._copy(small); bc._keep_edges(orphans, small.edge_point % 3 != 0)
    seq = [small, big, no_free, band, no_edges, small, no_odo, orphans, big, small]
    caps = caps_of(seq)
    ba = LocalBA(*caps)
    ba.set_mode(mode)
    for k, w in enumerate(seq):
        device_load(ba, w) if k % 3 != 2 else ba.set_problem(w)
        check_step(ba, w, caps, mode, iters=4)


def test_mode_switches_after_device_loads():
    a = synth.ba_config("C3")
    h, d = pair(a, mode=1)
    for mode in (1, 2, 0, 1):
        h.set_mode(mode); d.set_mode(mode)
        h.reset(); d.reset()
        assert run(d, 5) == run(h, 5)


# ------------------------------------------------------------------------------------------------------------ 3. shards
@pytest.mark.parametrize("world", [2, 3])
@pytest.mark.parametrize("path", ["multi-launch", "persistent"])
def test_sharded_device_loads(world, path, monkeypatch):
    prob = bc.strict("tail_nf23")[0]
    monkeypatch.setenv("SE2GPU_BA_PK_GRID", pk_grid_share(world))
    mode = 1 if path == "multi-launch" else 0

    def setup(bas, device):
        if path == "persistent":
            LocalBA.attach_local(bas)
        if device:
            for ba in bas:
                device_load(ba, prob)

    want = run_local_shards(prob, world, 6, mode=mode, setup=lambda bas: setup(bas, False))
    got = run_local_shards(prob, world, 6, mode=mode, setup=lambda bas: setup(bas, True))
    for r in range(world):
        assert got[r][0] == want[r][0]
        for a, b in zip(got[r][1:], want[r][1:]):
            assert a.tobytes() == b.tobytes(), f"rank {r} differs"


def test_sharded_structure_equals_host():
    prob = bc.strict("reversed_nf28")[0]
    for world in (2, 3):
        for rank in range(world):
            h, d = LocalBA(*caps_of([prob])), LocalBA(*caps_of([prob]))
            for ba in (h, d):
                ba.set_shard(rank, world, lambda *a: None)
            h.set_problem(prob)
            device_load(d, prob)
            assert_same_structure(d, h, f"rank {rank}/{world}: ")


# ------------------------------------------------------------------------------------------------------------ 4. errors
def assert_nothing_loaded(ba):
    lib = _capi.lib()
    st = np.zeros(4, _capi.BA_STATS_DTYPE)
    p = np.zeros((64, 3))
    assert lib.se2gpu_ba_optimize_from(ba.h, 0, 4, None, _capi.ptr(st), None, None) == ERR_INVALID
    assert lib.se2gpu_ba_get(ba.h, _capi.ptr(p), _capi.ptr(p)) == ERR_INVALID
    assert lib.se2gpu_ba_debug_structure(ba.h, 0, None, 0) == ERR_INVALID


def raw_load(ba, prob, tensors, **override):
    ptrs = [_capi.ptr(t) for t in tensors]
    for k, v in override.items():
        ptrs[FIELDS.index(k)] = v
    tcb = np.ascontiguousarray(prob.Tcb, np.float64)
    return _capi.lib().se2gpu_ba_set_problem_device(ba.h, prob.P, prob.L, prob.E, prob.O, *ptrs, prob.fx, prob.cx, prob.cy,
                                                    _capi.ptr(tcb), prob.huber_delta)


def test_rejected_windows_leave_none_loaded():
    a = synth.ba_window(10, 600, seed=12)
    caps = caps_of([a])
    lib = _capi.lib()
    bad = []
    for field, k, v in (("edge_pose", 3, a.P), ("edge_pose", 0, -1), ("edge_point", 5, a.L), ("edge_point", 1, -7),
                        ("odo_i", 2, a.P + 5), ("odo_j", 0, -1)):
        q = bc._copy(a); getattr(q, field)[k] = v
        bad.append((q, ERR_INVALID, {}))
    bad.append((a, ERR_INVALID, {"edge_point": None}))
    bad.append((a, ERR_INVALID, {"odo_info": None}))
    bad.append((a, ERR_INVALID, {"poses": None}))
    ba = LocalBA(*caps)
    for q, rc, override in bad:
        device_load(ba, a)
        assert raw_load(ba, q, on_device(q), **override) == rc, _capi.last_error()
        assert_nothing_loaded(ba)
        device_load(ba, a)                                  # the pre-failure topology: rebuilt, equal to a fresh host load
        check_step(ba, a, caps, 0)
    too_big = synth.ba_window(caps[0] + 2, 600, seed=14)
    with pytest.raises(_capi.Se2GpuError, match=rf"\({ERR_CAPACITY}\)"):
        device_load(ba, too_big)
    assert_nothing_loaded(ba)
    assert lib.se2gpu_ba_set_problem_device(ba.h, 0, 1, 1, 1, *([None] * 11), 1.0, 0.0, 0.0, None, 1.0) == ERR_INVALID
    assert lib.se2gpu_ba_debug_structure(None, 0, None, 0) == ERR_INVALID


# ------------------------------------------------------------------------------------------------------- 5. the stream
def test_inputs_written_on_the_context_stream():
    prob = synth.ba_config("C3")
    ref = fresh_host(prob, caps_of([prob]), 0)
    stream = torch.cuda.Stream(device=DEV)
    ba = LocalBA(*caps_of([prob]))
    ba.set_stream(stream.cuda_stream)
    host = on_device(prob)
    with torch.cuda.stream(stream):
        torch.cuda._sleep(20_000_000)                       # the inputs are written well after the call is made
        t = [torch.empty_like(x) for x in host]
        for dst, src in zip(t, host):
            dst.copy_(src)
        device_load(ba, prob, t)
        for x in t:                                         # overwritten right after the call returns
            x.fill_(0) if x.dtype != torch.float64 else x.fill_(float("nan"))
    stream.synchronize()
    assert_same_structure(ba, ref)
    assert run(ba, 8) == run(ref, 8)


# ---------------------------------------------------------------------------------------------------- 6. Omega on the device
def omega_inputs(prob, seed=3):
    rng = np.random.default_rng(seed)
    E, P, L = prob.E, prob.P, prob.L
    view = rng.uniform([-2, -1, 2], [2, 1, 8], (E, 3)).astype(np.float32)
    Rcw = np.stack([np.linalg.qr(rng.normal(size=(3, 3)))[0] for _ in range(P)]).astype(np.float32).reshape(P, 9)
    twb = rng.normal(0, 3, (P, 2)).astype(np.float32)
    pos = rng.normal(0, 5, (L, 3)).astype(np.float32)
    octave = rng.integers(0, 8, E).astype(np.int32)
    sig2 = (1.2 ** (2 * np.arange(8))).astype(np.float32)
    return view, Rcw, twb, pos, octave, sig2


def test_build_information_device_and_the_device_chain():
    prob = synth.ba_config("C3")
    view, Rcw, twb, pos, octave, sig2 = omega_inputs(prob)
    lib = _capi.lib()
    ep, lp = np.ascontiguousarray(prob.edge_pose, np.int32), np.ascontiguousarray(prob.edge_point, np.int32)
    info_h = np.zeros((prob.E, 3))
    args = (500.0, 1e6, 1.0)
    assert lib.se2gpu_ba_build_information(prob.P, prob.L, prob.E, _capi.ptr(view), _capi.ptr(ep), _capi.ptr(lp), _capi.ptr(octave),
                                           _capi.ptr(Rcw), _capi.ptr(twb), _capi.ptr(pos), _capi.ptr(sig2), 8, *args,
                                           _capi.ptr(info_h), 0) == 0
    d = [torch.from_numpy(x).to(DEV) for x in (view, ep, lp, octave, Rcw, twb, pos, sig2)]
    info_d = torch.zeros((prob.E, 3), dtype=torch.float64, device=DEV)
    stream = torch.cuda.current_stream(DEV).cuda_stream
    assert lib.se2gpu_ba_build_information_device(prob.P, prob.L, prob.E, *[_capi.ptr(x) for x in d[:7]], _capi.ptr(d[7]), 8,
                                                  *args, _capi.ptr(info_d), C.c_void_p(stream)) == 0
    torch.cuda.synchronize()
    assert info_d.cpu().numpy().tobytes() == info_h.tobytes()
    # Omega -> set_problem_device -> optimize equals the host chain
    q = bc._copy(prob); q.info = info_h
    ref = fresh_host(q, caps_of([q]), 0)
    t = on_device(q)
    t[FIELDS.index("info")] = info_d.reshape(-1)
    ba = LocalBA(*caps_of([q]))
    device_load(ba, q, t)
    assert run(ba, 8) == run(ref, 8)
    # out-of-range indices: NaN information, no fault
    bad = d[1].clone(); bad[0] = prob.P + 100
    assert lib.se2gpu_ba_build_information_device(prob.P, prob.L, prob.E, _capi.ptr(d[0]), _capi.ptr(bad), *[_capi.ptr(x) for x in d[2:7]],
                                                  _capi.ptr(d[7]), 8, *args, _capi.ptr(info_d), C.c_void_p(stream)) == 0
    torch.cuda.synchronize()
    out = info_d.cpu().numpy()
    assert np.isnan(out[0]).all() and out[1:].tobytes() == info_h[1:].tobytes()
