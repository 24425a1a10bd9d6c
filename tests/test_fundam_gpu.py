"""Track::removeOutliers on the GPU (se2gpu_remove_outliers[_device]) against the oracle, bit for bit: matches12 after
the call, nInlier, F and the number of hypotheses run, on every scene of tests/golden/fundam_golden.npz."""
import ctypes as C

import numpy as np
import pytest

from oracle import pyfundam
from se2lam_b200 import _capi
from se2lam_b200._capi import KP_DTYPE
from se2lam_b200.geometry import removeOutliers
from tests import fundam_cases

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def cases():
    out = []
    for s in fundam_cases.load():
        kp1, kp2, m = s.keypoints(KP_DTYPE)
        out.append((s, kp1, kp2, m, pyfundam.remove_outliers(kp1, kp2, m)))
    return out


def _check(got, want, tag):
    nin, m, F, it = got
    wn, wm, wF, wit = want
    assert nin == wn and np.array_equal(m, wm), tag
    assert F.tobytes() == wF.tobytes(), (tag, F, wF)
    assert it == wit, (tag, it, wit)


def test_batches_of_64_equal_the_oracle(cases):
    for a in range(0, len(cases), 64):
        chunk = cases[a:a + 64]
        res = removeOutliers([c[1] for c in chunk], [c[2] for c in chunk], [c[3] for c in chunk], return_details=True)
        for c, r in zip(chunk, res):
            _check(r, c[4], (c[0].i, c[0].n, c[0].branch))


def test_pair_by_pair_equals_the_oracle(cases):
    for c in cases[::3]:
        _check(removeOutliers(c[1], c[2], c[3], return_details=True), c[4], (c[0].i, c[0].n))


def test_inputs_not_modified_and_all_unmatched(cases):
    s, kp1, kp2, m, _ = cases[-1]
    m0 = m.copy()
    nin, out = removeOutliers(kp1, kp2, np.full_like(m, -1))
    assert nin == 0 and (out == -1).all() and np.array_equal(m, m0)


def test_device_entry_with_counts_below_capacity(cases):
    torch = pytest.importorskip("torch")
    sel = [c for c in cases if 15 <= c[0].n <= 300][:48] + [c for c in cases if c[0].n in (0, 7, 9)][:16]
    B = len(sel)
    cap1 = max(len(c[1]) for c in sel) + 13; cap2 = max(len(c[2]) for c in sel) + 5
    k1 = np.zeros((B, cap1), KP_DTYPE); k2 = np.zeros((B, cap2), KP_DTYPE); m = np.full((B, cap1), 77, np.int32)
    n1 = np.array([len(c[1]) for c in sel], np.int32); n2 = np.array([len(c[2]) for c in sel], np.int32)
    for b, c in enumerate(sel):
        k1[b, :n1[b]] = c[1]; k2[b, :n2[b]] = c[2]; m[b, :n1[b]] = c[3]
    dev = torch.device("cuda:0")
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a).view(np.uint8) if a.dtype == KP_DTYPE else a).to(dev)
    dk1, dk2, dm, dn1, dn2 = t(k1), t(k2), t(m), t(n1), t(n2)
    dnin = torch.zeros(B, dtype=torch.int32, device=dev); dF = torch.zeros(B * 9, dtype=torch.float64, device=dev)
    dit = torch.zeros(B, dtype=torch.int32, device=dev)
    stream = torch.cuda.current_stream(dev).cuda_stream
    rc = _capi.lib().se2gpu_remove_outliers_device(B, _capi.ptr(dk1), _capi.ptr(dn1), cap1, _capi.ptr(dk2), _capi.ptr(dn2), cap2,
                                                    _capi.ptr(dm), _capi.ptr(dnin), _capi.ptr(dF), _capi.ptr(dit), C.c_void_p(stream))
    _capi.check(rc, "se2gpu_remove_outliers_device")
    torch.cuda.synchronize()
    mm, nin, F, it = dm.cpu().numpy(), dnin.cpu().numpy(), dF.cpu().numpy().reshape(B, 3, 3), dit.cpu().numpy()
    for b, c in enumerate(sel):
        _check((int(nin[b]), mm[b, :n1[b]], F[b], int(it[b])), c[4], c[0].i)
        assert (mm[b, n1[b]:] == 77).all()          # entries past the count are not touched


def test_invalid_arguments():
    L = _capi.lib()
    kp = np.zeros(4, KP_DTYPE); m = np.array([0, 1, 5, -1], np.int32); nin = np.zeros(1, np.int32)
    p = _capi.ptr
    assert L.se2gpu_remove_outliers(-1, p(kp), None, 4, p(kp), None, 4, p(m), p(nin), None, None, 0) == -3
    assert L.se2gpu_remove_outliers(1, p(kp), None, 4, p(kp), None, 4, p(m), p(nin), None, None, 0) == -3   # 5 >= n2
    assert L.se2gpu_remove_outliers(1, p(kp), None, 4, p(kp), None, 4, p(m), None, None, None, 0) == -3
    big = np.zeros(8193, KP_DTYPE); mb = np.full(8193, -1, np.int32)
    assert L.se2gpu_remove_outliers(1, p(big), None, 8193, p(kp), None, 4, p(mb), p(nin), None, None, 0) == -4
    assert L.se2gpu_remove_outliers_device(1, None, None, 4, None, None, 4, None, None, None, None, None) == -3
    assert L.se2gpu_remove_outliers(0, None, None, 0, None, None, 0, None, None, None, None, 0) == 0


def test_device_niters_lookup_equals_libm_exhaustively():
    L = _capi.lib()
    for lo in range(1, 8193, 2048):
        hi = min(lo + 2047, 8192)
        n = np.concatenate([np.full(k + 1, k, np.int32) for k in range(lo, hi + 1)])
        good = np.concatenate([np.arange(k + 1, dtype=np.int32) for k in range(lo, hi + 1)])
        M = np.full(len(n), 1000, np.int32); out = np.zeros(len(n), np.int32)
        _capi.check(L.se2gpu_fundam_debug_niters(len(n), _capi.ptr(n), _capi.ptr(good), _capi.ptr(M), _capi.ptr(out), 0), "niters")
        assert np.array_equal(out, pyfundam.niters_range(lo, hi, 1000)), lo
