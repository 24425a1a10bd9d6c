"""Independent restatement of the localization oracle's own logic (oracle/loc_oracle.cpp) with Python sets and numpy float32
— TEST INFRASTRUCTURE ONLY. tests/test_loc_host.py runs oracle/pyloc.py's Localizer chain on each scene family once with
these functions and once with the C++ ones, and checks the two bit for bit.

Each function takes the map dict of se2lam_b200.loc (numpy arrays) and has the C++ function's signature in Python form.
"""
from __future__ import annotations

import numpy as np

F = np.float32


def _obs(m, k):
    return {int(v) for v in m["kf_obs"][m["kf_obs_ptr"][k]:m["kf_obs_ptr"][k + 1]]}


def pose(cfg, odom, ref_odom, ref_Tcw):
    """UpdatePoseCurr: the tracker's restated Se2 (glibc cosf / sinf through float32 numpy) and the float gemm order"""
    def norm(t):
        t = float(t)
        if -np.pi <= t < np.pi:
            return t
        t = t - np.floor(t / (2 * np.pi)) * 2 * np.pi
        if t >= np.pi:
            t -= 2 * np.pi
        if t < -np.pi:
            t += 2 * np.pi
        return t
    from oracle import pytrack                             # float32 cosf / sinf of glibc, as the reference calls them
    cosf, sinf = pytrack.lib().track_oracle_cosf, pytrack.lib().track_oracle_sinf
    o = [F(v) for v in odom]; r = [F(v) for v in ref_odom]
    o[2], r[2] = F(norm(o[2])), F(norm(r[2]))
    dx, dy = F(r[0] - o[0]), F(r[1] - o[1])
    dth = F(norm(F(r[2] - o[2])))
    c, s = F(cosf(o[2])), F(sinf(o[2]))
    x, y, th = F(F(c * dx) + F(s * dy)), F(F(-s * dx) + F(c * dy)), F(norm(dth))
    ct, st = F(cosf(th)), F(sinf(th))
    M = np.array([[ct, -st, 0, x], [st, ct, 0, y], [0, 0, 1, 0], [0, 0, 0, 1]], F)

    def mul(A, B):
        R = np.zeros((4, 4), F)
        for i in range(4):
            for j in range(4):
                t = F(A[i, 0] * B[0, j])
                for k in range(1, 4):
                    t = F(t + F(A[i, k] * B[k, j]))
                R[i, j] = t
        return R
    T = mul(mul(np.asarray(cfg["cTb"], F), M), np.asarray(cfg["bTc"], F))
    return mul(T, np.asarray(ref_Tcw, F))


def project(K, T, pos, bounds):
    """(in [n] u1, uv [n,2] f4): camprjc(K, se3map(T, pos)) with float sums from 0, inImgBound inclusive"""
    K, T, P = np.asarray(K, F), np.asarray(T, F), np.asarray(pos, F).reshape(-1, 3)
    c = [F(0) + T[r, 0] * P[:, 0] for r in range(3)]
    c = [(c[r] + T[r, 1] * P[:, 1]) + T[r, 2] * P[:, 2] + T[r, 3] for r in range(3)]
    q = [((F(0) + K[r, 0] * c[0]) + K[r, 1] * c[1]) + K[r, 2] * c[2] for r in range(3)]
    with np.errstate(divide="ignore", invalid="ignore"):
        u, v = (q[0] / q[2]).astype(F), (q[1] / q[2]).astype(F)
    x0, x1, y0, y1 = (F(b) for b in bounds)
    return ((u >= x0) & (u <= x1) & (v >= y0) & (v <= y1)).astype(np.uint8), np.stack([u, v], 1).astype(F)


def covis(m, local_kfs, obs_mp, cov):
    """UpdateCovisKFCurr: cov updated in place; returns the keyframes that sat on the integer boundary 10 * count == n"""
    cur = {int(v) for v in obs_mp if v >= 0}
    edge = 0
    for k in np.flatnonzero(local_kfs):
        c = len(cur & _obs(m, int(k)))
        if c > 0.1 * len(cur):
            cov[k] = 1
        elif 10 * c == len(cur):
            edge += 1
    return edge


def local_map(m, cov, hops, cap):
    """UpdateLocalMap(hops): (local_kfs [K] u1, ascending list (at most cap), full count)"""
    K = len(m["kf_kp_ptr"]) - 1
    kfs = {int(k) for k in np.flatnonzero(cov)}
    for _ in range(hops):
        for k in set(kfs):
            kfs |= {int(v) for v in m["kf_cov"][m["kf_cov_ptr"][k]:m["kf_cov_ptr"][k + 1]]}
    mps = set()
    for k in kfs:
        mps |= {j for j in _obs(m, k) if not m["mp_null"][j] and m["mp_good_prl"][j]}
    lk = np.zeros(K, np.uint8)
    lk[sorted(kfs)] = 1
    lst = sorted(mps)
    return lk, lst[:cap], len(lst)


def loop_close(m, kf, pairs, obs_mp):
    """MatchLoopClose: obs_mp updated in place; returns (null points skipped, points without good parallax taken)"""
    nulls = bad = 0
    for ic, il in sorted(dict(pairs).items()):
        j = int(m["kf_obs_mp"][m["kf_kp_ptr"][kf] + il])
        if j < 0:
            continue
        if m["mp_null"][j]:
            nulls += 1
            continue
        bad += int(not m["mp_good_prl"][j])
        obs_mp[ic] = j
    return nulls, bad
