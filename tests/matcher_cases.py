"""Shared synthetic cases for the matcher tests (CPU oracle tests and GPU parity tests)."""
import numpy as np

from oracle.pyoracle import KP_DTYPE

f32 = np.float32
GRID_COLS, GRID_ROWS = 64, 48           # Frame.h:26-27
GRID = (f32(0.0), f32(0.0), f32(f32(64) / f32(640.0)), f32(f32(48) / f32(480.0)))

# Frame::computeBoundUn (Frame.cpp:187-205) of a 640x480 frame: cv::undistortPoints of the four image corners for
# K = [[520.9, 0, 325.1], [0, 521.0, 249.7], [0, 0, 1]], D = (0.2312, -0.7849, -0.0033, -0.0001, 0.9172), the camera of
# tests/test_orb_gpu.py::test_undistort_folded_into_level0. (minX, minY, maxX, maxY): a non-zero origin, non-round cells.
UNDIST_BOUNDS = (f32(12.059211), f32(11.455164), f32(629.42035), f32(473.11594))


def grid_of(minX, maxX, minY, maxY):
    """(minX, minY, invW, invH) as Frame.cpp:40-41 (and FrameView.grid()) compute them, in float32."""
    minX, maxX, minY, maxY = f32(minX), f32(maxX), f32(minY), f32(maxY)
    return (minX, minY, f32(f32(GRID_COLS) / f32(maxX - minX)), f32(f32(GRID_ROWS) / f32(maxY - minY)))


UNDIST_GRID = grid_of(UNDIST_BOUNDS[0], UNDIST_BOUNDS[2], UNDIST_BOUNDS[1], UNDIST_BOUNDS[3])


def round_half_away(v):
    """C++ round() of float32 values: halves go away from zero (-0.5 -> -1). In float64, v + 0.5 is exact."""
    v = np.asarray(v, np.float64)
    return (np.sign(v) * np.floor(np.abs(v) + 0.5)).astype(int)


def grid_pos(kp, grid):
    """Frame::PosInGrid (Frame.cpp:209-220) of every keypoint: (posX, posY, inside)."""
    minX, minY, invW, invH = (f32(g) for g in grid)
    px = round_half_away(((kp["x"] - minX) * invW).astype(f32))
    py = round_half_away(((kp["y"] - minY) * invH).astype(f32))
    return px, py, (px >= 0) & (px < GRID_COLS) & (py >= 0) & (py < GRID_ROWS)


def half_cell_coords(lo, inv, halves, reach=256):
    """{h: v} with float32 v such that fl(fl(v - lo) * inv) == h exactly, searched among the `reach` float32 neighbours on
    each side of lo + h / inv; halves that no float32 coordinate hits exactly are left out."""
    lo, inv = f32(lo), f32(inv)
    h = np.asarray(halves, np.float64)
    up = (float(lo) + h / float(inv)).astype(f32)
    dn = up.copy()
    found = np.full(len(h), np.nan, f32)
    for _ in range(reach):
        for v in (up, dn):
            hit = np.isnan(found) & (((v - lo) * inv).astype(f32) == h)
            found[hit] = v[hit]
        up, dn = np.nextafter(up, f32(np.inf)), np.nextafter(dn, f32(-np.inf))
    return {float(hh): f32(v) for hh, v in zip(h, found) if not np.isnan(v)}


def empty_window_positions(grid, r):
    """Window centres (x, y) whose GetFeaturesInArea window lies entirely left of, right of, above and below the grid: the
    reference returns before visiting a cell (nMaxCellX < 0, nMinCellX >= 64, ...). Also the centres one pixel inside each
    of those limits, whose window reaches the first / last column or row."""
    minX, minY, invW, invH = (float(g) for g in grid)
    maxX, maxY = minX + GRID_COLS / invW, minY + GRID_ROWS / invH
    cx, cy = (minX + maxX) / 2, (minY + maxY) / 2
    left, right = minX - r - 1.0 / invW, maxX + r
    above, below = minY - r - 1.0 / invH, maxY + r
    out = [(left - 1, cy), (left - 40, cy + 30), (right + 1, cy), (right + 25, cy - 30),
           (cx, above - 1), (cx + 30, above - 35), (cx, below + 1), (cx - 30, below + 20)]
    inside = [(left + 1, cy), (right - 1, cy), (cx, above + 1), (cx, below - 1)]
    return np.asarray(out, f32), np.asarray(inside, f32)


def _flip(rng, d, nbits):
    for b in rng.choice(256, nbits, replace=False):
        d[b // 8] ^= np.uint8(1 << (b % 8))


def _edge_database(rng, n, grid):
    """n keypoints over the grid and a 30 px margin around it (so some lie left of it - negative x among them - right of
    it, above it and below its last row), then keypoints exactly on half cells in x and in y: -0.5 (round() puts it in
    cell -1: outside), 63.5 / 47.5 (cell 64 / 48: outside) and every half in between that a float32 coordinate hits."""
    minX, minY, invW, invH = grid
    maxX, maxY = f32(minX + f32(GRID_COLS / float(invW))), f32(minY + f32(GRID_ROWS / float(invH)))
    kp = random_keypoints(rng, n)
    kp["x"] = rng.uniform(float(minX) - 30, float(maxX) + 30, n).astype(f32)
    kp["y"] = rng.uniform(float(minY) - 30, float(maxY) + 30, n).astype(f32)
    hx = half_cell_coords(minX, invW, np.arange(-1, GRID_COLS) + 0.5)
    hy = half_cell_coords(minY, invH, np.arange(-1, GRID_ROWS) + 0.5)
    assert {-0.5, GRID_COLS - 0.5} <= set(hx) and {-0.5, GRID_ROWS - 0.5} <= set(hy), "grid has no exact half-cell coordinates"
    k = 0
    for v in hx.values():
        kp["x"][k], kp["y"][k] = v, f32(rng.uniform(float(minY) + 25, float(maxY) - 25)); k += 1
    for v in hy.values():
        kp["x"][k], kp["y"][k] = f32(rng.uniform(float(minX) + 25, float(maxX) - 25)), v; k += 1
    return kp, k, hx, hy


def make_grid_edge_pair(seed=21, n=700, grid=UNDIST_GRID, win=20.0):
    """MatchByWindow on a grid with a non-zero origin and non-round cells: frame 2 = `_edge_database`, frame 1 = its keypoints
    shuffled with a few descriptor bits flipped, searched around their frame-2 position (so the half-cell and outside
    keypoints of frame 2 have a query that matches them when the grid holds them), plus queries whose window lies outside
    the grid or just reaches its edge."""
    rng = np.random.default_rng(seed)
    kp2, _, _, _ = _edge_database(rng, n, grid)
    d2 = rng.integers(0, 256, (n, 32), dtype=np.uint8)
    perm = rng.permutation(n)
    kp1 = kp2[perm].copy()
    kp1["angle"] = np.mod(kp1["angle"] - f32(9.0) + rng.normal(0, 2, n).astype(f32), 360).astype(f32)
    d1 = d2[perm].copy()
    for i in range(n):
        _flip(rng, d1[i], int(rng.integers(0, 16)))
    prev = np.stack([kp1["x"] + rng.normal(0, 1.5, n).astype(f32), kp1["y"] + rng.normal(0, 1.5, n).astype(f32)], axis=1).astype(f32)
    out, inside = empty_window_positions(grid, win)
    q = rng.choice(n, len(out) + len(inside), replace=False)
    prev[q] = np.concatenate([out, inside])
    dup = rng.choice(n, 60, replace=False)           # near-duplicates in frame 2: "already matched better" and steals
    kp2[dup[:30]] = kp2[dup[30:]]
    d2[dup[:30]] = d2[dup[30:]] ^ rng.integers(0, 2, (30, 32), dtype=np.uint8)
    return dict(kp=kp1, desc=d1), dict(kp=kp2, desc=d2), prev.copy(), dict(empty=q[:len(out)], edge=q[len(out):])


def random_keypoints(rng, n):
    kp = np.zeros(n, KP_DTYPE)
    octave = np.minimum(rng.geometric(0.35, n) - 1, 7)
    scale = (f32(1.2) ** octave).astype(f32)
    kp["x"] = (rng.integers(16, 500, n).astype(f32) * scale).clip(0, 639.5)
    kp["y"] = (rng.integers(16, 380, n).astype(f32) * scale).clip(0, 479.5)
    kp["octave"] = octave
    kp["angle"] = rng.uniform(0, 360, n).astype(f32)
    kp["size"] = 31 * scale
    kp["response"] = rng.integers(20, 120, n)
    kp["class_id"] = -1
    return kp


def make_frame_pair(seed=1, n=900, shift=(6.0, -4.0), drot=7.0, flip=12):
    """frame2 = frame1 moved by `shift` px with a few descriptor bits flipped, shuffled, plus clutter."""
    rng = np.random.default_rng(seed)
    kp1 = random_keypoints(rng, n)
    d1 = rng.integers(0, 256, (n, 32), dtype=np.uint8)
    perm = rng.permutation(n)
    kp2 = kp1[perm].copy()
    kp2["x"] = (kp2["x"] + f32(shift[0]) + rng.normal(0, 1.5, n).astype(f32)).astype(f32)
    kp2["y"] = (kp2["y"] + f32(shift[1]) + rng.normal(0, 1.5, n).astype(f32)).astype(f32)
    kp2["angle"] = np.mod(kp2["angle"] + f32(drot) + rng.normal(0, 2, n).astype(f32), 360).astype(f32)
    d2 = d1[perm].copy()
    for i in range(n):
        bits = rng.integers(0, 256, rng.integers(0, 2 * flip))
        for b in bits:
            d2[i, b // 8] ^= np.uint8(1 << (b % 8))
    # duplicates / near-duplicates so that the "already matched better" and steal-back paths fire
    dup = rng.choice(n, 120, replace=False)
    kp2[dup[:60]] = kp2[dup[60:]]
    d2[dup[:60]] = d2[dup[60:]] ^ rng.integers(0, 2, (60, 32), dtype=np.uint8)
    prev = np.stack([kp1["x"], kp1["y"]], axis=1).astype(f32).copy()
    return dict(kp=kp1, desc=d1), dict(kp=kp2, desc=d2), prev


def brute_candidates(kp2, x, y, r, min_level, max_level, grid=GRID):
    """GetFeaturesInArea by explicit grid construction (Frame.cpp:64-77, 222-286) in numpy float32; grid = (minX, minY, invW, invH)."""
    minX, minY, invW, invH = (f32(g) for g in grid)
    posx, posy, _ = grid_pos(kp2, grid)
    x, y, r = f32(x), f32(y), f32(r)
    x0 = max(0, int(np.floor(f32(f32(f32(x - f32(minX)) - r) * invW)))); x1 = min(63, int(np.ceil(f32(f32(f32(x - f32(minX)) + r) * invW))))
    y0 = max(0, int(np.floor(f32(f32(f32(y - f32(minY)) - r) * invH)))); y1 = min(47, int(np.ceil(f32(f32(f32(y - f32(minY)) + r) * invH))))
    if x0 >= 64 or x1 < 0 or y0 >= 48 or y1 < 0:
        return []
    out = []
    for ix in range(x0, x1 + 1):
        for iy in range(y0, y1 + 1):
            for i in np.flatnonzero((posx == ix) & (posy == iy)):
                if not (min_level == -1 and max_level == -1):
                    if kp2["octave"][i] < min_level or kp2["octave"][i] > max_level:
                        continue
                if abs(f32(kp2["x"][i] - x)) > r or abs(f32(kp2["y"][i] - y)) > r:
                    continue
                out.append(int(i))
    return out


def make_projection_case(seed=2, n=900, nmp=700):
    rng = np.random.default_rng(seed)
    kp = random_keypoints(rng, n)
    desc = rng.integers(0, 256, (n, 32), dtype=np.uint8)
    src = rng.integers(0, n, nmp)
    mp_uv = np.stack([kp["x"][src] + rng.normal(0, 4, nmp), kp["y"][src] + rng.normal(0, 4, nmp)], axis=1).astype(f32)
    mp_octave = np.clip(kp["octave"][src] + rng.integers(-1, 2, nmp), 0, 7).astype(np.int32)
    mp_desc = desc[src].copy()
    flips = rng.integers(0, 256, (nmp, 20))
    for i in range(nmp):
        for b in flips[i, :rng.integers(0, 20)]:
            mp_desc[i, b // 8] ^= np.uint8(1 << (b % 8))
    mp_valid = (rng.random(nmp) > 0.1).astype(np.uint8)
    kf_observed = (rng.random(n) < 0.15).astype(np.uint8)
    return dict(args=dict(kfkp=kp, kfdesc=desc, kf_observed=kf_observed, mp_valid=mp_valid, mp_uv=mp_uv, mp_octave=mp_octave,
                          mp_desc=mp_desc, grid=GRID, win_size=15, level_offset=2, nnratio=0.6))


def make_projection_edge_case(seed=22, n=700, nmp=500, grid=UNDIST_GRID, win_size=15, level_offset=2, nnratio=0.6, ntie=8):
    """MatchByProjection on a grid with a non-zero origin: the keyframe is `_edge_database` (every half-cell keypoint gets
    a map point predicted onto it), map points predicted around random keypoints, map points whose window lies outside the
    grid or just reaches its edge, and ORDER TIES: keypoint B and, at a higher index, keypoint A with the same
    descriptor at another octave, A exactly on an even half cell (round() puts it in B's cell, round-half-even one cell
    earlier) and B 0.3 cells further in the same row (column ties) or column (row ties). The map point between them sees
    best == best2 at different levels, accepts, and takes whichever the grid walk visits first (B)."""
    rng = np.random.default_rng(seed)
    minX, minY, invW, invH = grid
    kp, nhalf, hx, hy = _edge_database(rng, n, grid)
    desc = rng.integers(0, 256, (n, 32), dtype=np.uint8)
    kp["octave"][:nhalf] = rng.integers(1, 5, nhalf)       # octave 0 would make the window 0 px
    # order ties at the end of the keyframe: B = 2t + base, A = B + 1
    even_x = [h for h in hx if h > 0 and int(h) % 2 == 0][:ntie]
    even_y = [h for h in hy if h > 0 and int(h) % 2 == 0][:ntie]
    assert len(even_x) >= 4 and len(even_y) >= 4, "grid has too few even half cells"
    base = n - 2 * (len(even_x) + len(even_y))
    ties = []
    for t, (h, axis) in enumerate([(h, 0) for h in even_x] + [(h, 1) for h in even_y]):
        b, a = base + 2 * t, base + 2 * t + 1
        lo, inv = (minX, invW) if axis == 0 else (minY, invH)
        va = (hx if axis == 0 else hy)[h]
        vb = f32(float(lo) + (h + 0.3) / float(inv))
        other = f32(rng.uniform(float(minY) + 40, float(minY) + 400)) if axis == 0 else f32(rng.uniform(float(minX) + 40, float(minX) + 550))
        for i, v in ((a, va), (b, vb)):
            kp["x"][i], kp["y"][i] = (v, other) if axis == 0 else (other, v)
        kp["octave"][a], kp["octave"][b] = 1, 2
        desc[a] = desc[b]
        ties.append((b, a))
    # map points: one per half-cell keypoint, one per tie, the rest around random keypoints
    src_half = np.arange(nhalf)
    nrand = nmp - nhalf - len(ties) - 12
    src = rng.integers(nhalf, base, nrand)
    uv = [np.stack([kp["x"][src_half], kp["y"][src_half]], axis=1)]
    octv = [kp["octave"][src_half]]
    mdesc = [desc[src_half].copy()]
    uv.append(np.stack([(kp["x"][src] + rng.normal(0, 4, nrand)), (kp["y"][src] + rng.normal(0, 4, nrand))], axis=1))
    octv.append(np.clip(kp["octave"][src] + rng.integers(-1, 2, nrand), 0, 7))
    mdesc.append(desc[src].copy())
    b_i = np.array([b for b, _ in ties]); a_i = np.array([a for _, a in ties])
    uv.append(np.stack([(kp["x"][a_i] + kp["x"][b_i]) / 2, (kp["y"][a_i] + kp["y"][b_i]) / 2], axis=1))
    octv.append(np.full(len(ties), 2))
    mdesc.append(desc[b_i].copy())
    out, inside = empty_window_positions(grid, 2 * win_size)
    uv.append(np.concatenate([out, inside]))
    octv.append(np.full(12, 2))
    mdesc.append(desc[rng.integers(0, base, 12)].copy())
    mp_uv = np.concatenate(uv).astype(f32)
    mp_octave = np.concatenate(octv).astype(np.int32)
    mp_desc = np.concatenate(mdesc)
    for i in range(len(mp_desc)):
        _flip(rng, mp_desc[i], int(rng.integers(0, 12)))
    mp_valid = np.ones(len(mp_desc), np.uint8)
    mp_valid[nhalf + rng.choice(nrand, nrand // 10, replace=False)] = 0
    kf_observed = (rng.random(n) < 0.1).astype(np.uint8)
    kf_observed[:nhalf] = 0
    kf_observed[base:] = 0
    return dict(args=dict(kfkp=kp, kfdesc=desc, kf_observed=kf_observed, mp_valid=mp_valid, mp_uv=mp_uv, mp_octave=mp_octave,
                          mp_desc=mp_desc, grid=grid, win_size=win_size, level_offset=level_offset, nnratio=nnratio),
                ties=ties, tie_mps=nhalf + nrand + np.arange(len(ties)))


def make_projection_chain_case(seed=31, n=200, nmp=150, chain=48):
    """The projection version of a steal chain: `chain` valid map points predicted at keyframe keypoint 0, each closer to it in
    Hamming distance than the one before (50, 49, ..., 4) and the last two at the same distance. Keypoint 1 (same octave,
    20 bits further), keypoint 2 (octave 4, 10 bits further) and keypoint 3 (octave 0, 120 bits further) lie next to it.
    Even map points have octave 1 (15 px, levels 0-3): keypoint 1 is their second best at the same level, so the ratio rule
    rejects them while the distance to keypoint 0 is above 30. Odd map points have octave 2 (30 px, levels 0-4): keypoint 2 is
    their second best at another level, and they accept. The last map point cannot take keypoint 0 (vMatchesDistance is
    already equal) and takes keypoint 2 instead."""
    a = make_projection_case(seed=seed, n=n, nmp=nmp)["args"]
    rng = np.random.default_rng((seed, chain))
    kp, desc = a["kfkp"], a["kfdesc"]
    kp["x"][:4], kp["y"][:4], kp["octave"][:4] = [300, 305, 295, 300], [200, 200, 200, 205], [1, 1, 4, 0]
    bits = rng.permutation(256)
    r0, r12 = bits[:96], bits[96:]

    def flipped(d, b):
        d = d.copy()
        for x in b:
            d[x // 8] ^= np.uint8(1 << (x % 8))
        return d
    desc[1], desc[2], desc[3] = flipped(desc[0], r12[:20]), flipped(desc[0], r12[80:90]), flipped(desc[0], r12[:120])
    a["kf_observed"][:4] = 0
    for q in range(chain):
        d0 = max(50 - q, 50 - (chain - 2))
        a["mp_uv"][q] = (300 + 0.1 * q, 200)
        a["mp_octave"][q] = 1 if q % 2 == 0 else 2
        a["mp_desc"][q] = flipped(desc[0], r0[:d0])
        a["mp_valid"][q] = 1
    return a


def make_big_window_case(seed, nq, ndb):
    """MatchByWindow with a database larger than the query frame: make_frame_pair(nq), then frame 2 padded to ndb keypoints -
    half of the padding near-copies of frame-2 keypoints (moved up to a few pixels, 10-30 bits flipped: competing second
    bests), half random clutter."""
    f1, f2, prev = make_frame_pair(seed=seed, n=nq)
    rng = np.random.default_rng((seed, ndb))
    extra = ndb - nq
    src = rng.integers(0, nq, extra // 2)
    near = f2["kp"][src].copy()
    near["x"] = np.clip(near["x"] + rng.normal(0, 6, len(src)).astype(f32), 0, 639.5).astype(f32)
    near["y"] = np.clip(near["y"] + rng.normal(0, 6, len(src)).astype(f32), 0, 479.5).astype(f32)
    dnear = f2["desc"][src].copy()
    for i in range(len(src)):
        _flip(rng, dnear[i], int(rng.integers(10, 30)))
    kp2 = np.concatenate([f2["kp"], near, random_keypoints(rng, extra - len(src))])
    d2 = np.concatenate([f2["desc"], dnear, rng.integers(0, 256, (extra - len(src), 32), dtype=np.uint8)])
    return f1, dict(kp=kp2, desc=d2), prev


def make_big_projection_case(seed, n_kf, nmp, ntie=64):
    """make_projection_case at a large keyframe, plus ORDER TIES: pairs (B, A = B + n_kf / 2) of keypoints in one grid cell with
    the same descriptor at octaves 2 and 1, and a map point next to them (octave 2) that sees best == best2 at different
    levels, accepts, and takes whichever the grid walk visits first: B, the lower insertion index."""
    c = make_projection_case(seed=seed, n=n_kf, nmp=nmp)
    a = c["args"]
    rng = np.random.default_rng((seed, n_kf, ntie))
    kp, desc = a["kfkp"], a["kfdesc"]
    b_i = rng.choice(n_kf // 2, ntie, replace=False)
    a_i = b_i + n_kf // 2
    cx, cy = rng.integers(2, 62, ntie), rng.integers(2, 46, ntie)   # cell centres (10 px cells on the 640x480 grid)
    kp["x"][b_i], kp["y"][b_i] = (cx * 10 + 1).astype(f32), (cy * 10 - 1).astype(f32)
    kp["x"][a_i], kp["y"][a_i] = (cx * 10 - 1).astype(f32), (cy * 10 + 1).astype(f32)
    kp["octave"][b_i], kp["octave"][a_i] = 2, 1
    desc[a_i] = desc[b_i]
    a["kf_observed"][a_i] = 0
    a["kf_observed"][b_i] = 0
    q = np.arange(ntie)
    a["mp_uv"][q] = np.stack([cx * 10, cy * 10], axis=1).astype(f32)
    a["mp_octave"][q] = 2
    a["mp_valid"][q] = 1
    a["mp_desc"][q] = desc[b_i]
    for i in q:
        _flip(rng, a["mp_desc"][i], int(rng.integers(0, 8)))
    return a, list(zip(b_i.tolist(), a_i.tolist()))


def make_bow_case(seed=3, n=800, nnodes=120, n2_extra=0, chain=0):
    """KF2 = KF1 shuffled with a few descriptor bits flipped and 10 % of the features moved to nodes of one KF only.
    n2_extra: that many more KF2 features with random descriptors in KF1's nodes (a large database).
    chain: that many more KF1 features, all with the SAME descriptor c, in one extra node where KF2 holds g_0..g_7 at
    distances 2, 4, 7, 12, 21, 36, 61, 102 from c (each < 0.6 x the next). All of them want g_0 first; in the sequential loop
    the first takes it and every later one falls through to the nearest feature vbMatched2 leaves (g_1, g_2, ...)."""
    rng = np.random.default_rng(seed)

    def kf(desc, angle, node_of):
        nodes = np.unique(node_of)
        ptr = [0]; feat = []
        for nd in nodes:
            idx = np.flatnonzero(node_of == nd)
            feat.extend(idx.tolist()); ptr.append(len(feat))
        return dict(angle=angle.astype(f32), desc=desc, has_mp=(rng.random(len(desc)) < 0.8).astype(np.uint8), node=nodes.astype(np.int32),
                    ptr=np.asarray(ptr, np.int32), feat=np.asarray(feat, np.int32))
    if n2_extra or chain:
        k1, k2 = make_bow_case(seed, n, nnodes)
        rng = np.random.default_rng((seed, n2_extra, chain))     # not the stream the base case drew from
        a1, a2 = k1["angle"], k2["angle"]
        d1, d2 = k1["desc"], k2["desc"]
        node1 = np.repeat(k1["node"], np.diff(k1["ptr"]))[np.argsort(k1["feat"])]
        node2 = np.repeat(k2["node"], np.diff(k2["ptr"]))[np.argsort(k2["feat"])]
        if n2_extra:
            d2 = np.concatenate([d2, rng.integers(0, 256, (n2_extra, 32), dtype=np.uint8)])
            a2 = np.concatenate([a2, rng.uniform(0, 360, n2_extra).astype(f32)])
            node2 = np.concatenate([node2, rng.choice(k1["node"], n2_extra)])
        if chain:
            nd = (nnodes + 40) * 3
            c = rng.integers(0, 256, 32, dtype=np.uint8)
            g = np.repeat(c[None], 8, axis=0)
            bits = rng.permutation(256)
            for k, dist in enumerate((2, 4, 7, 12, 21, 36, 61, 102)):
                for b in bits[:dist]:
                    g[k, b // 8] ^= np.uint8(1 << (b % 8))
                bits = np.roll(bits, 29)
            ac = rng.uniform(0, 360, chain).astype(f32)
            d1 = np.concatenate([d1, np.repeat(c[None], chain, axis=0)])
            a1 = np.concatenate([a1, ac])
            node1 = np.concatenate([node1, np.full(chain, nd)])
            d2 = np.concatenate([d2, g])
            a2 = np.concatenate([a2, np.mod(ac[:8] + 11 + rng.normal(0, 3, 8), 360).astype(f32)])
            node2 = np.concatenate([node2, np.full(8, nd)])
        k1, k2 = kf(d1, a1, node1), kf(d2, a2, node2)
        if chain:
            k2["has_mp"][-8:] = 1
        return k1, k2
    d1 = rng.integers(0, 256, (n, 32), dtype=np.uint8)
    a1 = rng.uniform(0, 360, n)
    node1 = rng.integers(0, nnodes, n) * 3
    perm = rng.permutation(n)
    d2 = d1[perm].copy()
    for i in range(n):
        for b in rng.integers(0, 256, rng.integers(0, 24)):
            d2[i, b // 8] ^= np.uint8(1 << (b % 8))
    a2 = np.mod(a1[perm] + 11 + rng.normal(0, 3, n), 360)
    node2 = node1[perm].copy()
    moved = rng.random(n) < 0.1
    node2[moved] = rng.integers(0, nnodes + 20, moved.sum()) * 3 + 1     # nodes that exist in only one KF
    return kf(d1, a1, node1), kf(d2, a2, node2)
