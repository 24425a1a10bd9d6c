"""The global pose graph on graphs the seeded scenes of tests/test_global_ba_gpu.py never build: other fixed sets (none,
one in the middle or at the end, several that split the free graph, edges between fixed vertices, all fixed, all but one),
dense envelopes (a complete graph, a hub linked to every vertex of a loop) and the 256-thread strides of the kernel's loops.
The scenes are built here; the oracle (oracle/global_ba_oracle.cpp) is held to its numpy restatement on small members of
each family, and its own spread over every scene is measured against the bounds tests/test_global_ba_paths_gpu.py holds
the kernel to."""
import numpy as np
import pytest

from oracle import global_ba_numpy, pyfeat, pyglobal
from tests import test_global_ba_gpu as G
from tests import test_global_ba_oracle as O
from tools import featgraph_synth as FS
from tools import posegraph_synth as S


def fixed_at(g, *idx, every=False):
    """g with exactly the vertices idx fixed (every: all of them)."""
    f = np.ones(len(g["Tcw"]), np.uint8) if every else np.zeros(len(g["Tcw"]), np.uint8)
    f[list(idx)] = 1
    return dict(g, fixed=f)


def free_only(g, v):
    """g with every vertex fixed but v."""
    f = np.ones(len(g["Tcw"]), np.uint8)
    f[v] = 0
    return dict(g, fixed=f)


def link(g, rng, i, j):
    """A feature edge i -> j as posegraph_synth draws them: the true relative camera pose times a small perturbation, a
    random information inside InfoSE3's clamp range."""
    T = g["truth"]
    Z = S.perturb(rng, T[i].astype(float) @ S.inv(T[j].astype(float)), 0.005, 0.002)
    return (i, j, Z.astype(np.float32), S.info_matrix(rng))


def complete(seed, N):
    """Every pair of N vertices linked (odometry i -> i+1, feature edges i -> i+h for every other h); vertex 0 fixed, so
    the free graph is complete on N - 1 vertices and the first pivot column has N - 2 rows below it."""
    return S.graph(seed=seed, N=N, hops=tuple(range(2, N)))


def hub(seed, N, h):
    """A loop of N vertices, plus a feature edge between vertex h and every other vertex (h -> j above h, j -> h below)."""
    g = S.graph(seed=seed, N=N, kind="loop", hops=(2,))
    rng = np.random.default_rng(seed + 1000)
    g["edges"] = g["edges"] + [link(g, rng, min(h, j), max(h, j)) for j in range(N) if j != h]
    return g


def trimmed(seed, N, E, kind="loop"):
    """A graph of N vertices and exactly E edges: the odometry (cut to E when E < N - 1), then feature edges drawn from
    the graph's own without replacement, kept in their order."""
    g = S.graph(seed=seed, N=N, kind=kind, hops=(2, 3))
    odo, rest = g["edges"][:N - 1], g["edges"][N - 1:]
    if E <= N - 1:
        g["edges"] = odo[:E]
    else:
        keep = np.sort(np.random.default_rng(seed).choice(len(rest), E - (N - 1), replace=False))
        g["edges"] = odo + [rest[k] for k in keep]
    assert len(g["edges"]) == E
    return g


def split_chain(seed, N, cuts):
    """A chain with odometry only and the vertices in cuts fixed: the free graph falls into len(cuts) + 1 components, and
    each cut vertex has an edge into it (free -> fixed) and one out of it (fixed -> free)."""
    return fixed_at(S.graph(seed=seed, N=N, hops=()), *cuts)



def status_graph():
    """300 keyframes for the device entry's d_edge_status: two chains joined by one odometry edge (149 -> 150), each with
    a fixed vertex (0 and 225), and a last vertex (299) whose one edge is its odometry. Returns (graph, status [E]): the
    bridge and 299's edge are SE2GPU_FEAT_EDGE_TOO_FEW, as are 8 edges drawn at random, and 8 others carry status 2
    (NOT_PD), the first of them listed last in `counted`."""
    g = fixed_at(S.graph(seed=115, N=300, hops=(2, 3)), 0, 225)
    g["edges"] = [e for e in g["edges"] if (not (e[0] < 150 <= e[1]) or (e[0], e[1]) == (149, 150))
                  and (299 not in (e[0], e[1]) or (e[0], e[1]) == (298, 299))]
    E = len(g["edges"])
    pairs = [(e[0], e[1]) for e in g["edges"]]
    bridge, tail = pairs.index((149, 150)), pairs.index((298, 299))
    rng = np.random.default_rng(115)
    others = rng.permutation([k for k in range(E) if k not in (bridge, tail)])
    status = np.zeros(E, np.int32)
    status[[bridge, tail] + list(others[:8])] = 1
    status[others[8:16]] = 2
    return g, status


def without(g, drop):
    """g with the edges whose index is in drop left out."""
    drop = set(int(k) for k in drop)
    return dict(g, edges=[e for k, e in enumerate(g["edges"]) if k not in drop])


FEAT_COUNTS = {0: (9, 10, 11, 191, 192, 193, 12, 40), 1: (2, 3, 4, 191, 192, 193, 5, 40)}


def feat_graph():
    """A 200-keyframe chain seen through featgraph_synth's camera, and 24 keyframe pairs per CreateFeatEdge mode, each the
    true motion between keyframes a and a + 1 (mode 0 at a = 2, 10, ..., mode 1 at a = 6, 14, ...) with the point counts of
    FEAT_COUNTS in turn: both sides of min_points and of the 192-point staging. Returns (graph, {mode: [(a, b, pair)]})."""
    g = S.graph(seed=116, N=200, hops=(2, 3), Tbc=FS.TBC)
    pairs = {}
    for mode in (0, 1):
        pairs[mode] = []
        for k in range(24):
            a = 2 + 4 * mode + 8 * k
            n = FEAT_COUNTS[mode][k % 8]
            kw = dict(noise=0.3, outlier_share=0.1 if n >= 10 else 0.0, outlier_size=(0.2, 0.4)) if mode else {}
            pairs[mode].append((a, a + 1, FS.scene(500 + 50 * mode + k, n, motion=(0.3, 0.0, 0.03 * np.sin(0.2 * a)), **kw)))
    return g, pairs


def feat_graph_with_oracle_edges():
    """feat_graph with the feature-graph oracle's constraint of every pair that is not TOO_FEW."""
    g, pairs = feat_graph()
    edges = list(g["edges"])
    for mode in (0, 1):
        for a, b, p in pairs[mode]:
            o = pyfeat.run(mode, p["Tcw0"], p["Tcw1"], p["xyz"], p["z0"], p["z1"], p["info0"], p["info1"], pyfeat.params(Tbc=p["Tbc"]))
            if o["status"] != 1:
                edges.append((a, b, o["measure"], o["info"]))
    return dict(g, edges=edges)


SCENES = {
    # fixed sets
    "loop_none_fixed": lambda: fixed_at(S.graph(seed=101, N=120, kind="loop")),
    "covisibility_none_fixed": lambda: fixed_at(S.graph(seed=102, N=60, hops=(2, 3, 4, 5, 6))),
    "loop_fixed_middle": lambda: fixed_at(S.graph(seed=103, N=150, kind="loop"), 75),
    "loop_fixed_last": lambda: fixed_at(S.graph(seed=104, N=100, kind="loop"), 99),
    "chain_split_in_four": lambda: split_chain(105, 80, (20, 40, 60)),
    # fixed -> fixed (10 -> 11 and its feature edges), fixed -> free and free -> fixed
    "covisibility_fixed_pairs": lambda: fixed_at(S.graph(seed=106, N=50, hops=(2, 3)), 10, 11, 30),
    "loop_all_fixed": lambda: fixed_at(S.graph(seed=107, N=60, kind="loop"), every=True),
    "loop_all_but_one_fixed": lambda: free_only(S.graph(seed=108, N=60, kind="loop"), 30),
    # dense envelopes
    "complete_64_free": lambda: complete(109, 65),
    "hub_300": lambda: hub(110, 300, 150),
    # the kernel's 256-thread strides: N and E around 256, and n_free * 42 = 2 562 = 10 * 256 + 2 (the gathers of the
    # diagonal blocks)
    "stride_N255_E257": lambda: trimmed(111, 255, 257),
    "stride_N256_E256": lambda: trimmed(112, 256, 256),
    "stride_N257_E255": lambda: trimmed(113, 257, 255, kind="chain"),
    "stride_nf61": lambda: S.graph(seed=114, N=62, kind="loop", hops=(2, 3, 4)),
    # what the device-entry tests compare with: the status graph without its TOO_FEW edges, and the 200-keyframe graph
    # with the oracle's feature constraints
    "status_300_skipped_removed": lambda: without(*(lambda g, st: (g, np.flatnonzero(st == 1)))(*status_graph())),
    "feature_edges_200": feat_graph_with_oracle_edges,
}

# The oracle's spread on these scenes is measured by test_oracle_spread_is_far_below_the_gpu_bounds. The scenes with no
# fixed vertex hold their x / y / yaw gauge by the plane-motion priors' 1e-4 terms alone, yet their spread is 4e-13 in the
# estimates, as small as on the anchored scenes, so they are held to the usual bars, absolute poses included. The one
# scene that needs more is a one-lap loop of 100 keyframes: there the last iterations still move the estimates by 1e-8
# when the summation or elimination order changes (the same loop with vertex 0 fixed spreads as far), while the poses
# relative to vertex 0 spread by 1e-9. Its absolute estimates are held to the measured spread times 20; the relative
# poses, on every scene, to the usual estimate bar.
EST_ATOL = {"loop_fixed_last": 2e-7}


def est_atol(name):
    return EST_ATOL.get(name, G.EST_ATOL)


def relative_poses(poses):
    """X_0^-1 X_j of every vertex j, as [N, 12] (the rotation's nine entries, then the translation), from the [N, 7]
    (qx, qy, qz, qw, tx, ty, tz) estimates."""
    R = np.array([global_ba_numpy.quat_matrix(p[:4]) for p in poses])
    t = np.asarray(poses)[:, 4:]
    R0, t0 = R[0], t[0]
    Rr = np.einsum("ji,njk->nik", R0, R)
    tr = (t - t0) @ R0
    return np.concatenate([Rr.reshape(-1, 9), tr], 1)


def spread(name, make=None):
    """The oracle's spread over one scene: the worst relative chi2 difference on the compared iterations, the worst absolute
    estimate difference and the worst relative-pose difference of the two reordered runs against the plain one."""
    s = (make or SCENES[name])()
    prm = pyglobal.params(s["Tbc"])
    base = pyglobal.run(s, prm)
    n = G.compared_iterations(base["stats"])
    chi, est, rel = 0.0, 0.0, 0.0
    for other in (pyglobal.run(s, prm, reverse=True), pyglobal.run(s, prm, reverse_order=True)):
        assert other["iterations"] >= n, name
        for f in ("trials", "accepted", "terminate"):
            assert np.array_equal(base["stats"][f][:n], other["stats"][f][:n]), (name, f)
        for f in ("chi2_before", "chi2_after"):
            a, b = base["stats"][f][:n], other["stats"][f][:n]
            chi = max(chi, float(np.max(np.abs(a - b) / np.abs(a))) if n else 0.0)
        est = max(est, float(np.abs(base["poses"] - other["poses"]).max()))
        rel = max(rel, float(np.abs(relative_poses(base["poses"]) - relative_poses(other["poses"])).max()))
    return chi, est, rel


def test_scenes_have_the_shapes_they_are_named_for():
    from scipy.sparse import coo_matrix
    from scipy.sparse.csgraph import connected_components
    for name, make in SCENES.items():
        s = make()
        N, E, nf = len(s["Tcw"]), len(s["edges"]), int((np.asarray(s["fixed"]) == 0).sum())
        if name.startswith("stride_N"):
            n, e = (int(v) for v in name[len("stride_N"):].split("_E"))
            assert (N, E) == (n, e), name
        if name == "stride_nf61":
            assert nf * 42 % 256 == 2 and nf * 42 > 256
        if "none_fixed" in name:
            assert nf == N
        if name == "loop_all_fixed":
            assert nf == 0 and E > 0
        if name == "loop_all_but_one_fixed":
            assert nf == 1
    s = SCENES["chain_split_in_four"]()
    free = np.flatnonzero(s["fixed"] == 0)
    idx = -np.ones(len(s["Tcw"]), int); idx[free] = np.arange(len(free))
    fr, to = np.array([e[0] for e in s["edges"]]), np.array([e[1] for e in s["edges"]])
    keep = (idx[fr] >= 0) & (idx[to] >= 0)
    A = coo_matrix((np.ones(keep.sum()), (idx[fr[keep]], idx[to[keep]])), shape=(len(free), len(free)))
    assert connected_components(A, directed=False)[0] == 4
    s = SCENES["covisibility_fixed_pairs"]()
    f = np.asarray(s["fixed"], bool)
    kinds = {(bool(f[i]), bool(f[j])) for i, j, _, _ in s["edges"]}
    assert kinds == {(False, False), (True, True), (True, False), (False, True)}
    # the complete graph's first pivot column (whatever the order) has 63 rows below it: past 256 / 36 and 256 / 6 rows
    s = SCENES["complete_64_free"]()
    order = pyglobal.elimination_order(65, s["fixed"], np.array([e[0] for e in s["edges"]]), np.array([e[1] for e in s["edges"]]))
    assert len(order) == 64 and len(s["edges"]) == 65 * 64 // 2
    s = SCENES["hub_300"]()
    assert sum(150 in (e[0], e[1]) for e in s["edges"]) >= 299


SMALL = {
    "loop_none_fixed_12": lambda: fixed_at(S.graph(seed=201, N=12, kind="loop", hops=(2,))),
    "chain_fixed_3_of_16": lambda: fixed_at(S.graph(seed=202, N=16, hops=(2,)), 4, 5, 11),
    "complete_12": lambda: complete(203, 12),
}


# With no fixed vertex the restatement ends 4e-6 from the oracle in the absolute estimates, though the two agree to 1e-8
# in chi2 and to 1e-7 in the poses relative to vertex 0. The restatement linearises through numeric Jacobians and scipy
# rotations, which differ from the oracle's analytic ones at the 1e-8 level; with the x / y / yaw gauge held only by the
# priors' 1e-4 terms, LM carries that difference along the gauge. The oracle against itself (the spread test below) moves
# by 4e-13 there, so this is the restatement's linearisation, not the oracle's arithmetic. Such a graph is compared in its
# relative poses at the restatement's usual bar, and in its absolute poses at 1e-5.
NUMPY_NO_FIXED_EST_ATOL = 1e-5


@pytest.mark.parametrize("name", list(SMALL))
def test_oracle_matches_numpy_restatement(name):
    """The bars of tests/test_global_ba_oracle.py::test_oracle_matches_numpy_restatement, on a graph with no fixed vertex,
    one with three (two of them adjacent) and a complete graph."""
    g = SMALL[name]()
    o = pyglobal.run(g, pyglobal.params(g["Tbc"]))
    ref = global_ba_numpy.Graph(g, g["Tbc"])
    st = ref.optimize(15)
    n = next((k for k in range(len(st)) if st[k]["chi2_before"] - st[k]["chi2_after"] < 1e-10 * st[k]["chi2_before"]), len(st))
    assert n >= 1 and o["iterations"] >= n
    for k in range(n):
        for f in ("trials", "accepted", "terminate"):
            assert o["stats"][f][k] == st[k][f], (k, f)
        for f in ("chi2_before", "chi2_after"):
            assert o["stats"][f][k] == pytest.approx(st[k][f], rel=O.NUMPY_CHI2_RTOL), (k, f)
    atol = NUMPY_NO_FIXED_EST_ATOL if not np.any(g["fixed"]) else O.NUMPY_EST_ATOL
    for v, X in enumerate(ref.X):
        q = o["poses"][v]
        np.testing.assert_allclose(global_ba_numpy.quat_matrix(q[:4]), X[:3, :3], atol=atol)
        np.testing.assert_allclose(q[4:], X[:3, 3], atol=atol)
    R = np.array([X[:3, :3] for X in ref.X])
    t = np.array([X[:3, 3] for X in ref.X])
    rel = np.concatenate([np.einsum("ji,njk->nik", R[0], R).reshape(-1, 9), (t - t[0]) @ R[0]], 1)
    np.testing.assert_allclose(relative_poses(o["poses"]), rel, atol=O.NUMPY_EST_ATOL)


@pytest.mark.parametrize("name", list(SCENES))
def test_oracle_spread_is_far_below_the_gpu_bounds(name):
    """The oracle with its edges summed in descending order and factorised in the reversed elimination order, against the
    plain run: identical trials / accepted / terminate, and every bound the GPU test holds the kernel to on this scene at
    least 10x the spread."""
    chi, est, rel = spread(name)
    assert 10 * chi <= G.CHI2_RTOL, chi
    assert 10 * rel <= G.EST_ATOL, rel
    assert 10 * est <= est_atol(name), est


def test_failed_factorisation_after_an_infinite_chi2_with_no_fixed_vertex():
    """tests/test_global_ba_oracle.py::test_failed_factorisation_after_an_infinite_chi2_keeps_the_estimate on a graph with
    no fixed vertex, where lambda_0 is taken over every vertex: the same trajectory, which the GPU test expects."""
    g = SCENES["loop_none_fixed"]()
    g["edges"] = infinite_first_info(g["edges"])
    r = pyglobal.run(g, pyglobal.params(g["Tbc"]))
    start = pyglobal.run(g, pyglobal.params(g["Tbc"], iterations=0))
    big = np.finfo(np.float64).max
    assert r["status"] == 2 and r["iterations"] == 2
    assert [(int(s["trials"]), int(s["accepted"]), int(s["terminate"])) for s in r["stats"]] == [(1, 1, 0), (1, 0, 1)]
    assert r["stats"]["chi2_before"].tolist() == [np.inf, big] and r["stats"]["chi2_after"].tolist() == [big, big]
    assert np.array_equal(r["Tcw"], start["Tcw"]) and np.array_equal(r["poses"], start["poses"])


def infinite_first_info(edges):
    """edges with info[0, 0] = inf on the first one."""
    i, j, m, info = edges[0]
    info = np.array(info, np.float32)
    info[0, 0] = np.inf
    return [(i, j, m, info)] + list(edges[1:])
