"""Scenes for the map-point update tests (tests/test_mappoint_oracle.py, tests/test_mappoint_gpu.py): seeded scenes whose
mix reaches every branch of addObservation / eraseObservation, and the single-point cases built for one branch each."""
import numpy as np

from tools import mappoint_scenes as ms

# branch events of oracle/mappoint_numpy.py each scene family must reach
ADD_EVENTS = {"short_list", "already_good", "pkf0_older", "pkf0_self", "observer_beyond_6", "depth_below", "depth_above",
              "parallax_rejected", "triangulated", "abandoned", "null_reset", "main_unchanged", "main_changed",
              "null_kf_skipped", "median_tie", "two_adds"}
ERASE_EVENTS = {"erased_to_empty", "erase_main_changed", "main_unchanged", "null_kf_skipped"}


def add_scenes():
    """(name, scene) pairs of the add family: plain, no good parallax, many null keyframes and points, short lists"""
    return [("mixed", ms.scene(300, seed=101)),
            ("no_good_prl", ms.scene(300, seed=102, good_frac=0.0)),
            ("null_heavy", ms.scene(200, seed=103, null_frac=0.3)),
            ("short", ms.scene(200, seed=104, lengths=np.arange(200) % 3 + 1))]


def erase_scenes():
    return [("mixed", ms.scene(300, seed=201, mode="erase")),
            ("short", ms.scene(200, seed=202, mode="erase", lengths=np.arange(200) % 3 + 1, n_upd=(0.2, 0.4, 0.4)))]


def long_scene(mode="add"):
    """every list at or past the 32-entry shared-memory list: 32, 33 and the long lengths"""
    lengths = np.array([32, 33, 40, 47, 64, 97] * 6)
    return ms.scene(len(lengths), seed=301 if mode == "add" else 302, lengths=lengths, mode=mode, good_frac=0.0)


def split_updates(sc):
    """the scene's two-update points as two calls: the first with the list before the second insertion and only the first
    update, the second with the full list and only the second update. Returns (first, second) update sets and the lists
    of the first call: (obs_ptr, obs_kf, obs_idx, upd_ptr, upd_pos) twice."""
    mp, up, pos = sc["mp"], sc["upd_ptr"], sc["upd_pos"]
    M = len(mp["obs_ptr"]) - 1
    ptr1, kf1, idx1, u1p, u1 = [0], [], [], [0], []
    u2p, u2 = [0], []
    for m in range(M):
        a, b = mp["obs_ptr"][m], mp["obs_ptr"][m + 1]
        ups = list(pos[up[m]:up[m + 1]])
        last = ups[-1] if len(ups) == 2 else None
        keep = [j for j in range(b - a) if j != last]
        kf1 += list(mp["obs_kf"][a:b][keep]); idx1 += list(mp["obs_idx"][a:b][keep]); ptr1.append(len(kf1))
        first = [keep.index(q) for q in ups[:1 if last is not None else len(ups)]]
        u1 += first; u1p.append(len(u1))
        u2 += [last] if last is not None else []; u2p.append(len(u2))
    i4 = lambda x: np.asarray(x, np.int32)
    return (i4(ptr1), i4(kf1), i4(idx1), i4(u1p), i4(u1)), (i4(u2p), i4(u2))


# scenes of update sequences and list shapes the families above do not build, and the events they must reach
def many_updates_scene():
    """3 to 8 adds per point without good parallax: abandonments followed by enough re-adds for updateParallax to run
    on the rebuilt list"""
    return ms.scene(400, seed=111, updates=(3, 8), good_frac=0.0, lengths=np.arange(400) % 30 + 8)


def erase_main_scene():
    """every point erases its whole list, each time the entry of its current main keyframe"""
    return ms.scene(150, seed=211, mode="erase", erase_main=True, lengths=np.arange(150) % 40 + 1, kf_null_frac=0.1)


LIST_LENGTHS = (31, 32, 33, 255, 256, 257, 1000, 4000)


def list_length_scene(mode="add", lengths=LIST_LENGTHS):
    """lists on both sides of the 32-entry shared-memory list and long ones, with null keyframes and 3 to 8 updates (absent
    positions while an add runs, erased ones while an erase runs); every update of a list of N recomputes an N x N median"""
    lengths = np.repeat(lengths, [2 if L <= 257 else 1 for L in lengths])          # one each of the longest
    return ms.scene(len(lengths), seed=311 if mode == "add" else 312, lengths=lengths, mode=mode, good_frac=0.0,
                    updates=(3, 8), kf_null_frac=0.15)


NLEVELS = (1, 5, 12, 32)


def nlevels_scene(nlevels, mode="add"):
    return ms.scene(300, seed=500 + nlevels, mode=mode, nlevels=nlevels, updates=(1, 4), good_frac=0.2)
