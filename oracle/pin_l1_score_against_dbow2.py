"""Writes tests/golden/l1_score_golden.npz: seeded BowVector pairs and DBoW2's own L1Scoring::score of each, from
oracle/_ref/libdbow2_l1.so (oracle/dbow2_ref.mk, compiled from the reference's Thirdparty/DBoW2 sources).

    python oracle/pin_l1_score_against_dbow2.py

Cases: identical vectors, disjoint vectors (-0.0), either side empty, one common word, random overlaps of ORBvoc-like
sizes, and vectors whose ascending sum differs from a pairwise (tree) sum of the same terms. The file stores the pairs
flattened (words, values and the offsets of each vector) and the score bytes.
"""
from __future__ import annotations

import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tests.loop_cases import golden_pairs  # noqa: E402
from oracle import pyloop  # noqa: E402


def main():
    if pyloop.make_ref() is None:
        raise SystemExit("oracle/_ref/libdbow2_l1.so is missing: build it with oracle/dbow2_ref.mk from the reference tree")
    pairs = golden_pairs()
    words, values, off = [], [], [0]
    for (w1, v1), (w2, v2) in pairs:
        for w, v in ((w1, v1), (w2, v2)):
            words.append(w); values.append(v); off.append(off[-1] + len(w))
    scores = np.array([pyloop.dbow2_score(w1, v1, w2, v2) for (w1, v1), (w2, v2) in pairs])
    out = os.path.join(ROOT, "tests", "golden", "l1_score_golden.npz")
    np.savez_compressed(out, words=np.concatenate(words).astype(np.int32), values=np.concatenate(values).astype(np.float64),
                        offsets=np.asarray(off, np.int64), scores=scores)
    print(f"{len(pairs)} pairs -> {out}")


if __name__ == "__main__":
    main()
