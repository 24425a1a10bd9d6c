"""--dump-outputs for the solver bench tools: every output of a tool's last run as DIR/<tag>_<name>.npy, so two builds can
be compared byte for byte with cmp."""
from __future__ import annotations

import os

import numpy as np


def _bytes(v):
    return np.ascontiguousarray(np.asarray(v)).reshape(-1).view(np.uint8)


def save(out_dir, tag, outputs):
    """outputs: name -> array or scalar, or a list of such dicts (one per problem of a batch), whose entries are written
    concatenated as raw bytes; None entries (outputs a problem did not produce) are skipped."""
    os.makedirs(out_dir, exist_ok=True)
    if isinstance(outputs, list):
        names = sorted({k for r in outputs for k in r})
        outputs = {k: np.concatenate([_bytes(r[k]) for r in outputs if r.get(k) is not None] or [np.zeros(0, np.uint8)])
                   for k in names}
    for name, v in outputs.items():
        np.save(os.path.join(out_dir, f"{tag}_{name}.npy"), np.asarray(v))
