"""Loader for the shortest-path label fixtures written by tests/golden/make_golden_labels.py."""
from __future__ import annotations

import os

import numpy as np

LABELS_DIR = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "labels")
NAMES = ("mazes032_test", "all064_test", "mixed064_test", "synthetic")


def load(name: str):
    """(maps float32 [B,H,W], goal_idx int32 [B], dists float32 [B,H,W], action int8 [B,H,W])"""
    z = np.load(os.path.join(LABELS_DIR, name + ".npz"))
    B, H, W = (int(v) for v in z["shape"])
    if "maps" in z.files:
        maps = z["maps"]
    else:
        maps = np.unpackbits(z["obst_bits"], axis=1)[:, :H * W].reshape(B, H, W).astype(np.float32)
    return maps, z["goal_idx"], z["dists"].astype(np.float32), z["action"]
