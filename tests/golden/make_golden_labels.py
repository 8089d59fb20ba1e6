#!/usr/bin/env python
"""Fixtures for the shortest-path label kernels (tests/golden/labels/*.npz), from the planning-datasets files the
reference ships (planning-datasets/data/{mpd,street}/*.npz):

  mazes032_test   the whole test split of mazes_032_moore_c8 (100 maps, 32x32)
  all064_test     the whole test split of all_064_moore_c16 (400 maps, 64x64)
  mixed064_test   the whole test split of street/mixed_064_moore_c16 (400 maps, 64x64)
  synthetic       12 maps 24x40 with walled-off regions, goals on the border / corner / inside a closed room, an
                  obstacle goal and a non-binary map; their labels are the oracle's (oracle/labels_oracle.c)

Arrays per file: shape [B,H,W] int32; obst_bits (np.packbits of each map's cells != 0, raster order); goal_idx
int32 [B]; dists int16 [B,H,W] (the shipped opt_dists); action int8 [B,H,W] (the shipped one-hot policy's action,
one member of the maximal set the reference drew at random); maps float32 [B,H,W] only where a map is not binary.

    python tests/golden/make_golden_labels.py      # needs a checkout of the reference
"""
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
DATA = "/root/reference/planning-datasets/data"
OUT = os.path.join(HERE, "labels")


def save(name, desc, maps, goal_idx, dists, action):
    B, H, W = maps.shape
    arrays = dict(meta=np.array(json.dumps({"desc": desc})), shape=np.array([B, H, W], np.int32),
                  obst_bits=np.packbits((maps != 0).reshape(B, -1), axis=1), goal_idx=goal_idx.astype(np.int32),
                  dists=dists.reshape(B, H, W).astype(np.int16), action=action.reshape(B, H, W).astype(np.int8))
    if not np.isin(maps, (0.0, 1.0)).all():
        arrays["maps"] = maps.astype(np.float32)
    os.makedirs(OUT, exist_ok=True)
    np.savez_compressed(os.path.join(OUT, name + ".npz"), **arrays)


def shipped(rel, name):
    z = np.load(os.path.join(DATA, rel))
    maps, goals, pol, dists = (z[f"arr_{8 + j}"] for j in range(4))
    B = maps.shape[0]
    goal_idx = goals.reshape(B, -1).argmax(1)
    save(name, f"{rel} test split ({B} maps): shipped goals, opt_dists and policy actions", maps,
         goal_idx, dists[:, 0], pol[:, :, 0].argmax(1))


def synthetic():
    sys.path.insert(0, ROOT)
    from oracle import labels as label_oracle

    rng = np.random.RandomState(7)
    B, H, W = 12, 24, 40
    maps = (rng.rand(B, H, W) > 0.3).astype(np.float32)
    maps[:, :, 19] = 0.0                       # a wall: the right half is unreachable unless a gap is opened
    maps[0::2, 5, 19] = 1.0
    goal_idx = np.zeros(B, np.int64)
    corners = [0, W - 1, (H - 1) * W, H * W - 1]
    for b in range(B):
        goal_idx[b] = corners[b % 4] if b < 4 else rng.randint(0, W) if b < 8 else (H - 1) * W + rng.randint(0, W)
    maps[np.arange(B), goal_idx // W, goal_idx % W] = 1.0
    g = 9 * W + 9                              # map 8: a goal inside a closed 3x3 ring
    maps[8, 8:11, 8:11] = 0.0
    maps[8, 9, 9] = 1.0
    goal_idx[8] = g
    goal_idx[9] = 3 * W + 3                    # map 9: the goal is an obstacle (still the source of the search)
    maps[9, 3, 3] = 0.0
    maps[10] *= np.where(rng.rand(H, W) > 0.5, 0.5, 1.0).astype(np.float32)   # map 10: non-binary values
    d, _, act = label_oracle.opt_labels(maps, goal_idx.astype(np.int32))
    save("synthetic", "24x40 maps with a dividing wall, corner / border / walled-in / obstacle goals and one non-binary "
                      "map; labels from the CPU oracle", maps, goal_idx, d[:, 0], act[:, 0])


def main():
    shipped("mpd/mazes_032_moore_c8.npz", "mazes032_test")
    shipped("mpd/all_064_moore_c16.npz", "all064_test")
    shipped("street/mixed_064_moore_c16.npz", "mixed064_test")
    synthetic()
    for f in sorted(os.listdir(OUT)):
        print(f, os.path.getsize(os.path.join(OUT, f)))


if __name__ == "__main__":
    main()
