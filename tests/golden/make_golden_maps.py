#!/usr/bin/env python
"""Fixture for the map kernel (tests/golden/maps/sources.npz): decoded map images of the planning-datasets generator
and the maps it shipped for them.

  mp_*      the 100 `mazes` test images and the first 3 test images of each other family, 201x201 uint8 (PNG decoded
            and converted to L), with the shipped 32x32 map of each (mpd/<family>_032_moore_c8.npz arr_8)
  tiled_*   the sources of the first 24 Tiled MP train maps (mpd/all_064_moore_c16.npz arr_0): tiled_pos are their
            places in the natural-sort list of the 6 400 original/*/train/*.png images, which
            np.random.RandomState(1372).choice(6400, 4) per tile draws; tiled_maps are the shipped 64x64 maps

Maps are stored as np.packbits of their cells (1.0 -> 1) in raster order.

    python tests/golden/make_golden_maps.py [--data DIR]      # needs a checkout of the reference
"""
import argparse
import glob
import os
import sys

import numpy as np
from PIL import Image

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
import maps_oracle as mo  # noqa: E402

FAMILIES = ("alternating_gaps", "bugtrap_forest", "forest", "gaps_and_forest", "mazes", "multiple_bugtraps",
            "shifting_gaps", "single_bugtrap")
N_TILES = 24


def decode(path):
    return np.asarray(Image.open(path).convert("L"), dtype=np.uint8)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--data", default="/root/reference/planning-datasets/data")
    mpd = os.path.join(ap.parse_args().data, "mpd")
    names, images, maps = [], [], []
    for fam in FAMILIES:
        paths = sorted(glob.glob(os.path.join(mpd, "original", fam, "test", "*.png")), key=mo.natural_key)
        shipped = np.load(os.path.join(mpd, f"{fam}_032_moore_c8.npz"))["arr_8"]
        n = len(paths) if fam == "mazes" else 3
        for i in range(n):
            names.append(f"{fam}/test/{os.path.basename(paths[i])}")
            images.append(decode(paths[i]))
            maps.append(shipped[i])
    train = sorted(glob.glob(os.path.join(mpd, "original", "*", "train", "*.png")), key=mo.natural_key)
    rng = np.random.RandomState(1372)
    draws = np.stack([rng.choice(len(train), 4) for _ in range(N_TILES)])
    pos = np.unique(draws)
    tiled = np.load(os.path.join(mpd, "all_064_moore_c16.npz"))["arr_0"][:N_TILES]
    np.savez_compressed(
        os.path.join(HERE, "maps", "sources.npz"),
        mp_names=np.array(names), mp_images=np.stack(images),
        mp_maps=np.packbits(np.stack(maps).reshape(len(maps), -1) != 0, axis=1),
        tiled_count=np.int64(len(train)), tiled_pos=pos.astype(np.int64),
        tiled_images=np.stack([decode(train[p]) for p in pos]),
        tiled_maps=np.packbits(tiled.reshape(N_TILES, -1) != 0, axis=1))


if __name__ == "__main__":
    main()
