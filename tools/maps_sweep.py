#!/usr/bin/env python
"""Pin the map oracle (tests/maps_oracle.py: Pillow's bicubic resize + Otsu + threshold) to every map the
planning-datasets generator made from images:

  MP        all splits of the 8 mpd/*_032_moore_c8.npz files (8 000 maps) from original/<family>/<split>/*.png
  Tiled MP  the 3 200 train maps of mpd/all_064_moore_c16.npz: the 6 400 original/*/train/*.png maps in natural-sort
            order, tiled 2x2 with np.random.seed(1372) + np.random.choice(6400, 4) per tile (the generator's draws;
            its validation and test tiles follow label draws and are not replayed)

For each: the number of maps that differ from the shipped map (expected 0).  Needs a checkout of the reference (the
datasets are not part of this repository):

    python tools/maps_sweep.py [--data DIR] [--out profiles/maps_sweep.json]
"""
import argparse
import glob
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DEFAULT_DATA = "/root/reference/planning-datasets/data"
FAMILIES = ("alternating_gaps", "bugtrap_forest", "forest", "gaps_and_forest", "mazes", "multiple_bugtraps",
            "shifting_gaps", "single_bugtrap")
SPLITS = (("train", 0), ("validation", 4), ("test", 8))


def oracle_maps(pattern: str, size: int) -> np.ndarray:
    from PIL import Image

    import maps_oracle as mo

    paths = sorted(glob.glob(pattern), key=mo.natural_key)
    return np.stack([mo.make_map(np.asarray(Image.open(p).convert("L")), size, size)[0] for p in paths])


def sweep(data_dir: str = DEFAULT_DATA) -> dict:
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import maps_oracle as mo

    mpd = os.path.join(data_dir, "mpd")
    out, t0 = {"mp": {}, "tiled_mp_train": {}}, time.time()
    tot_maps = tot_diff = 0
    for fam in FAMILIES:
        z = np.load(os.path.join(mpd, f"{fam}_032_moore_c8.npz"))
        for split, k in SPLITS:
            got = oracle_maps(os.path.join(mpd, "original", fam, split, "*.png"), 32)
            ship = z[f"arr_{k}"]
            diff = int((got != ship).reshape(len(ship), -1).any(1).sum()) if got.shape == ship.shape else len(ship)
            out["mp"][f"{fam}/{split}"] = {"maps": len(ship), "differ": diff}
            tot_maps += len(ship)
            tot_diff += diff
    srcs = oracle_maps(os.path.join(mpd, "original", "*", "train", "*.png"), 32)
    ship = np.load(os.path.join(mpd, "all_064_moore_c16.npz"))["arr_0"]
    rng = np.random.RandomState(1372)
    tiles = np.stack([mo.montage(srcs[rng.choice(len(srcs), 4)], 2) for _ in range(len(ship))])
    out["tiled_mp_train"] = {"sources": len(srcs), "maps": len(ship),
                             "differ": int((tiles != ship).reshape(len(ship), -1).any(1).sum())}
    out["total"] = {"mp_maps": tot_maps, "mp_differ": tot_diff, "tiled_maps": len(ship),
                    "tiled_differ": out["tiled_mp_train"]["differ"], "seconds": round(time.time() - t0, 1)}
    return out


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--data", default=DEFAULT_DATA, help="planning-datasets/data of a reference checkout")
    ap.add_argument("--out", default=None, help="write the JSON record here")
    args = ap.parse_args()
    res = sweep(args.data)
    text = json.dumps(res, indent=1)
    print(json.dumps(res["total"]))
    if args.out:
        with open(args.out, "w") as f:
            f.write(text + "\n")


if __name__ == "__main__":
    main()
