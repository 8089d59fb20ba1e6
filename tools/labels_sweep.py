#!/usr/bin/env python
"""Pin the label oracle (oracle/labels_oracle.c) to every map the planning-datasets generator shipped: all splits of
the 10 .npz files under planning-datasets/data/{mpd,street} (16 000 maps).  For every map, with the shipped goal:

  dist mismatches    cells whose oracle distance differs from the shipped opt_dists
  policy mismatches  cells whose shipped one-hot action is NOT in the oracle's maximal-action set

Both must be 0.  The shipped files are all Moore datasets.  With --mechanism news the same maps and goals pin the
oracle's NEWS mode to the generator's own code instead of to shipped arrays:

  dist mismatches     cells whose oracle NEWS distance differs from dijkstra_dist(maze, NorthEastWestSouth(), goal)
                      (the generator's dijkstra.py / mechanism.py, staged into oracle/_ref by build())
  max-set mismatches  cells whose oracle NEWS mask differs from the maximal-action set of extract_policy
                      (data.py:40-58, restated by extract_policy_max_sets) over those distances

Both must be 0.  Needs a checkout of the reference (the datasets are not part of this repository):

    python tools/labels_sweep.py [--data DIR] [--out profiles/labels_sweep.json]
    python tools/labels_sweep.py --mechanism news [--out profiles/labels_sweep_news.json]
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
# actions of the generator's mechanisms in order (mechanism.py:58, :140-149): N, E, W, S, NE, NW, SE, SW as (dy, dx)
MOVES = ((-1, 0), (0, 1), (0, -1), (1, 0), (-1, 1), (-1, -1), (1, 1), (1, -1))


def extract_policy_max_sets(maze, value, num_actions: int):
    """extract_policy (data.py:40-58) without its random draw: for every cell of maze [H,W] the bit mask of the actions
    whose neighbors_func target (a move off the grid or onto a cell whose value is 0.0 stays put) has the maximal
    value [H,W], as uint8.  Its loop starts from max_val = -sys.maxsize, below every value, so the first action always
    enters the set, later ones replace it when greater and join it when equal: the set of maximal actions."""
    H, W = maze.shape
    y, x = np.mgrid[0:H, 0:W]
    vals = []
    for dy, dx in MOVES[:num_actions]:
        ty, tx = y + dy, x + dx
        ok = (ty >= 0) & (ty < H) & (tx >= 0) & (tx < W)
        ok[ok] = maze[ty[ok], tx[ok]] != 0.0
        vals.append(np.where(ok, value[np.where(ok, ty, y), np.where(ok, tx, x)], value))
    vals = np.stack(vals)
    best = vals.max(0)
    return sum((vals[a] == best).astype(np.uint8) << a for a in range(num_actions)).astype(np.uint8)


def generator_news_dists(job):
    """dijkstra_dist(maze, NorthEastWestSouth(), (0, gy, gx))[0] of the generator's staged dijkstra.py / mechanism.py
    for maps [b,H,W] and flat goals [b], as float32 [b,H,W] (one worker of sweep_news)."""
    maps, goal_idx, stage = job
    if stage not in sys.path:
        sys.path.insert(0, stage)
    from dijkstra import dijkstra_dist
    from mechanism import NorthEastWestSouth

    mech, W = NorthEastWestSouth(), maps.shape[-1]
    return np.stack([dijkstra_dist(m.astype(np.float64), mech, (0, int(g) // W, int(g) % W))[0]
                     for m, g in zip(maps, goal_idx)]).astype(np.float32)


def sweep(data_dir: str = DEFAULT_DATA, chunk: int = 400) -> dict:
    if ROOT not in sys.path:
        sys.path.insert(0, ROOT)
    from oracle import labels as label_oracle

    files = sorted(glob.glob(os.path.join(data_dir, "*", "*.npz")))
    per_file, tot = {}, {"maps": 0, "cells": 0, "dist_mismatch_cells": 0, "dist_mismatch_maps": 0,
                         "policy_not_in_max_set_cells": 0}
    t0 = time.time()
    for f in files:
        name = os.path.relpath(f, data_dir)
        z = np.load(f)
        row = {"maps": 0, "dist_mismatch_cells": 0, "dist_mismatch_maps": 0, "policy_not_in_max_set_cells": 0}
        for k in (0, 4, 8):
            maps, goals = z[f"arr_{k}"], z[f"arr_{k + 1}"]
            pol, dists = z[f"arr_{k + 2}"], z[f"arr_{k + 3}"]
            B, H, W = maps.shape
            for i in range(0, B, chunk):
                m = maps[i:i + chunk]
                g = goals[i:i + chunk].reshape(len(m), -1).argmax(1).astype(np.int32)
                d, mask, _ = label_oracle.opt_labels(m, g)
                bad = d[:, 0] != dists[i:i + chunk, 0]
                row["dist_mismatch_cells"] += int(bad.sum())
                row["dist_mismatch_maps"] += int(bad.reshape(len(m), -1).any(1).sum())
                shipped = pol[i:i + chunk, :, 0].argmax(1)                      # [b,H,W] the action drawn by the reference
                inset = (mask[:, 0] >> shipped.astype(np.uint8)) & 1
                row["policy_not_in_max_set_cells"] += int((inset == 0).sum())
            row["maps"] += B
            tot["cells"] += B * H * W
        per_file[name] = row
        for key in ("maps", "dist_mismatch_cells", "dist_mismatch_maps", "policy_not_in_max_set_cells"):
            tot[key] += row[key]
    return {"files": per_file, "total": tot, "seconds": time.time() - t0}


def sweep_news(data_dir: str = DEFAULT_DATA, chunk: int = 50, workers: int = 0) -> dict:
    """The NEWS oracle's labels against the generator's NEWS code on every shipped map with its shipped goal."""
    import multiprocessing

    if ROOT not in sys.path:
        sys.path.insert(0, ROOT)
    from oracle import labels as label_oracle

    if not label_oracle.stage_reference():
        raise SystemExit("the generator's dijkstra.py / mechanism.py are not staged (needs a reference checkout)")
    files = sorted(glob.glob(os.path.join(data_dir, "*", "*.npz")))
    keys = ("maps", "dist_mismatch_cells", "dist_mismatch_maps", "max_set_mismatch_cells", "unreached_cells")
    per_file, tot = {}, dict.fromkeys(keys + ("cells",), 0)
    t0 = time.time()
    with multiprocessing.Pool(workers or os.cpu_count()) as pool:
        for f in files:
            name = os.path.relpath(f, data_dir)
            z = np.load(f)
            row = dict.fromkeys(keys, 0)
            for k in (0, 4, 8):
                maps = z[f"arr_{k}"].astype(np.float32)
                goal_idx = z[f"arr_{k + 1}"].reshape(len(maps), -1).argmax(1).astype(np.int32)
                B, H, W = maps.shape
                jobs = [(maps[i:i + chunk], goal_idx[i:i + chunk], label_oracle.REF_STAGE)
                        for i in range(0, B, chunk)]
                ref = np.concatenate(pool.map(generator_news_dists, jobs))
                d, mask, _ = label_oracle.opt_labels(maps, goal_idx, mechanism="news")
                bad = d[:, 0] != ref
                row["dist_mismatch_cells"] += int(bad.sum())
                row["dist_mismatch_maps"] += int(bad.reshape(B, -1).any(1).sum())
                row["unreached_cells"] += int((ref == -H * W).sum())
                for i in range(B):
                    want = extract_policy_max_sets(maps[i], ref[i], 4)
                    row["max_set_mismatch_cells"] += int((mask[i, 0] != want).sum())
                row["maps"] += B
                tot["cells"] += B * H * W
            per_file[name] = row
            for key in keys:
                tot[key] += row[key]
            print(f"{name:40s} maps {row['maps']:5d}  dist mismatches {row['dist_mismatch_cells']}  "
                  f"max-set mismatches {row['max_set_mismatch_cells']}", flush=True)
    return {"mechanism": "news", "reference": "planning_datasets_utils dijkstra_dist(maze, NorthEastWestSouth(), goal) "
            "and the max set of extract_policy", "files": per_file, "total": tot, "seconds": time.time() - t0}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--data", default=DEFAULT_DATA)
    ap.add_argument("--out", default=None, help="write the result as JSON here")
    ap.add_argument("--mechanism", default="moore", choices=("moore", "news"))
    args = ap.parse_args()
    if args.mechanism == "news":
        r = sweep_news(args.data)
        t = r["total"]
        print(f"TOTAL maps {t['maps']} cells {t['cells']}: dist mismatches {t['dist_mismatch_cells']}, "
              f"max-set mismatches {t['max_set_mismatch_cells']} ({r['seconds']:.1f} s)")
        if args.out:
            with open(args.out, "w") as fh:
                json.dump(r, fh, indent=1)
        return 0 if t["dist_mismatch_cells"] == 0 and t["max_set_mismatch_cells"] == 0 else 1
    r = sweep(args.data)
    for name, row in r["files"].items():
        print(f"{name:40s} maps {row['maps']:5d}  dist mismatches {row['dist_mismatch_cells']}  "
              f"policy actions outside the max set {row['policy_not_in_max_set_cells']}")
    t = r["total"]
    print(f"TOTAL maps {t['maps']} cells {t['cells']}: dist mismatches {t['dist_mismatch_cells']}, "
          f"policy actions outside the max set {t['policy_not_in_max_set_cells']} ({r['seconds']:.1f} s)")
    if args.out:
        with open(args.out, "w") as fh:
            json.dump(r, fh, indent=1)
    return 0 if t["dist_mismatch_cells"] == 0 and t["policy_not_in_max_set_cells"] == 0 else 1


if __name__ == "__main__":
    sys.exit(main())
