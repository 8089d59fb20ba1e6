#!/usr/bin/env python
"""Pin the label oracle (oracle/labels_oracle.c) to every map the planning-datasets generator shipped: all splits of
the 10 .npz files under planning-datasets/data/{mpd,street} (16 000 maps).  For every map, with the shipped goal:

  dist mismatches    cells whose oracle distance differs from the shipped opt_dists
  policy mismatches  cells whose shipped one-hot action is NOT in the oracle's maximal-action set

Both must be 0.  Needs a checkout of the reference (the datasets are not part of this repository):

    python tools/labels_sweep.py [--data DIR] [--out profiles/labels_sweep.json]
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--data", default=DEFAULT_DATA)
    ap.add_argument("--out", default=None, help="write the result as JSON here")
    args = ap.parse_args()
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
