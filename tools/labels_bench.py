#!/usr/bin/env python
"""Throughput of the shortest-path label kernel (nastar_labels.cuh, neural_astar.utils.data.compute_opt_labels) on an
H100, with the card's name and power limit read in the same run, next to the planning-datasets generator's own
dijkstra_dist on the same machine's host cores (staged into oracle/_ref by build(); "not available" otherwise).

Workloads: the 1000 mazes_032 maps with their shipped goals (tests/golden/inputs_mazes032_all1000.npz) and 1024
Config-5-style 256x256 maps (tools/c5_data.py, seed 1234).  Timing: CUDA events around 10 back-to-back calls, median
of 3 trials, inputs device-resident.  Each workload is timed with the Moore labels and, in the same run, with the NEWS
labels (mechanism="news": 4-connected wavefronts, 4 policy targets; the "news" row).  Prints one JSON object; --out
also writes it to a file.

    python tools/labels_bench.py [--out profiles/h100_labels_bench.json]
"""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for _p in (ROOT, os.path.join(ROOT, "neural-astar_b200"), os.path.join(ROOT, "tests"), os.path.join(ROOT, "tools")):
    if _p not in sys.path:
        sys.path.insert(0, _p)

import numpy as np  # noqa: E402
import torch  # noqa: E402


def timed(fn, reps=10):
    for _ in range(3):
        fn()
    trials = []
    for _ in range(3):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(reps):
            fn()
        b.record()
        torch.cuda.synchronize()
        trials.append(a.elapsed_time(b) / reps)
    return sorted(trials)[1], trials


def power_limit_w(index):
    try:
        import pynvml as nv

        nv.nvmlInit()
        return nv.nvmlDeviceGetEnforcedPowerLimit(nv.nvmlDeviceGetHandleByIndex(index)) / 1e3
    except Exception:
        return None


def cpu_reference(maps, goal_idx, n=4):
    from oracle import labels as label_oracle

    if not label_oracle.stage_reference():
        return "not available (the generator's dijkstra.py / mechanism.py were not staged)"
    sys.path.insert(0, label_oracle.REF_STAGE)
    from dijkstra import dijkstra_dist
    from mechanism import Moore

    mech = Moore()
    W = maps.shape[-1]
    t0 = time.perf_counter()
    for i in range(n):
        g = int(goal_idx[i])
        dijkstra_dist(maps[i, 0].astype(np.float64), mech, (0, g // W, g % W))
    ms = (time.perf_counter() - t0) * 1e3 / n
    return {"what": f"planning_datasets_utils.dijkstra.dijkstra_dist (the generator's own), {n} mazes_032 maps, one "
                    "host core", "ms_per_map": ms, "maps_per_s": 1e3 / ms,
            "extract_policy": "not measured: it lives in planning_datasets_utils/data.py, whose imports (natsort, "
                              "skimage, PIL, tqdm) are not installed"}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    from c5_data import c5_maps
    from golden_util import Golden
    from neural_astar import _native
    from neural_astar.utils.data import compute_opt_labels

    assert torch.cuda.is_available(), "labels_bench measures the GPU kernel: no GPU found"
    dev = torch.device("cuda:0")
    out = {"kernel": "nastar::opt_labels_kernel (BFS wavefronts on u32 row words + policy, one CTA per map)",
           "timing": "CUDA events around 10 back-to-back calls, median of 3 trials; inputs device-resident",
           "device": torch.cuda.get_device_name(dev), "power_limit_w": power_limit_w(0)}
    g = Golden("inputs_mazes032_all1000")
    o1k = g.obst.astype(np.float32)
    c5o, _, c5g = c5_maps(1024, 256, 256, 1234)
    for name, maps_np, goal_idx in (("mazes_032_all1000", o1k, g.z["goal_idx"]),
                                    ("c5_256x256_b1024", c5o, c5g.reshape(len(c5g), -1).argmax(1))):
        maps = torch.from_numpy(maps_np).to(dev)
        gi = torch.from_numpy(np.asarray(goal_idx, np.int32)).to(dev)
        goals = torch.zeros_like(maps).view(len(maps), -1).scatter_(1, gi.long()[:, None], 1.0).view_as(maps)
        B = maps.shape[0]
        rows = {}
        for mech in ("moore", "news"):
            k_ms, k_trials = timed(lambda: _native.opt_labels(maps, gi, mech))
            a_ms, _ = timed(lambda: compute_opt_labels(maps, goals, mech))
            d = _native.opt_labels(maps, gi, mech)[0].view(B, -1)
            reached = d.masked_fill(d <= -d.shape[1], 0)
            rows[mech] = {"kernel_ms": k_ms, "kernel_ms_trials": k_trials, "maps_per_s": B / (k_ms * 1e-3),
                          "compute_opt_labels_ms": a_ms, "compute_opt_labels_maps_per_s": B / (a_ms * 1e-3),
                          "max_bfs_depth": int(-reached.min())}
        out[name] = {"maps": B, "grid": f"{maps.shape[-2]}x{maps.shape[-1]}", **rows["moore"], "news": rows["news"]}
    out["cpu_reference"] = cpu_reference(o1k, g.z["goal_idx"])
    line = json.dumps(out)
    print(line)
    if args.out:
        with open(args.out, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
