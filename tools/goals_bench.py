#!/usr/bin/env python
"""Throughput of the goal kernel (nastar_goals.cuh; neural_astar.utils.data.sample_device_goal_maps) on an H100, with
the card's name and power limit read in the same run, next to the host sample_goal_maps on one host core.

Workloads (maps device-resident, edge_size = H/4 as the planning-datasets generator uses for its mazes):
  mazes_032_all1000   the 1000 mazes_032 maps (tests/golden/inputs_mazes032_all1000.npz);
  all_064_test400     the 400 all_064 test maps (tests/golden/inputs_all064_test400.npz);
  c5_256x256_b1024    1024 Config-5 256x256 maps (tools/c5_data.py, seed 1234);
  random_512x512_b256 256 Bernoulli(0.2) 512x512 maps, seed 512.
Per workload: the kernel alone (_native.sample_goals, fixed draws), sample_device_goal_maps (torch.randint draws, the
kernel and the status read-back), compute_opt_labels alone, and goals + compute_opt_labels back to back; CUDA events
around 10 back-to-back calls, median of 3 trials.  The host arm times sample_goal_maps per map over a subset, host clock.
Prints one JSON object; --out also writes it to a file.

    python tools/goals_bench.py [--out profiles/h100_goals_bench.json]
"""
import argparse
import json
import os
import random
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for _p in (ROOT, os.path.join(ROOT, "neural-astar_b200"), os.path.join(ROOT, "tests"), os.path.join(ROOT, "tools")):
    if _p not in sys.path:
        sys.path.insert(0, _p)

import numpy as np  # noqa: E402
import torch  # noqa: E402

from labels_bench import timed  # noqa: E402
from wlabels_bench import power_limit_w  # noqa: E402


def workloads():
    from c5_data import c5_maps
    from golden_util import Golden

    yield "mazes_032_all1000", Golden("inputs_mazes032_all1000").obst, 100
    yield "all_064_test400", Golden("inputs_all064_test400").obst, 100
    yield "c5_256x256_b1024", c5_maps(1024, 256, 256, 1234)[0], 20
    yield "random_512x512_b256", (np.random.RandomState(512).rand(256, 1, 512, 512) >= 0.2).astype(np.float32), 8


def host_ms_per_map(maps, edge, n):
    from neural_astar.utils.data import sample_goal_maps

    sub = maps[:n]
    sample_goal_maps(sub[:1], edge_size=edge, rng=random.Random(0))
    t0 = time.perf_counter()
    sample_goal_maps(sub, edge_size=edge, rng=random.Random(0))
    return (time.perf_counter() - t0) * 1e3 / len(sub)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    from neural_astar import _native
    from neural_astar.utils.data import compute_opt_labels, sample_device_goal_maps

    assert torch.cuda.is_available(), "goals_bench measures the GPU kernel: no GPU found"
    torch.set_num_threads(1)
    dev = torch.device("cuda:0")
    out = {"kernel": "nastar::sample_goals_kernel (union-find over the map's cells, one CTA per map)",
           "timing": "CUDA events around 10 back-to-back calls, median of 3 trials; maps device-resident",
           "device": torch.cuda.get_device_name(dev), "power_limit_w": power_limit_w(0),
           "host_arm": "utils.data.sample_goal_maps (scipy.ndimage.label + random.choice per map), one host core, "
                       "host clock over the first maps of the workload"}
    for name, maps_np, n_host in workloads():
        B, _, H, W = maps_np.shape
        edge = H // 4
        md = torch.from_numpy(maps_np).to(dev)
        g = torch.Generator(device=dev)
        g.manual_seed(0)
        draws = torch.randint(-2 ** 31, 2 ** 31, (B,), dtype=torch.int32, device=dev, generator=g)
        k_ms, k_trials = timed(lambda: _native.sample_goals(md, draws, edge))
        s_ms, _ = timed(lambda: sample_device_goal_maps(md, edge, generator=g))
        goals = sample_device_goal_maps(md, edge, generator=g)
        l_ms, _ = timed(lambda: compute_opt_labels(md, goals))
        gl_ms, _ = timed(lambda: compute_opt_labels(md, sample_device_goal_maps(md, edge, generator=g)))
        host = host_ms_per_map(maps_np, edge, n_host)
        in_smem = H * W * 4 + (H * W + 31) // 32 * 8 <= 225 * 1024
        out[name] = {"maps": B, "grid": f"{H}x{W}", "edge_size": edge,
                     "union_find_plane": "shared memory" if in_smem else "the goal plane in HBM",
                     "kernel_ms": k_ms, "kernel_ms_trials": k_trials, "kernel_us_per_map": k_ms * 1e3 / B,
                     "kernel_maps_per_s": B / (k_ms * 1e-3), "sample_device_goal_maps_ms": s_ms,
                     "compute_opt_labels_ms": l_ms, "goals_plus_compute_opt_labels_ms": gl_ms,
                     "goals_plus_labels_maps_per_s": B / (gl_ms * 1e-3),
                     "host_sample_goal_maps": {"maps": min(n_host, B), "ms_per_map": host},
                     "speedup_kernel_vs_host": host * B / k_ms}
    line = json.dumps(out)
    print(line)
    if args.out:
        with open(args.out, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
