#!/usr/bin/env python
"""4-connected (NEWS) search against Moore on the GPU, with the card's name and power limit read in the same run.

    python tools/news_bench.py --out profiles/h100_news_bench.json

Rows (CUDA events, median of three trials, NEWS and Moore measured alternately on the same inputs):
  kernel_100     the search alone (_native.forward), the 100 mazes_032 test problems of tests/golden/news/
                 news_mazes032_vanilla: map as cost (VanillaAstar) and the checkpoint's learned costs
  kernel_100k    the same problems tiled to B = 100 000
  pipelined      a NeuralAstar inference step (checkpoint weights) through PipelinedPlanner, B = 1000
A NEWS step opens at most 4 cells instead of 8 but may need more steps: the mean selection steps per map are reported
next to each time.
"""
import argparse
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
for p in (ROOT, os.path.join(ROOT, "neural-astar_b200"), os.path.join(ROOT, "tests"), HERE):
    if p not in sys.path:
        sys.path.insert(0, p)

import numpy as np  # noqa: E402
import torch  # noqa: E402

from labels_bench import power_limit_w, timed  # noqa: E402

MECHS = ("news", "moore")


def _inputs(dev, reps):
    from golden_util import Golden

    v, n = Golden("news/news_mazes032_vanilla"), Golden("news/news_mazes032_neural")
    t = [torch.from_numpy(x).to(dev).repeat(reps, 1, 1, 1) for x in (v.obst, v.start, v.goal, n.cost)]
    return t


def kernel_rows(dev, reps, n_timed):
    from neural_astar import _native

    maps, start, goal, learned = _inputs(dev, reps)
    T = 32 * 32
    out = {}
    for kind, cost in (("vanilla", maps), ("learned", learned)):
        row = {}
        for mech in MECHS * 2:   # alternate: NEWS, Moore, NEWS, Moore; the second pair is kept
            ms, trials = timed(lambda: _native.forward(cost, start, goal, maps, 0.5, T, mechanism=mech), n_timed)
            ns = _native.forward(cost, start, goal, maps, 0.5, T, mechanism=mech)[3]
            row[mech] = {"ms": ms, "trials_ms": trials, "maps_per_s": cost.shape[0] / ms * 1e3,
                         "mean_steps": float(ns.float().mean())}
        row["news_over_moore"] = row["news"]["ms"] / row["moore"]["ms"]
        out[kind] = row
    return out


def pipelined_row(dev, B=1000, n_batches=20):
    from neural_astar.planner import NeuralAstar
    from neural_astar.utils.inference import PipelinedPlanner

    state = np.load(os.path.join(ROOT, "tests", "golden", "mazes032_ckpt_planner_state.npz"))
    maps, start, goal, _ = _inputs(dev, B // 100)
    row = {}
    for mech in MECHS * 2:
        na = NeuralAstar(encoder_arch="CNN", mechanism=mech)
        sd = {k: torch.from_numpy(state[k]) for k in state.files}
        sd["astar.neighbor_filter"] = na.astar.neighbor_filter.detach().clone()
        na.load_state_dict(sd)
        na = na.to(dev).eval()
        pipe = PipelinedPlanner(na, maps, start, goal)

        def run():
            for _ in range(n_batches):
                pipe.submit(maps, start, goal)
            pipe.drain()

        ms, trials = timed(run, 3)
        row[mech] = {"ms_per_batch": ms / n_batches, "trials_ms": trials, "maps_per_s": B * n_batches / ms * 1e3}
    row["news_over_moore"] = row["news"]["ms_per_batch"] / row["moore"]["ms_per_batch"]
    return row


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None, help="also write the JSON line to this file")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("news_bench measures the GPU search: no CUDA device")
    dev = torch.device("cuda:0")
    out = {"what": "NEWS (4-connected) vs Moore search, CUDA events, median of 3 trials",
           "device": torch.cuda.get_device_name(dev), "power_limit_w": power_limit_w(0)}
    out["kernel_100"] = kernel_rows(dev, 1, 200)
    out["kernel_100k"] = kernel_rows(dev, 1000, 5)
    out["pipelined_B1000"] = pipelined_row(dev)
    line = json.dumps(out)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
