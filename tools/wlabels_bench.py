#!/usr/bin/env python
"""Throughput of the vertex-weighted shortest-path kernel (nastar_wlabels.cuh; neural_astar.utils.data
compute_weighted_opt_labels / shortest_path_maps) on an H100, with the card's name and power limit read in the same
run, next to scipy.sparse.csgraph.dijkstra per map on one host core (a point of comparison, not an oracle: it sums in
float64 and does not produce the policy).

Workloads (inputs device-resident, one start and one goal per map):
  warcraft_12x12_b10000  10 000 all-passable 12x12 maps, costs uniform in [0.1, 10), start top-left, goal bottom-right;
  mazes_032_all1000      the 1000 mazes_032 problems, costs from the shipped checkpoint's encoder, map passability;
  all_064_test400        the 400 all_064 test problems, unit costs on their passable cells;
  random_128x128_b1024   1024 random 128x128 maps, 20 % obstacles, costs uniform in [0.1, 10), random start and goal.
Timing: CUDA events around 10 back-to-back calls, median of 3 trials.  --mechanism takes moore (default, 8 moves)
and/or news (4 moves N, E, W, S); with both, every timing alternates them trial by trial on the same inputs, the
first mechanism's row stays at the top level of each workload and the other is nested under its name.  Prints one JSON
object; --out also writes it.

    python tools/wlabels_bench.py [--out profiles/h100_wlabels_bench.json]
    python tools/wlabels_bench.py --mechanism news moore [--out profiles/h100_wlabels_bench_news.json]
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


_MOVES = ((-1, 0), (0, 1), (0, -1), (1, 0), (-1, 1), (-1, -1), (1, 1), (1, -1))
NUM_MOVES = {"moore": 8, "news": 4}     # NEWS moves are the first four Moore actions


def timed_alternating(fns, reps=10):
    """labels_bench.timed for several callables at once: each warmed up, then 3 trials in which every callable is
    timed in turn (CUDA events around `reps` back-to-back calls), so they share the same stretch of time.  Returns
    (median ms, trials) per callable."""
    for fn in fns:
        for _ in range(3):
            fn()
    trials = [[] for _ in fns]
    for _ in range(3):
        for i, fn in enumerate(fns):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            for _ in range(reps):
                fn()
            b.record()
            torch.cuda.synchronize()
            trials[i].append(a.elapsed_time(b) / reps)
    return [(sorted(t)[1], t) for t in trials]


def scipy_graph(cost, passable, goal, moves=_MOVES):
    """the reversed move graph: an edge t -> v of weight c[t] for every move v -> t"""
    from scipy.sparse import csr_matrix

    H, W = cost.shape
    ys, xs = np.mgrid[0:H, 0:W]
    src_ok = passable.ravel() != 0
    src_ok[goal] = False
    enter_ok = passable.ravel() != 0
    enter_ok[goal] = True
    rows, cols, w = [], [], []
    for dy, dx in moves:
        ty, tx = ys + dy, xs + dx
        inside = (ty >= 0) & (ty < H) & (tx >= 0) & (tx < W)
        v, t = (ys * W + xs)[inside], (ty * W + tx)[inside]
        keep = src_ok[v] & enter_ok[t]
        rows.append(t[keep])
        cols.append(v[keep])
        w.append(cost.ravel()[t[keep]].astype(np.float64))
    return csr_matrix((np.concatenate(w), (np.concatenate(rows), np.concatenate(cols))), shape=(H * W, H * W))


def scipy_arm(cost, passable, goal_idx, n, moves=_MOVES):
    from scipy.sparse.csgraph import dijkstra

    n = min(n, len(cost))
    build = solve = 0.0
    for i in range(n):
        t0 = time.perf_counter()
        g = scipy_graph(cost[i], passable[i], int(goal_idx[i]), moves)
        t1 = time.perf_counter()
        dijkstra(g, directed=True, indices=int(goal_idx[i]))
        t2 = time.perf_counter()
        build += t1 - t0
        solve += t2 - t1
    ms = (build + solve) * 1e3 / n
    return {"maps": n, "ms_per_map": ms, "maps_per_s": 1e3 / ms, "dijkstra_only_ms_per_map": solve * 1e3 / n}


def workloads(dev):
    from golden_util import Golden
    from neural_astar.planner import NeuralAstar

    rs = np.random.RandomState(1234)
    B, H, W = 10000, 12, 12
    wc = rs.uniform(0.1, 10.0, size=(B, 1, H, W)).astype(np.float32)
    yield ("warcraft_12x12_b10000", wc, np.ones_like(wc), np.zeros(B, np.int32), np.full(B, H * W - 1, np.int32))

    g = Golden("inputs_mazes032_all1000")
    state = np.load(os.path.join(ROOT, "tests", "golden", "mazes032_ckpt_planner_state.npz"))
    na = NeuralAstar(encoder_arch="CNN")
    na.load_state_dict({k: torch.from_numpy(state[k]) for k in state.files})
    na = na.to(dev).eval()
    maps, start, goal = (torch.from_numpy(x).to(dev) for x in (g.obst, g.start, g.goal))
    with torch.no_grad():
        cost = torch.cat([na.encode(maps[i:i + 100], start[i:i + 100], goal[i:i + 100]) for i in range(0, 1000, 100)])
    yield ("mazes_032_all1000", cost.cpu().numpy(), g.obst, g.z["start_idx"], g.z["goal_idx"])

    g = Golden("inputs_all064_test400")
    yield ("all_064_test400", (g.obst != 0).astype(np.float32), g.obst, g.z["start_idx"], g.z["goal_idx"])

    B, H, W = 1024, 128, 128
    cost = rs.uniform(0.1, 10.0, size=(B, 1, H, W)).astype(np.float32)
    pas = (rs.rand(B, 1, H, W) >= 0.2).astype(np.float32)
    s, gl = rs.randint(0, H * W, size=B).astype(np.int32), rs.randint(0, H * W, size=B).astype(np.int32)
    pas.reshape(B, -1)[np.arange(B), s] = 1.0
    pas.reshape(B, -1)[np.arange(B), gl] = 1.0
    yield ("random_128x128_b1024", cost, pas, s, gl)


def power_limit_w(index):
    """the enforced power limit in W (NVML, else a read-only nvidia-smi query), None if neither answers"""
    from labels_bench import power_limit_w as nvml_power_limit_w

    w = nvml_power_limit_w(index)
    if w is None:
        import subprocess

        try:
            w = float(subprocess.check_output(["nvidia-smi", "-i", str(index), "--query-gpu=power.limit",
                                               "--format=csv,noheader,nounits"], text=True).strip())
        except Exception:
            w = None
    return w


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--scipy-maps", type=int, default=50, help="maps per workload for the scipy arm")
    ap.add_argument("--mechanism", nargs="+", choices=sorted(NUM_MOVES), default=["moore"],
                    help="moore (8 moves) and/or news (4 moves); several are timed alternately")
    args = ap.parse_args()
    mechs = list(dict.fromkeys(args.mechanism))
    from neural_astar import _native
    from neural_astar.utils.data import compute_weighted_opt_labels, shortest_path_maps

    assert torch.cuda.is_available(), "wlabels_bench measures the GPU kernel: no GPU found"
    dev = torch.device("cuda:0")
    out = {"kernel": "nastar::weighted_labels_kernel (frontier Bellman-Ford + hop wavefronts + policy + roll-out, "
                     "one CTA per map, all state in shared memory)",
           "timing": "CUDA events around 10 back-to-back calls, median of 3 trials; inputs device-resident" +
                     ("; mechanisms alternated trial by trial" if len(mechs) > 1 else ""),
           "mechanism": mechs,
           "device": torch.cuda.get_device_name(dev), "power_limit_w": power_limit_w(0),
           "scipy_arm": "scipy.sparse.csgraph.dijkstra per map on one host core, float64, distances only (graph "
                        "construction included in ms_per_map); a point of comparison, not an oracle"}
    for name, cost_np, pas_np, start_np, goal_np in workloads(dev):
        B, _, H, W = cost_np.shape
        cost, pas = (torch.from_numpy(np.ascontiguousarray(x, np.float32)).to(dev) for x in (cost_np, pas_np))
        si = torch.from_numpy(np.asarray(start_np, np.int32)).to(dev)
        gi = torch.from_numpy(np.asarray(goal_np, np.int32)).to(dev)
        sm = torch.zeros_like(cost).view(B, -1).scatter_(1, si.long()[:, None], 1.0).view_as(cost)
        gm = torch.zeros_like(cost).view(B, -1).scatter_(1, gi.long()[:, None], 1.0).view_as(cost)
        k = timed_alternating([lambda m=m: _native.weighted_labels(cost, gi, pas, si, m) for m in mechs])
        kl = timed_alternating([lambda m=m: _native.weighted_labels(cost, gi, pas, mechanism=m) for m in mechs])
        a = timed_alternating([lambda m=m: compute_weighted_opt_labels(cost, gm, passable=pas, mechanism=m)
                               for m in mechs])
        p = timed_alternating([lambda m=m: shortest_path_maps(cost, sm, gm, passable=pas, mechanism=m)
                               for m in mechs])
        rows = {}
        for i, m in enumerate(mechs):
            (k_ms, k_trials), (kl_ms, _), (a_ms, _), (p_ms, _) = k[i], kl[i], a[i], p[i]
            r = _native.weighted_labels(cost, gi, pas, si, m)
            hops, status, pcost = r[1].view(B, -1), r[6], r[5]
            reached = (status & 4) == 0
            rows[m] = {"kernel_ms": k_ms, "kernel_ms_trials": k_trials, "maps_per_s": B / (k_ms * 1e-3),
                       "kernel_without_paths_ms": kl_ms, "compute_weighted_opt_labels_ms": a_ms,
                       "shortest_path_maps_ms": p_ms, "shortest_path_maps_maps_per_s": B / (p_ms * 1e-3),
                       "start_unreachable_maps": int((~reached).sum()), "max_hops": int(hops.max()),
                       "mean_path_cells": float((hops.gather(1, si.long()[:, None])[:, 0][reached] + 1).double()
                                                .mean()),
                       "mean_path_cost": float(pcost[reached].double().mean()),
                       "scipy": scipy_arm(cost_np[:, 0], pas_np[:, 0], goal_np, args.scipy_maps,
                                          _MOVES[:NUM_MOVES[m]])}
        out[name] = {"maps": B, "grid": f"{H}x{W}", **rows[mechs[0]], **{m: rows[m] for m in mechs[1:]}}
    line = json.dumps(out)
    print(line)
    if args.out:
        with open(args.out, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
