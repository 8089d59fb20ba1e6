#!/usr/bin/env python
"""Time of the reference heap A* on the GPU (nastar_pq.cuh; pq_astar(semantics="reference")) on an H100, with the
card's name and power limit read in the same run, next to the C oracle and the reference's own pq_astar on one host
core, and the differentiable engine (pq_astar's "engine" semantics, whose results differ) for context.

Workloads:
  mazes032_ckpt_100   the mazes_032 test split (100 maps) with the shipped checkpoint's costs (encoder on the GPU)
  all064_400          the 400 all_064 test problems, cost == map
  c5_256_binary_1024  1024 Config-5 256x256 maps (tools/c5_data.py, seed 1234), cost == map
  c5_256_random_1024  the same maps with random costs in [0, 1) (seed 1234)
GPU arms: CUDA events around back-to-back calls of the kernel alone (inputs device-resident, no status read), median
of 3 trials.  Host arms: host clock; the reference (staged in oracle/_ref/, with tests/pqdict_shim.py as pqdict) runs
on a subset of the maps where it would take minutes, and its time is then extrapolated to the whole batch and labelled
so.  Also counts how many of the 1000 mazes_032 problems with the checkpoint's costs, and of the 400 all_064 problems
with random costs, give different histories or paths under the two semantics, at g_ratio 0.5, 0.2 and 0.8.

--placement LIB_SHARED LIB_GLOBAL times the kernel with its state forced into shared memory and into the global
workspace on square maps of several sides, from two builds of the library:
    nvcc <the Makefile's flags> -DNASTAR_PQ_SMEM_MAX_BYTES=232448 -shared -o LIB_SHARED csrc/nastar_api.cu
    nvcc <the Makefile's flags> -DNASTAR_PQ_SMEM_MAX_BYTES=0 -shared -o LIB_GLOBAL csrc/nastar_api.cu

    python tools/pq_bench.py [--out profiles/h100_pq_bench.json] [--placement LIB_SHARED LIB_GLOBAL]
"""
import argparse
import contextlib
import ctypes
import io
import json
import os
import sys
import time

os.environ.setdefault("OMP_NUM_THREADS", "1")   # the C oracle on one host core
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for _p in (ROOT, os.path.join(ROOT, "neural-astar_b200"), os.path.join(ROOT, "tests"), os.path.join(ROOT, "tools")):
    if _p not in sys.path:
        sys.path.insert(0, _p)

import numpy as np  # noqa: E402
import torch  # noqa: E402

from labels_bench import timed  # noqa: E402
from wlabels_bench import power_limit_w  # noqa: E402


def workloads(planner):
    from c5_data import c5_maps
    from golden_util import Golden

    mz = Golden("inputs_mazes032_all1000")
    sl = slice(900, 1000)
    with torch.no_grad():
        cost = planner.encode(*(torch.from_numpy(x[sl]).cuda() for x in (mz.obst, mz.start, mz.goal))).cpu().numpy()
    yield "mazes032_ckpt_100", cost, mz.start[sl], mz.goal[sl], mz.obst[sl], 100
    a = Golden("inputs_all064_test400")
    yield "all064_400", a.obst, a.start, a.goal, a.obst, 40
    obst, start, goal = c5_maps(1024, 256, 256, seed=1234)
    yield "c5_256_binary_1024", obst, start, goal, obst, 4
    cost = np.random.RandomState(1234).rand(1024, 1, 256, 256).astype(np.float32)
    yield "c5_256_random_1024", cost, start, goal, obst, 4


def reference_seconds(solve, cost, start, goal, obst, n):
    t0 = time.perf_counter()
    for b in range(n):
        with contextlib.redirect_stdout(io.StringIO()):
            solve(cost[b, 0].astype(np.float64), start[b, 0], goal[b, 0], obst[b, 0], 0.5)
    return time.perf_counter() - t0


def raw_pq(lib_path):
    """nastar_b200_pq_astar of another build of the library, with _native's signature"""
    from neural_astar import _native

    L = ctypes.CDLL(lib_path)
    for name in ("nastar_b200_pq_astar", "nastar_b200_pq_astar_workspace_bytes"):
        fn = getattr(L, name)
        fn.restype, fn.argtypes = _native._SIGNATURES[name]

    def run(c, s, g, o, out):
        B, _, H, W = c.shape
        hist, paths, status, exp, ws = out
        N = H * W
        rc = L.nastar_b200_pq_astar(c.data_ptr(), N, s.data_ptr(), N, g.data_ptr(), N, o.data_ptr(), N, B, H, W, 0.5,
                                    hist.data_ptr(), paths.data_ptr(), status.data_ptr(), exp.data_ptr(),
                                    ws.data_ptr(), ws.numel(), torch.cuda.current_stream().cuda_stream)
        assert rc == 0, rc

    return L, run


def placement_sweep(lib_shared, lib_global):
    from c5_data import c5_maps

    res = []
    libs = {k: raw_pq(p) for k, p in (("shared", lib_shared), ("global", lib_global))}
    for side in (32, 36, 40, 44, 48, 64, 80, 104):
        B = 2048 if side <= 64 else 1024
        obst, start, goal = c5_maps(B, side, side, seed=side)
        cost = np.random.RandomState(side).rand(B, 1, side, side).astype(np.float32)
        c, s, g, o = (torch.from_numpy(x).cuda() for x in (cost, start, goal, obst))
        row = {"side": side, "B": B, "state_bytes": 20 * side * side}
        outs = {}
        for k, (L, run) in libs.items():
            ws_bytes = int(L.nastar_b200_pq_astar_workspace_bytes(B, side, side))
            out = (torch.empty((B, 1, side, side), device="cuda"),
                   torch.empty((B, 1, side, side), dtype=torch.int64, device="cuda"),
                   torch.empty(B, dtype=torch.int32, device="cuda"), torch.empty(B, dtype=torch.int32, device="cuda"),
                   torch.empty(ws_bytes, dtype=torch.uint8, device="cuda"))
            ms, trials = timed(lambda: run(c, s, g, o, out), reps=3)
            row[f"{k}_ms"] = round(ms, 3)
            outs[k] = [t.cpu() for t in out[:4]]
        row["outputs_equal"] = all(torch.equal(a, b) for a, b in zip(outs["shared"], outs["global"]))
        print(json.dumps(row), flush=True)
        res.append(row)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--placement", nargs=2, metavar=("LIB_SHARED", "LIB_GLOBAL"), default=None)
    args = ap.parse_args()
    from neural_astar import _native
    from neural_astar.planner import NeuralAstar
    from oracle import pq as pq_oracle
    from pq_golden import staged_solve_single

    assert torch.cuda.is_available(), "pq_bench measures the GPU kernel: no GPU found"
    torch.set_num_threads(1)
    dev = torch.device("cuda:0")
    out = {"kernel": "nastar::pq_astar_kernel (the reference's heap A*, one warp per map, persistent one-warp CTAs)",
           "timing": "GPU arms: CUDA events around back-to-back kernel calls, median of 3 trials; host arms: host clock",
           "device": torch.cuda.get_device_name(dev), "power_limit_w": power_limit_w(0),
           "oracle_arm": "oracle/pq_oracle.c (gcc -O2), one host core",
           "reference_arm": "the reference's pq_astar.solve_single (staged, pqdict shim), one host core",
           "engine_arm": "the differentiable engine with no step cap (pq_astar semantics='engine'): different results",
           "workloads": {}}
    state = np.load(os.path.join(ROOT, "tests", "golden", "mazes032_ckpt_planner_state.npz"))
    planner = NeuralAstar(encoder_arch="CNN")
    planner.load_state_dict({k: torch.from_numpy(state[k]) for k in state.files})
    planner = planner.cuda().eval()
    solve = staged_solve_single()
    for name, cost, start, goal, obst, n_ref in workloads(planner):
        B, _, H, W = obst.shape
        c, s, g, o = (torch.from_numpy(np.ascontiguousarray(x, dtype=np.float32)).cuda()
                      for x in (cost, start, goal, obst))
        ms, trials = timed(lambda: _native.pq_astar(c, s, g, o, 0.5), reps=3 if H > 64 else 10)
        hist, paths, status, exp = (t.cpu().numpy() for t in _native.pq_astar(c, s, g, o, 0.5))
        t0 = time.perf_counter()
        ref = pq_oracle.pq_astar(cost, start, goal, obst, 0.5)
        oracle_s = time.perf_counter() - t0
        assert all(np.array_equal(a, b) for a, b in zip((hist, paths, status, exp), ref)), name
        eng_ms, _ = timed(lambda: _native.forward(c, s, g, o, 0.5, H * W, False), reps=3 if H > 64 else 10)
        row = {"B": B, "H": H, "W": W, "kernel_ms": round(ms, 3), "kernel_trials_ms": [round(t, 3) for t in trials],
               "maps_per_s": round(B / ms * 1e3, 1), "expansions_mean": round(float(exp.mean()), 1),
               "solved": int((status == 0).sum()), "oracle_1core_ms": round(oracle_s * 1e3, 1),
               "engine_ms": round(eng_ms, 3), "kernel_equals_oracle": True}
        if solve is not None:
            sec = reference_seconds(solve, cost, start, goal, obst, min(n_ref, B))
            row["reference_1core_ms"] = round(sec * B / min(n_ref, B) * 1e3, 1)
            row["reference_maps_timed"] = min(n_ref, B)
            row["reference_extrapolated"] = n_ref < B
        out["workloads"][name] = row
        print(name, json.dumps(row), flush=True)
    # how far the default ("engine") semantics is from the reference's on learned costs
    from golden_util import Golden

    mz = Golden("inputs_mazes032_all1000")
    maps, start, goal = (torch.from_numpy(x).cuda() for x in (mz.obst, mz.start, mz.goal))
    from neural_astar.planner.pq_astar import pq_astar

    with torch.no_grad():
        costs = {"mazes032_1000_ckpt": (planner.encode(maps, start, goal), maps, start, goal)}
    a = Golden("inputs_all064_test400")
    m4, s4, g4 = (torch.from_numpy(x).cuda() for x in (a.obst, a.start, a.goal))
    costs["all064_400_random"] = (torch.from_numpy(np.random.RandomState(64).rand(a.B, 1, a.H, a.W).astype(
        np.float32)).cuda(), m4, s4, g4)
    dev_out = {}
    for name, (cost, maps, start, goal) in costs.items():
        for gr in (0.5, 0.2, 0.8):
            e = pq_astar(cost, start, goal, maps, g_ratio=gr, semantics="engine")
            r = pq_astar(cost, start, goal, maps, g_ratio=gr, semantics="reference")
            dh = (e.histories != r.histories).flatten(1).any(1)
            dp = (e.paths != r.paths).flatten(1).any(1)
            dl = e.paths.flatten(1).sum(1) != r.paths.flatten(1).sum(1)
            dev_out[f"{name}_g{gr}"] = {"maps": int(cost.shape[0]), "histories_differ": int(dh.sum()),
                                        "paths_differ": int(dp.sum()), "path_length_differs": int(dl.sum())}
            print(f"{name}_g{gr}", json.dumps(dev_out[f"{name}_g{gr}"]), flush=True)
    out["engine_vs_reference"] = dev_out
    out["engine_vs_reference_note"] = ("maps whose histories / paths differ between pq_astar's two semantics; "
                                       "mazes032_1000_ckpt: checkpoint costs from the GPU encoder; all064_400_random: "
                                       "random costs in [0, 1), seed 64")
    if args.placement:
        out["placement"] = placement_sweep(*args.placement)
    text = json.dumps(out, indent=1)
    print(text)
    if args.out:
        with open(args.out, "w") as fh:
            fh.write(text + "\n")


if __name__ == "__main__":
    main()
