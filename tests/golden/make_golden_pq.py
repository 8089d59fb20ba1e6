#!/usr/bin/env python
"""Goldens of the reference's heap A* (`pq_astar.solve_single`, use_differentiable_astar=False) under tests/golden/pq/,
by RUNNING THE REFERENCE's own code: the staged copy in oracle/_ref/ (oracle/stage_ref.py, run by build()), with
tests/pqdict_shim.py injected as `pqdict` (see its docstring for what that assumes about pqdict 1.2.0).

    python tests/golden/make_golden_pq.py     # where oracle/_ref/ is staged

Costs are cast to float64 before `solve_single`: the reference's pinned NumPy 1 computes g_ratio * cost[nb] in fp64
(a Python float times an np.float32 scalar), NumPy >= 2 in fp32; the widening is exact and gives NumPy 1's result.

Files (one g_ratio and one shape each; costs stored as fp32, outputs bit-packed, plus status and expansions):
  fixture64            the reference test's 64x64 fixture (tests/astar_test.py), cost == map
  mazes032_ckpt_g{05,02,08}  the 100 mazes_032 test problems with the shipped checkpoint's costs (CPU encoder)
  ties32_g{10,00}      open and symmetric 32x32 maps, cost == map, at g = 1 (pure g) and g = 0 (pure h)
  ties32_costs         random maps with costs quantised to {0, 1/4, 1/2, 1}, and with all-zero costs
  edge32               start == goal, goal on an obstacle, start on an obstacle, a walled-off goal, negative and zero
                       costs
  line1x40, line40x1   one-row and one-column maps
  edge_{20x12,5x40,33x31}  the inputs of the existing edge fixtures, with seeded random costs
  large128, large256   one learned-cost map each: the large128_learned costs, and the checkpoint's costs on a
                       large256_vanilla map
"""
from __future__ import annotations

import contextlib
import io
import json
import os
import sys
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
OUT = os.path.join(HERE, "pq")
sys.path.insert(0, os.path.dirname(HERE))
import pqdict_shim  # noqa: E402

_pq = types.ModuleType("pqdict")
_pq.pqdict = pqdict_shim.pqdict
sys.modules["pqdict"] = _pq
_smp = types.ModuleType("segmentation_models_pytorch")
_smp.Unet = None
sys.modules["segmentation_models_pytorch"] = _smp
sys.path.insert(0, os.path.join(ROOT, "oracle", "_ref"))
import torch  # noqa: E402
from neural_astar.planner import NeuralAstar  # noqa: E402  the staged reference
from neural_astar.planner.pq_astar import solve_single  # noqa: E402

from golden_util import Golden  # noqa: E402


def pack(x) -> np.ndarray:
    x = np.asarray(x)
    return np.packbits(x.reshape(x.shape[0], -1) != 0, axis=1)


def run(cost, start, goal, obst, g_ratio):
    """solve_single per map; returns hist, paths, status (0 solved, 1 goal not found), expansions (closed cells)."""
    hist, paths, status, exp = [], [], [], []
    for c, s, g, m in zip(cost, start, goal, obst):
        with contextlib.redirect_stdout(io.StringIO()) as out:
            h, p = solve_single(c[0].astype(np.float64), s[0], g[0], m[0], g_ratio)
        hist.append(h); paths.append(p)
        status.append(1 if "goal not found" in out.getvalue() else 0)
        exp.append(int(h.sum()))
    return np.stack(hist), np.stack(paths), np.array(status, np.int32), np.array(exp, np.int32)


def save(name, desc, g_ratio, cost, start, goal, obst):
    B, _, H, W = obst.shape
    cost = np.asarray(cost, np.float32)
    hist, paths, status, exp = run(cost, start, goal, obst, g_ratio)
    flat = lambda x: x.reshape(B, -1)  # noqa: E731
    meta = dict(desc=desc, g_ratio=g_ratio, numpy=np.__version__,
                reference="omron-sinicx/neural-astar @473edbbd (src/neural_astar/planner/pq_astar.py solve_single)",
                pqdict="tests/pqdict_shim.py")
    os.makedirs(OUT, exist_ok=True)
    path = os.path.join(OUT, name + ".npz")
    np.savez_compressed(path, meta=np.array(json.dumps(meta)), shape=np.array([B, H, W], np.int32),
                        obst_bits=pack(obst[:, 0]), start_idx=flat(start).argmax(1).astype(np.int32),
                        goal_idx=flat(goal).argmax(1).astype(np.int32), cost=cost.reshape(B, H, W),
                        hist_bits=pack(hist), path_bits=pack(paths), status=status, expansions=exp)
    print(f"pq/{name}: B={B} {H}x{W} g={g_ratio} solved={int((status == 0).sum())} "
          f"expansions={int(exp.sum())} {os.path.getsize(path) / 1024:.1f} KiB")


def onehot(B, H, W, idx):
    x = np.zeros((B, 1, H * W), np.float32)
    x[np.arange(B), 0, np.asarray(idx)] = 1
    return x.reshape(B, 1, H, W)


def ckpt_encoder():
    z = np.load(os.path.join(HERE, "mazes032_ckpt_planner_state.npz"))
    planner = NeuralAstar(encoder_arch="CNN")
    planner.load_state_dict({k: torch.from_numpy(np.asarray(z[k])) for k in z.files})
    return planner.eval()


def ckpt_costs(planner, obst, start, goal):
    with torch.no_grad():
        return planner.encode(*(torch.from_numpy(x) for x in (obst, start, goal))).numpy()


def main():
    torch.set_num_threads(8)
    rng = np.random.RandomState(20261016)
    planner = ckpt_encoder()

    fx = Golden("fixture64_vanilla")
    save("fixture64", "the reference test's 64x64 fixture, cost == map", 0.5, fx.obst, fx.start, fx.goal, fx.obst)

    mz = Golden("inputs_mazes032_all1000")
    sl = slice(900, 1000)   # the test split
    obst, start, goal = mz.obst[sl], mz.start[sl], mz.goal[sl]
    cost = ckpt_costs(planner, obst, start, goal)
    for tag, g in (("05", 0.5), ("02", 0.2), ("08", 0.8)):
        save(f"mazes032_ckpt_g{tag}", "mazes_032 test split, shipped checkpoint's costs", g, cost, start, goal, obst)

    # open and symmetric maps: every tie the heap can meet
    H = W = 32
    obst = np.ones((6, 1, H, W), np.float32)
    obst[3, 0, 8:24, 15:17] = 0    # a symmetric wall between start and goal
    obst[4, 0, 12:20, 12:20] = 0   # a centred block
    obst[5, 0] = rng.rand(H, W) > 0.15
    s_idx = [0, 16 * W, 5 * W + 5, 16 * W + 3, 0, 2 * W + 2]
    g_idx = [H * W - 1, 16 * W + 31, 26 * W + 26, 16 * W + 28, H * W - 1, 29 * W + 29]
    start, goal = onehot(6, H, W, s_idx), onehot(6, H, W, g_idx)
    obst[5, 0].flat[[s_idx[5], g_idx[5]]] = 1
    save("ties32_g10", "open and symmetric maps, cost == map, pure g", 1.0, obst, start, goal, obst)
    save("ties32_g00", "open and symmetric maps, cost == map, pure h", 0.0, obst, start, goal, obst)

    B = 8
    obst = (rng.rand(B, 1, H, W) > 0.25).astype(np.float32)
    s_idx, g_idx = rng.randint(0, H * W, B), rng.randint(0, H * W, B)
    start, goal = onehot(B, H, W, s_idx), onehot(B, H, W, g_idx)
    for b in range(B):
        obst[b, 0].flat[[s_idx[b], g_idx[b]]] = 1
    cost = rng.choice(np.array([0, 0.25, 0.5, 1], np.float32), size=(B, 1, H, W))
    cost[B // 2:] = 0
    save("ties32_costs", "costs in {0, 1/4, 1/2, 1} (maps 0-3) and all-zero costs (maps 4-7)", 0.5, cost, start, goal,
         obst)

    # edge cases on 32x32
    B = 7
    obst = (rng.rand(B, 1, H, W) > 0.2).astype(np.float32)
    s_idx = [100, 40, 33, 0, 70, 500, 900]
    g_idx = [100, 900, 990, H * W - 1, 980, 20, 60]
    for b in range(B):
        obst[b, 0].flat[[s_idx[b], g_idx[b]]] = 1
    obst[1, 0].flat[900] = 0                       # goal on an obstacle: unreachable
    obst[2, 0].flat[33] = 0                        # start on an obstacle: never tested, the search runs
    obst[3, 0, 28:32, 28:32] = 0                   # a walled-off goal
    obst[3, 0, 29:32, 29:32] = 1
    cost = rng.rand(B, 1, H, W).astype(np.float32)
    cost[4] -= 0.5                                 # negative costs
    cost[5] = -rng.rand(H, W)
    cost[6] = 0
    cost[6, 0, 10:20] = -1
    save("edge32", "start == goal, goal on an obstacle, start on an obstacle, walled-off goal, negative and zero costs",
         0.5, cost, onehot(B, H, W, s_idx), onehot(B, H, W, g_idx), obst)

    for name, (H, W) in (("line1x40", (1, 40)), ("line40x1", (40, 1))):
        B = 4
        obst = np.ones((B, 1, H, W), np.float32)
        obst[3].flat[20] = 0
        s_idx, g_idx = [0, 39, 10, 0], [39, 0, 30, 39]
        save(name, "one-row / one-column maps, the last one cut", 0.5, rng.rand(B, 1, H, W),
             onehot(B, H, W, s_idx), onehot(B, H, W, g_idx), obst)

    for shape in ("20x12", "5x40", "33x31"):
        e = Golden(f"edge_rand_{shape}")
        save(f"edge_{shape}", f"inputs of edge_rand_{shape}, seeded random costs in [0, 1)", 0.5,
             rng.rand(e.B, 1, e.H, e.W), e.start, e.goal, e.obst)

    lg = Golden("large128_learned")
    save("large128", "large128_learned map 0 and its costs", 0.5, lg.cost[:1], lg.start[:1], lg.goal[:1], lg.obst[:1])
    lv = Golden("large256_vanilla")
    o, s, g = lv.obst[:1], lv.start[:1], lv.goal[:1]
    save("large256", "large256_vanilla map 0, the shipped checkpoint's costs", 0.5, ckpt_costs(planner, o, s, g), s, g, o)


if __name__ == "__main__":
    main()
