#!/usr/bin/env python
"""Reference-pinned vectors of the 4-connected (NEWS) search, made by RUNNING THE REFERENCE.

    python tests/golden/make_golden_news.py        # build container only (needs /root/reference)

The reference's own DifferentiableAstar / VanillaAstar / NeuralAstar (src/neural_astar/planner) are given the
planning-datasets generator's NorthEastWestSouth pieces, exactly as a user of the reference configures them:
    astar.neighbor_filter.data = NorthEastWestSouth.get_neighbor_filter()     (mechanism.py:113-121)
    astar.get_heuristic        = NorthEastWestSouth.get_heuristic             (mechanism.py:123-131)
mechanism.py is loaded by file path (it imports only numpy and torch).  Every stored output comes from the reference;
the CPU label oracle in NEWS mode (oracle/labels.py) is only used to draw starts that can reach the goal over
4-connected moves (4-connectivity splits regions that Moore joins, and an unreachable goal makes the reference raise
IndexError).  Files, under tests/golden/news/ (all square: the generator's heuristic reads size = shape[-1]):
  news_mazes032_vanilla   mazes_032 test split (100 maps), shipped goals, VanillaAstar: engine 1
  news_mazes032_neural    the same problems with the shipped checkpoint's learned costs (eval), then one training-mode
                          batch (Tmax 0.25) with the autograd gradient of sum(histories * rand_G): engine 1
  news_mazes032_lowg      16 of them at g_ratio = 0.2 (batch-coupled) with learned costs and a gradient
  news_all064_vanilla     40 all_064 test maps, 64x64, VanillaAstar: engine 4
  news_large128_learned   2 random 128x128 maps with random learned costs: engine 2
  news_all064_learned     8 more all_064 test maps with random learned costs (eval), then one training-mode batch
                          (Tmax 0.25) with the autograd gradient of sum(histories * rand_G): engine 4
  news_all064_lowg        4 of them at g_ratio = 0.3 (batch-coupled) with a gradient
  news_large144_learned   2 random 144x144 maps with random learned costs: engine 3
  news_mazes032_gr08      mazes_032 test maps 84..99, new starts and random learned costs, g_ratio = 0.8, with a
                          gradient: engine 1

    python tests/golden/make_golden_news.py --more   # only the last four
"""
import importlib.util
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))
import make_golden as mg  # noqa: E402  (stubs the unused third-party imports, puts the reference on sys.path)
import torch  # noqa: E402
from neural_astar.planner import VanillaAstar  # noqa: E402  (the reference's)
from neural_astar.planner.differentiable_astar import DifferentiableAstar  # noqa: E402

from oracle import labels as label_oracle  # noqa: E402

# a directory of their own: tests/golden/*.npz are Moore search vectors that golden_util.all_names() hands to every
# Moore parity test
mg.OUT = os.path.join(HERE, "news")
os.makedirs(mg.OUT, exist_ok=True)

_spec = importlib.util.spec_from_file_location(
    "ref_mechanism", f"{mg.REF}/planning-datasets/planning_datasets_utils/mechanism.py")
mechanism = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(mechanism)
NEWS = mechanism.NorthEastWestSouth


def make_news(astar):
    """Configure a reference DifferentiableAstar for the generator's NEWS mechanism."""
    astar.neighbor_filter.data = NEWS.get_neighbor_filter()
    astar.get_heuristic = NEWS.get_heuristic
    return astar


def run_news(cost, start, goal, obst, g_ratio=0.5, Tmax=1.0, training=False, grad_hist=None):
    astar = make_news(DifferentiableAstar(g_ratio=g_ratio, Tmax=Tmax))
    astar.train(training)
    need_grad = grad_hist is not None
    cost = cost.clone().requires_grad_(need_grad)
    out = astar(cost, start, goal, obst, store_intermediate_results=True)
    frames = out.intermediate_results[:-1]
    trace = torch.stack([fr["paths"].reshape(fr["paths"].shape[0], -1).argmax(1) for fr in frames], 1)
    res = dict(hist=out.histories.detach(), paths=out.paths.detach(), T_batch=len(frames), trace=trace.to(torch.int32))
    if need_grad:
        loss = (out.histories * grad_hist).sum()
        loss.backward()
        res["grad_cost"] = cost.grad.detach()
    return res


def news_starts(maps, goal_idx, seed):
    """One start per map, uniform over the cells that reach the goal over 4-connected moves (goal excluded)."""
    rng = np.random.RandomState(seed)
    dists = label_oracle.opt_labels(maps, goal_idx, mechanism="news")[0]
    B, _, H, W = maps.shape
    start = np.zeros((B, 1, H, W), np.float32)
    for b in range(B):
        d = dists[b, 0].reshape(-1)
        cand = np.flatnonzero((d > -(H * W)) & (d < 0))
        start[b, 0].reshape(-1)[cand[rng.randint(len(cand))]] = 1.0
    return torch.from_numpy(start)


def check_heuristic():
    """The project's get_news_heuristic restates NEWS.get_heuristic; pin the reference's values on square inputs."""
    g = torch.zeros(3, 1, 32, 32)
    g[0, 0, 0, 0] = g[1, 0, 31, 5] = g[2, 0, 17, 9] = 1
    return g, NEWS.get_heuristic(g[:, 0])


def load_split(npz, n):
    z = np.load(f"{mg.MPD}/{npz}")
    maps = torch.from_numpy(z["arr_8"][:n].astype(np.float32)).unsqueeze(1)   # test split: maps, goals
    goals = torch.from_numpy(z["arr_9"][:n].astype(np.float32))                 # already [n, 1, H, W]
    return maps, goals


def main():
    torch.manual_seed(0)
    # --- mazes_032, shipped goals, vanilla ---------------------------------------------------------
    maps, goals = load_split("mazes_032_moore_c8.npz", 100)
    gi = mg.onehot_idx(goals)
    starts = news_starts(maps.numpy(), gi, 1)
    with torch.no_grad():
        planner = VanillaAstar()
        make_news(planner.astar)
        out = planner(maps, starts, goals)
    res = run_news(maps, starts, goals, maps)
    assert torch.equal(out.histories, res["hist"]) and torch.equal(out.paths, res["paths"])
    mg.save("news_mazes032_vanilla", dict(desc="mazes_032 test split, NEWS VanillaAstar", g_ratio=0.5, vanilla=True,
                                          mechanism="news"), **mg.common_arrays(maps, starts, goals, res))

    # --- the same problems with the checkpoint's learned costs ----------------------------------------
    planner, _ = mg.load_ckpt_planner()
    make_news(planner.astar)
    with torch.no_grad():
        cost = planner.encode(maps, starts, goals)
        out = planner(maps, starts, goals)
    res = run_news(cost, starts, goals, maps)
    assert torch.equal(out.histories, res["hist"]) and torch.equal(out.paths, res["paths"])
    arrays = mg.common_arrays(maps, starts, goals, res, cost=cost)
    rand_G = torch.from_numpy(np.random.RandomState(5).randn(100, 1, 32, 32).astype(np.float32))
    tr = run_news(cost, starts, goals, maps, Tmax=0.25, training=True, grad_hist=rand_G)
    arrays.update(train_hist_bits=mg.pack(tr["hist"][:, 0]), train_path_bits=mg.pack(tr["paths"][:, 0]),
                  train_T_batch=np.int32(tr["T_batch"]), train_trace=tr["trace"].numpy(),
                  rand_G=rand_G[:, 0].numpy(), train_grad_cost=tr["grad_cost"][:, 0].numpy())
    hq, hv = check_heuristic()
    arrays.update(heur_goal_idx=mg.onehot_idx(hq), heur_values=hv.numpy().astype(np.float32))
    mg.save("news_mazes032_neural", dict(desc="mazes_032 test split, checkpoint costs, NEWS; train Tmax 0.25 + grad",
                                         g_ratio=0.5, Tmax_train=0.25, mechanism="news"), **arrays)

    # --- g_ratio = 0.2, batch-coupled ----------------------------------------------------------------
    sl = slice(0, 16)
    res = run_news(cost[sl], starts[sl], goals[sl], maps[sl], g_ratio=0.2, grad_hist=rand_G[sl])
    arrays = mg.common_arrays(maps[sl], starts[sl], goals[sl], res, cost=cost[sl])
    arrays.update(rand_G=rand_G[sl, 0].numpy(), rand_grad_cost=res["grad_cost"][:, 0].numpy())
    mg.save("news_mazes032_lowg", dict(desc="16 mazes_032 problems, checkpoint costs, NEWS, g_ratio 0.2 + grad",
                                       g_ratio=0.2, mechanism="news"), **arrays)

    # --- all_064, 64x64 ------------------------------------------------------------------------------
    maps, goals = load_split("all_064_moore_c16.npz", 40)
    starts = news_starts(maps.numpy(), mg.onehot_idx(goals), 2)
    res = run_news(maps, starts, goals, maps)
    mg.save("news_all064_vanilla", dict(desc="40 all_064 test maps, NEWS VanillaAstar", g_ratio=0.5, vanilla=True,
                                        mechanism="news"), **mg.common_arrays(maps, starts, goals, res))

    # --- 128x128, learned costs ------------------------------------------------------------------------
    rng = np.random.RandomState(11)
    maps = torch.from_numpy((rng.rand(2, 1, 128, 128) > 0.25).astype(np.float32))
    goals = torch.zeros_like(maps)
    goals[0, 0, 100, 110] = goals[1, 0, 5, 120] = 1
    maps[goals > 0] = 1
    starts = news_starts(maps.numpy(), mg.onehot_idx(goals), 3)
    cost = torch.from_numpy(rng.rand(2, 1, 128, 128).astype(np.float32))
    res = run_news(cost, starts, goals, maps)
    mg.save("news_large128_learned", dict(desc="2 random 128x128 maps, random costs, NEWS", g_ratio=0.5,
                                          mechanism="news"), **mg.common_arrays(maps, starts, goals, res, cost=cost))
    more()


def more():
    """Learned costs above 32x32, a batch-coupled 64x64 batch, a generic-engine workspace map and g_ratio 0.8.  Host
    memory: the reference keeps ~10 [B,H,W] fp32 tensors per step of a differentiated loop, so B x steps is kept to
    about 1 GB (all064 training: 8 maps x 1024 steps) to 3 GB (all064 lowg: 4 maps x at most 4096 steps)."""
    # --- all_064 maps 40..47 with random learned costs: eval, then a training batch with a gradient ------------------
    maps, goals = load_split("all_064_moore_c16.npz", 48)
    maps, goals = maps[40:], goals[40:]
    starts = news_starts(maps.numpy(), mg.onehot_idx(goals), 4)
    rng = np.random.RandomState(21)
    cost = torch.from_numpy(rng.rand(8, 1, 64, 64).astype(np.float32))
    res = run_news(cost, starts, goals, maps)
    arrays = mg.common_arrays(maps, starts, goals, res, cost=cost)
    rand_G = torch.from_numpy(rng.randn(8, 1, 64, 64).astype(np.float32))
    tr = run_news(cost, starts, goals, maps, Tmax=0.25, training=True, grad_hist=rand_G)
    arrays.update(train_hist_bits=mg.pack(tr["hist"][:, 0]), train_path_bits=mg.pack(tr["paths"][:, 0]),
                  train_T_batch=np.int32(tr["T_batch"]), train_trace=tr["trace"].numpy(),
                  rand_G=rand_G[:, 0].numpy(), train_grad_cost=tr["grad_cost"][:, 0].numpy())
    mg.save("news_all064_learned", dict(desc="8 all_064 test maps, random costs, NEWS; train Tmax 0.25 + grad",
                                        g_ratio=0.5, Tmax_train=0.25, mechanism="news"), **arrays)

    # --- 4 of them at g_ratio 0.3: batch-coupled, eval length, with a gradient --------------------------------------
    sl = slice(0, 4)
    res = run_news(cost[sl], starts[sl], goals[sl], maps[sl], g_ratio=0.3, grad_hist=rand_G[sl])
    arrays = mg.common_arrays(maps[sl], starts[sl], goals[sl], res, cost=cost[sl])
    arrays.update(rand_G=rand_G[sl, 0].numpy(), rand_grad_cost=res["grad_cost"][:, 0].numpy())
    mg.save("news_all064_lowg", dict(desc="4 all_064 test maps, random costs, NEWS, g_ratio 0.3 + grad", g_ratio=0.3,
                                     mechanism="news"), **arrays)

    # --- 144x144: the generic engine's HBM workspace -----------------------------------------------------------------
    rng = np.random.RandomState(12)
    maps = torch.from_numpy((rng.rand(2, 1, 144, 144) > 0.25).astype(np.float32))
    goals = torch.zeros_like(maps)
    goals[0, 0, 130, 20] = goals[1, 0, 71, 140] = 1
    maps[goals > 0] = 1
    starts = news_starts(maps.numpy(), mg.onehot_idx(goals), 5)
    cost = torch.from_numpy(rng.rand(2, 1, 144, 144).astype(np.float32))
    with torch.no_grad():
        res = run_news(cost, starts, goals, maps)
    mg.save("news_large144_learned", dict(desc="2 random 144x144 maps, random costs, NEWS", g_ratio=0.5,
                                          mechanism="news"), **mg.common_arrays(maps, starts, goals, res, cost=cost))

    # --- mazes_032 at g_ratio 0.8, random costs, eval with a gradient ------------------------------------------------
    maps, goals = load_split("mazes_032_moore_c8.npz", 100)
    maps, goals = maps[84:], goals[84:]
    starts = news_starts(maps.numpy(), mg.onehot_idx(goals), 6)
    rng = np.random.RandomState(23)
    cost = torch.from_numpy(rng.rand(16, 1, 32, 32).astype(np.float32))
    rand_G = torch.from_numpy(rng.randn(16, 1, 32, 32).astype(np.float32))
    res = run_news(cost, starts, goals, maps, g_ratio=0.8, grad_hist=rand_G)
    arrays = mg.common_arrays(maps, starts, goals, res, cost=cost)
    arrays.update(rand_G=rand_G[:, 0].numpy(), rand_grad_cost=res["grad_cost"][:, 0].numpy())
    mg.save("news_mazes032_gr08", dict(desc="16 mazes_032 test maps, random costs, NEWS, g_ratio 0.8 + grad",
                                       g_ratio=0.8, mechanism="news"), **arrays)


if __name__ == "__main__":
    if sys.argv[1:] == ["--more"]:   # only the files added after the first five
        more()
    else:
        main()
