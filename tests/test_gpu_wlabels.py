"""GPU tests of the vertex-weighted shortest-path kernel (nastar_wlabels.cuh): bit-exact against the CPU oracle on the
label fixtures, on mazes_032 with the shipped checkpoint's costs and on seeded random cost maps; the unit-cost
reduction; planner paths against the optimum; determinism and launch count; dataset round trips."""
import os
import random
import sys

import numpy as np
import pytest
import torch

import labels_golden
from golden_util import Golden

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

pytestmark = pytest.mark.gpu

KEYS = ("dists", "hops", "act_mask", "action", "path_maps", "path_costs", "status")


@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    return torch.device("cuda:0")


def _cu(x, dev):
    return torch.from_numpy(np.ascontiguousarray(x)).to(dev)


def _kernel(cost, goal_idx, dev, passable=None, start_idx=None):
    from neural_astar import _native

    out = _native.weighted_labels(_cu(np.asarray(cost, np.float32), dev), _cu(np.asarray(goal_idx, np.int32), dev),
                                  None if passable is None else _cu(np.asarray(passable, np.float32), dev),
                                  None if start_idx is None else _cu(np.asarray(start_idx, np.int32), dev))
    torch.cuda.synchronize()
    return {k: None if v is None else v.cpu().numpy() for k, v in zip(KEYS, out)}


def _assert_matches_oracle(cost, goal_idx, dev, passable=None, start_idx=None):
    from oracle import wlabels

    k = _kernel(cost, goal_idx, dev, passable, start_idx)
    o = wlabels.weighted_labels(cost, goal_idx, passable, start_idx)
    for key in KEYS:
        if key not in o:
            assert k[key] is None
            continue
        a, b = k[key], o[key]
        assert a.shape == b.shape and a.dtype == b.dtype, key
        assert np.array_equal(a.view(np.uint8), b.view(np.uint8)), \
            f"{key} differs from the oracle on {int((a != b).sum())} entries"
    return k


def _reachable_starts(k, rs):
    B = k["hops"].shape[0]
    h = k["hops"].reshape(B, -1)
    starts = np.zeros(B, np.int32)
    for b in range(B):
        cand = np.flatnonzero(h[b] >= 0)
        starts[b] = cand[rs.randint(len(cand))] if len(cand) else 0
    return starts


def test_kernel_matches_oracle_on_label_fixtures(dev):
    """Unit costs on the shortest-path label fixtures (cost = passable = map), with reachable starts."""
    rs = np.random.RandomState(0)
    for name in labels_golden.NAMES:
        maps, goal_idx, _, _ = labels_golden.load(name)
        B, H, W = maps.shape
        if H > 128 or W > 128:
            continue
        cost = (maps != 0).astype(np.float32)
        k = _assert_matches_oracle(cost, goal_idx, dev, maps)
        _assert_matches_oracle(cost, goal_idx, dev, maps, _reachable_starts(k, rs))


def _ckpt_costs(dev):
    """mazes_032 (all 1000 problems) with the cost maps of the shipped checkpoint's encoder"""
    from neural_astar.planner import NeuralAstar

    state = np.load(os.path.join(ROOT, "tests", "golden", "mazes032_ckpt_planner_state.npz"))
    na = NeuralAstar(encoder_arch="CNN")
    na.load_state_dict({k: torch.from_numpy(state[k]) for k in state.files})
    na = na.to(dev).eval()
    g = Golden("inputs_mazes032_all1000")
    maps, start, goal = (_cu(x, dev) for x in (g.obst, g.start, g.goal))
    with torch.no_grad():
        cost = torch.cat([na.encode(maps[i:i + 100], start[i:i + 100], goal[i:i + 100]) for i in range(0, 1000, 100)])
    return na, g, maps, start, goal, cost


def test_learned_costs_match_oracle_and_bound_neural_astar(dev):
    from neural_astar.utils.data import shortest_path_maps
    from neural_astar.utils.training import path_cost_metrics

    na, g, maps, start, goal, cost = _ckpt_costs(dev)
    c = cost.cpu().numpy()
    _assert_matches_oracle(c, g.z["goal_idx"], dev, g.obst, g.z["start_idx"])
    paths, pcost = shortest_path_maps(cost, start, goal, passable=maps)
    assert torch.isfinite(pcost).all()
    # the optimal masks are optimal under the metric
    p_opt, ratio = path_cost_metrics(paths, cost, pcost)
    assert p_opt == 1.0 and abs(ratio - 1.0) < 1e-5
    # every Neural A* path that reaches its start costs at least the optimum (fp64 sum vs fp32 fold: N * 2^-24)
    with torch.no_grad():
        out = torch.cat([na.perform_astar(cost[i:i + 100], start[i:i + 100], goal[i:i + 100], maps[i:i + 100]).paths
                         for i in range(0, 1000, 100)]).float()
    complete = (out * start).sum((1, 2, 3)) > 0
    na_cost = torch.where(out != 0, cost.double(), 0.0).sum((1, 2, 3))
    assert complete.sum() > 900
    assert (na_cost[complete] >= pcost.double()[complete] * (1 - 32 * 32 * 2.0 ** -24)).all()
    p_na, ratio_na = path_cost_metrics(out[complete], cost[complete], pcost[complete])
    print(f"Neural A* on mazes_032 (checkpoint costs): p_opt {p_na:.3f}, mean cost ratio {ratio_na:.4f}")
    assert ratio_na >= 1.0 - 1e-5


def _random_problem(B, H, W, seed):
    """Random costs with zero-cost and absorbed cells, obstacles and the edge cases of DESIGN.md §11."""
    rs = np.random.RandomState(seed)
    N = H * W
    cost = rs.uniform(0.01, 5.0, size=(B, H, W)).astype(np.float32)
    cost[rs.rand(B, H, W) < 0.1] = 0.0
    cost[rs.rand(B, H, W) < 0.05] = 1e-9
    cost[rs.rand(B, H, W) < 0.05] = 1e4
    passable = (rs.rand(B, H, W) >= 0.2).astype(np.float32)
    goal = rs.randint(0, N, size=B).astype(np.int32)
    start = rs.randint(0, N, size=B).astype(np.int32)
    passable.reshape(B, -1)[np.arange(B), goal] = 1.0
    passable.reshape(B, -1)[np.arange(B), start] = 1.0
    passable.reshape(B, -1)[0, goal[0]] = 0.0           # a goal that is not passable is still the source
    gy, gx = divmod(int(goal[1]), W)                    # map 1: every neighbour of the goal blocked
    passable[1, max(gy - 1, 0):gy + 2, max(gx - 1, 0):gx + 2] = 0.0
    passable[1, gy, gx] = 1.0
    if start[1] == goal[1]:
        start[1] = (goal[1] + 2 * W) % N
    passable[2].fill(1.0)                               # map 2: an unreachable start, walled in
    sy, sx = divmod(int(start[2]), W)
    passable[2, max(sy - 1, 0):sy + 2, max(sx - 1, 0):sx + 2] = 0.0
    passable[2, sy, sx] = 1.0
    goal[2] = (start[2] + 2 * W + 2) % N if H > 3 else (start[2] + 3) % N
    passable.reshape(B, -1)[2, goal[2]] = 1.0
    start[3] = goal[3]                                  # start == goal
    cost[4] = 0.0                                       # map 4: every cost zero
    cost[5] = np.float32(1e-9)                          # map 5: absorbed costs beside a huge goal cost
    cost[5].reshape(-1)[goal[5]] = 1e4
    cost[6].reshape(-1)[rs.randint(N)] = -1.0           # map 6: a negative cost on a passable cell
    passable[6].fill(1.0)
    goal[7] = N + 5                                     # map 7: no goal
    return cost, passable, goal, start


@pytest.mark.parametrize("H,W", [(12, 12), (5, 40), (33, 31), (64, 64), (100, 72), (128, 128)])
def test_kernel_matches_oracle_on_random_costs(dev, H, W):
    B = 24
    cost, passable, goal, start = _random_problem(B, H, W, seed=H * 1000 + W)
    k = _assert_matches_oracle(cost, goal, dev, passable, start)
    _assert_matches_oracle(cost, goal, dev, passable)                 # without starts
    _assert_matches_oracle(cost, goal, dev, None, start)              # every cell passable
    st = k["status"]
    assert st[3] == 0 and (st[[0, 4, 5]] & ~4 == 0).all()    # valid maps (their random starts may be cut off)
    assert st[1] & 4 and st[2] & 4 and st[6] == 1 | 4 and st[7] == 2 | 4
    assert k["path_costs"][3] == cost[3].reshape(-1)[goal[3]] and k["path_maps"][3].sum() == 1
    assert k["path_maps"][2].sum() == 0 and np.isinf(k["path_costs"][2])
    hs = k["hops"].reshape(B, -1)[np.arange(B), start]
    ok = st == 0
    assert np.array_equal(k["path_maps"].reshape(B, -1).sum(1)[ok], hs[ok] + 1.0)


def test_unit_reduction_equals_compute_opt_labels(dev):
    from neural_astar.utils.data import compute_opt_labels, compute_weighted_opt_labels

    maps, goal_idx, _, _ = labels_golden.load("mazes032_test")
    B, H, W = maps.shape
    keep = maps.reshape(B, -1)[np.arange(B), goal_idx] != 0
    maps, goal_idx = maps[keep], goal_idx[keep]
    B = maps.shape[0]
    goals = np.zeros((B, 1, H, W), np.float32)
    goals.reshape(B, -1)[np.arange(B), goal_idx] = 1
    md, gm = _cu(maps[:, None], dev), _cu(goals, dev)
    upol, ud, um = compute_opt_labels(md, gm)
    wpol, wd, wm, hops = compute_weighted_opt_labels((md != 0).float(), gm, passable=md)
    reach = torch.isfinite(wd)
    assert torch.equal(reach, ud > -H * W)
    assert torch.equal(wd[reach], ud[reach]) and torch.equal(hops[reach].float(), -ud[reach])
    nongoal = reach & (gm == 0)
    assert torch.equal(wm[nongoal], um[nongoal])
    assert torch.equal(wpol[nongoal.unsqueeze(1).expand_as(wpol)], upol[nongoal.unsqueeze(1).expand_as(upol)])
    assert (wpol.sum(1)[~nongoal] == 0).all()


def test_vanilla_astar_paths_have_path_len_cells(dev):
    from neural_astar.planner import VanillaAstar
    from neural_astar.utils.data import compute_weighted_opt_labels, sample_goal_maps, shortest_path_maps

    B, H, W = 32, 32, 32
    rs = np.random.RandomState(5)
    maps = (rs.rand(B, 1, H, W) > 0.3).astype(np.float32)
    goals = sample_goal_maps(maps, rng=random.Random(5))
    md, gm = _cu(maps, dev), _cu(goals, dev)
    _, _, _, hops = compute_weighted_opt_labels(md, gm, passable=md)
    hn = hops.cpu().numpy().reshape(B, -1)
    starts = np.zeros_like(goals)
    for b in range(B):
        cand = np.flatnonzero(hn[b] > 0)
        starts.reshape(B, -1)[b, cand[rs.randint(len(cand))]] = 1
    sm = _cu(starts, dev)
    paths, pcost = shortest_path_maps(md, sm, gm, passable=md)
    want = paths.sum((1, 2, 3))
    assert torch.equal(want, pcost)                     # unit costs: the path cost counts its cells
    out = VanillaAstar().to(dev).eval()(md, sm, gm)
    assert torch.equal(out.paths.sum((1, 2, 3)).float(), want)


def test_deterministic_and_one_launch(dev):
    from neural_astar import _native

    cost, passable, goal, start = _random_problem(64, 64, 64, seed=11)
    args = (_cu(cost, dev), _cu(goal, dev), _cu(passable, dev), _cu(start, dev))
    a = _native.weighted_labels(*args)
    torch.cuda.synchronize()
    before = _native.launch_count()
    b = _native.weighted_labels(*args)
    torch.cuda.synchronize()
    assert _native.launch_count() - before == 1
    for x, y in zip(a, b):
        assert torch.equal(x.view(torch.uint8), y.view(torch.uint8))


def test_shape_above_the_limit_raises(dev):
    from neural_astar.utils.data import compute_weighted_opt_labels

    with pytest.raises(ValueError):
        compute_weighted_opt_labels(torch.ones(1, 1, 129, 8, device=dev), torch.zeros(1, 1, 129, 8, device=dev))
    bad = torch.ones(2, 1, 8, 8, device=dev)
    bad[1, 0, 3, 3] = float("nan")
    with pytest.raises(ValueError, match=r"\[1\]"):
        compute_weighted_opt_labels(bad, torch.zeros(2, 1, 8, 8, device=dev))


def test_warcraft_round_trip(dev, tmp_path):
    from neural_astar.utils.data import WarCraftDataset, save_warcraft_dataset, shortest_path_maps

    B, H, W = 16, 12, 12
    rs = np.random.RandomState(2)
    images = rs.rand(B, 3, 96, 96).astype(np.float32)
    cost = _cu(rs.uniform(0.5, 9.0, size=(B, 1, H, W)).astype(np.float32), dev)
    start = torch.zeros(B, 1, H, W, device=dev)
    goal = torch.zeros(B, 1, H, W, device=dev)
    start[:, :, 0, 0] = 1
    goal[:, :, -1, -1] = 1
    paths, _ = shortest_path_maps(cost, start, goal)
    save_warcraft_dataset(str(tmp_path), "train", images, paths)
    ds = WarCraftDataset(str(tmp_path), "train")
    assert len(ds) == B
    for i in range(B):
        img, s, g, traj = ds[i]
        assert np.array_equal(img, (np.rint(images[i] * 255).astype(np.uint8) / 255.0).astype(np.float32))
        assert np.array_equal(traj, paths[i].cpu().numpy())
        assert traj[0, 0, 0] == 1 and traj[0, -1, -1] == 1


def test_weighted_planning_dataset_round_trip(dev, tmp_path):
    """A weighted dataset written with save_planning_dataset loads in MazeDataset, and its expert trajectories are the
    shortest_path_maps paths for the same starts, goal excluded."""
    from neural_astar.utils.data import (MazeDataset, compute_weighted_opt_labels, sample_goal_maps,
                                         save_planning_dataset, shortest_path_maps)

    B, H, W = 24, 32, 32
    rs = np.random.RandomState(9)
    maps = (rs.rand(B, 1, H, W) > 0.25).astype(np.float32)
    goals = sample_goal_maps(maps, rng=random.Random(9))
    cost = _cu(rs.uniform(0.1, 4.0, size=(B, 1, H, W)).astype(np.float32), dev)
    md, gm = _cu(maps, dev), _cu(goals, dev)
    pol, dists, _, _ = compute_weighted_opt_labels(cost, gm, passable=md)
    split = (maps[:, 0], goals, pol, dists)
    path = str(tmp_path / "weighted.npz")
    save_planning_dataset(path, split, split, split)
    ds = MazeDataset(path, "test")
    np.random.seed(0)
    for i in range(B):
        m, s, g, traj = ds[i]
        assert np.array_equal(m[0], maps[i, 0]) and np.array_equal(g, goals[i])
        p, _ = shortest_path_maps(cost[i:i + 1], _cu(s[None], dev), gm[i:i + 1], passable=md[i:i + 1])
        want = p[0].cpu().numpy() * (1 - goals[i])
        assert np.array_equal(traj, want)
