"""GPU tests of the NEWS (4-connected) vertex-weighted shortest-path kernel (nastar_wlabels.cuh, kNews): bit-exact
against the C oracle's NEWS mode (oracle/wlabels_oracle.c) on the label fixtures, on the NEWS goldens' learned costs
and on seeded random cost maps; the Moore case of the new entry point against the old one; NEWS planner paths against
the NEWS optimum; determinism, launch count and dataset round trips."""
import ctypes
import os
import random
import sys

import numpy as np
import pytest
import torch

import labels_golden
from golden_util import Golden
from oracle import wlabels

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

pytestmark = pytest.mark.gpu

KEYS = ("dists", "hops", "act_mask", "action", "path_maps", "path_costs", "status")
NEWS_STEPS = {(-1, 0), (1, 0), (0, -1), (0, 1)}


@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    return torch.device("cuda:0")


def _cu(x, dev):
    return torch.from_numpy(np.ascontiguousarray(x)).to(dev)


def _kernel(cost, goal_idx, dev, passable=None, start_idx=None, mechanism="news"):
    from neural_astar import _native

    out = _native.weighted_labels(_cu(np.asarray(cost, np.float32), dev), _cu(np.asarray(goal_idx, np.int32), dev),
                                  None if passable is None else _cu(np.asarray(passable, np.float32), dev),
                                  None if start_idx is None else _cu(np.asarray(start_idx, np.int32), dev),
                                  mechanism)
    torch.cuda.synchronize()
    return {k: None if v is None else v.cpu().numpy() for k, v in zip(KEYS, out)}


def _assert_matches_oracle(cost, goal_idx, dev, passable=None, start_idx=None):
    k = _kernel(cost, goal_idx, dev, passable, start_idx)
    o = wlabels.weighted_labels(cost, goal_idx, passable, start_idx, mechanism="news")
    for key in KEYS:
        if key not in o:
            assert k[key] is None
            continue
        a, b = k[key], o[key]
        assert a.shape == b.shape and a.dtype == b.dtype, key
        assert np.array_equal(a.view(np.uint8), b.view(np.uint8)), \
            f"{key} differs from the NEWS oracle on {int((a != b).sum())} entries"
    assert k["act_mask"].max() < 16
    return k


def _reachable_starts(k, rs):
    B = k["hops"].shape[0]
    h = k["hops"].reshape(B, -1)
    starts = np.zeros(B, np.int32)
    for b in range(B):
        cand = np.flatnonzero(h[b] >= 0)
        starts[b] = cand[rs.randint(len(cand))] if len(cand) else 0
    return starts


def test_news_kernel_matches_oracle_on_label_fixtures(dev):
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


@pytest.mark.parametrize("name", ["news/news_mazes032_neural", "news/news_large128_learned"])
def test_news_kernel_matches_oracle_on_learned_costs(dev, name):
    """The shipped checkpoint's costs of the NEWS search goldens, map passability, their starts and goals."""
    g = Golden(name)
    k = _assert_matches_oracle(g.cost, g.z["goal_idx"], dev, g.obst, g.z["start_idx"])
    assert (k["status"] == 0).all()
    _assert_matches_oracle(g.cost, g.z["goal_idx"], dev, g.obst)


def _random_problem(B, H, W, seed):
    """Random costs with zero-cost, absorbed and 1e4 cells, obstacles and the edge cases of DESIGN.md §11, walled
    4-connected (the diagonal neighbours of a walled cell stay open)."""
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
    if N < 25:
        return cost, passable, goal, start

    def wall(b, idx):
        y, x = divmod(int(idx), W)
        for dy, dx in NEWS_STEPS:
            if 0 <= y + dy < H and 0 <= x + dx < W:
                passable[b, y + dy, x + dx] = 0.0

    passable.reshape(B, -1)[0, goal[0]] = 0.0           # a goal that is not passable is still the source
    wall(1, goal[1])                                    # map 1: the goal's 4 neighbours blocked
    if abs(int(start[1]) - int(goal[1])) <= W + 1:
        start[1] = (goal[1] + 2 * W) % N
    passable.reshape(B, -1)[1, start[1]] = 1.0
    passable[2].fill(1.0)                               # map 2: an unreachable start, walled in
    wall(2, start[2])
    goal[2] = (start[2] + 2 * W + 2) % N
    passable.reshape(B, -1)[2, goal[2]] = 1.0
    start[3] = goal[3]                                  # start == goal
    cost[4] = 0.0                                       # map 4: every cost zero
    cost[5] = np.float32(1e-9)                          # map 5: absorbed costs beside a huge goal cost
    cost[5].reshape(-1)[goal[5]] = 1e4
    cost[6].reshape(-1)[rs.randint(N)] = -1.0           # map 6: a negative cost on a passable cell
    passable[6].fill(1.0)
    goal[7] = N + 5                                     # map 7: no goal
    return cost, passable, goal, start


@pytest.mark.parametrize("H,W", [(1, 1), (12, 12), (5, 40), (33, 31), (64, 64), (100, 72), (128, 128)])
def test_news_kernel_matches_oracle_on_random_costs(dev, H, W):
    B = 24
    cost, passable, goal, start = _random_problem(B, H, W, seed=H * 1000 + W + 7)
    k = _assert_matches_oracle(cost, goal, dev, passable, start)
    _assert_matches_oracle(cost, goal, dev, passable)                 # without starts
    _assert_matches_oracle(cost, goal, dev, None, start)              # every cell passable
    st = k["status"]
    if H * W < 25:
        assert (st == 0).all() and (k["path_maps"].reshape(B, -1).sum(1) == 1).all()
        return
    assert st[3] == 0 and (st[[0, 4, 5]] & ~4 == 0).all()
    assert st[1] & 4 and st[2] & 4 and st[6] == 1 | 4 and st[7] == 2 | 4
    assert k["path_costs"][3] == cost[3].reshape(-1)[goal[3]] and k["path_maps"][3].sum() == 1
    assert k["path_maps"][2].sum() == 0 and np.isinf(k["path_costs"][2])
    hs = k["hops"].reshape(B, -1)[np.arange(B), start]
    ok = st == 0
    assert ok.sum() >= 8
    assert np.array_equal(k["path_maps"].reshape(B, -1).sum(1)[ok], hs[ok] + 1.0)


def test_moore_mech_equals_the_old_entry_point(dev):
    """nastar_b200_weighted_labels_mech(NASTAR_MECH_MOORE) and nastar_b200_weighted_labels give the same bits."""
    from neural_astar import _native

    cost, passable, goal, start = _random_problem(24, 100, 72, seed=21)
    c, p, g, s = _cu(cost, dev), _cu(passable, dev), _cu(goal, dev), _cu(start, dev)
    new = _native.weighted_labels(c, g, p, s, mechanism="moore")
    old = [torch.empty_like(x) for x in new]
    L = _native.lib()
    with torch.cuda.device(dev):
        stream = ctypes.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
        rc = L.nastar_b200_weighted_labels(c.data_ptr(), 100 * 72, p.data_ptr(), 100 * 72, g.data_ptr(),
                                           s.data_ptr(), 24, 100, 72, *(x.data_ptr() for x in old), stream)
    assert rc == 0
    torch.cuda.synchronize()
    for x, y in zip(new, old):
        assert torch.equal(x.view(torch.uint8), y.view(torch.uint8))
    news = _native.weighted_labels(c, g, p, s, mechanism="news")
    assert not torch.equal(news[0], new[0])             # the mechanism reaches the kernel


def test_news_deterministic_and_one_launch(dev):
    from neural_astar import _native

    cost, passable, goal, start = _random_problem(64, 64, 64, seed=11)
    args = (_cu(cost, dev), _cu(goal, dev), _cu(passable, dev), _cu(start, dev))
    a = _native.weighted_labels(*args, mechanism="news")
    torch.cuda.synchronize()
    before = _native.launch_count()
    b = _native.weighted_labels(*args, mechanism="news")
    torch.cuda.synchronize()
    assert _native.launch_count() - before == 1
    for x, y in zip(a, b):
        assert torch.equal(x.view(torch.uint8), y.view(torch.uint8))


def test_news_compute_weighted_opt_labels_has_four_actions(dev):
    from neural_astar.utils.data import compute_weighted_opt_labels

    cost, passable, goal, _ = _random_problem(24, 33, 31, seed=4)
    ok = [0, 1, 2, 3, 4, 5]                                           # maps without bad costs or a missing goal
    cost, passable, goal = cost[ok], passable[ok], goal[ok]
    B, H, W = cost.shape
    gm = np.zeros((B, 1, H, W), np.float32)
    gm.reshape(B, -1)[np.arange(B), goal] = 1
    pol, dists, mask, hops = compute_weighted_opt_labels(_cu(cost[:, None], dev), _cu(gm, dev),
                                                         passable=_cu(passable[:, None], dev), mechanism="news")
    assert pol.shape == (B, 4, 1, H, W) and pol.dtype == torch.float32
    k = _kernel(cost, goal, dev, passable)
    assert np.array_equal(dists.cpu().numpy(), k["dists"]) and np.array_equal(hops.cpu().numpy(), k["hops"])
    assert np.array_equal(mask.cpu().numpy(), k["act_mask"])
    act = k["action"][:, 0]
    p = pol.cpu().numpy()[:, :, 0]
    assert np.array_equal(p.sum(1), (act >= 0).astype(np.float32))
    assert np.array_equal(p.argmax(1)[act >= 0], act[act >= 0])
    with pytest.raises(ValueError, match="mechanism"):
        compute_weighted_opt_labels(_cu(cost[:, None], dev), _cu(gm, dev), mechanism="hex")


def test_news_planner_paths_cost_at_least_the_news_optimum(dev):
    """The NEWS Neural A* paths of the mazes_032 golden (the shipped checkpoint's costs) never cost less than the NEWS
    optimum, within path_cost_metrics' rtol; the Moore optimum never exceeds the NEWS one."""
    from neural_astar.utils.data import shortest_path_maps
    from neural_astar.utils.training import path_cost_metrics

    g = Golden("news/news_mazes032_neural")
    cost, maps, start, goal = (_cu(x, dev) for x in (g.cost, g.obst, g.start, g.goal))
    paths, news_opt = shortest_path_maps(cost, start, goal, passable=maps, mechanism="news")
    _, moore_opt = shortest_path_maps(cost, start, goal, passable=maps)
    assert torch.isfinite(news_opt).all() and torch.isfinite(moore_opt).all()
    p_opt, ratio = path_cost_metrics(paths, cost, news_opt)
    assert p_opt == 1.0 and abs(ratio - 1.0) < 1e-5
    na_paths = _cu(g.bits("path_bits").astype(np.float32), dev)
    assert ((na_paths * start).sum((1, 2, 3)) == 1).all() and ((na_paths * goal).sum((1, 2, 3)) == 1).all()
    na_cost = torch.where(na_paths != 0, cost.double(), 0.0).sum((1, 2, 3))
    assert (na_cost >= news_opt.double() * (1 - 1e-5)).all()
    p_na, ratio_na = path_cost_metrics(na_paths, cost, news_opt)
    p_moore, ratio_moore = path_cost_metrics(na_paths, cost, moore_opt)
    assert ratio_na >= 1.0 - 1e-5 and ratio_moore >= ratio_na
    assert (moore_opt <= news_opt).all()
    lower = int((moore_opt < news_opt).sum())
    print(f"NEWS Neural A* on news_mazes032_neural: against the NEWS optimum p_opt {p_na:.3f}, cost ratio "
          f"{ratio_na:.4f}; against the Moore optimum p_opt {p_moore:.3f}, cost ratio {ratio_moore:.4f}; "
          f"Moore optimum strictly lower on {lower}/{g.B} maps")


def test_news_vanilla_astar_paths_have_hop_plus_one_cells(dev):
    from neural_astar.planner import VanillaAstar
    from neural_astar.utils.data import compute_weighted_opt_labels, sample_goal_maps, shortest_path_maps

    B, H, W = 32, 32, 32
    rs = np.random.RandomState(15)
    maps = (rs.rand(B, 1, H, W) > 0.3).astype(np.float32)
    goals = sample_goal_maps(maps, rng=random.Random(15))
    md, gm = _cu(maps, dev), _cu(goals, dev)
    _, _, _, hops = compute_weighted_opt_labels(md, gm, passable=md, mechanism="news")
    hn = hops.cpu().numpy().reshape(B, -1)
    starts = np.zeros_like(goals)
    for b in range(B):
        cand = np.flatnonzero(hn[b] > 0)
        starts.reshape(B, -1)[b, cand[rs.randint(len(cand))]] = 1
    sm = _cu(starts, dev)
    paths, pcost = shortest_path_maps(md, sm, gm, passable=md, mechanism="news")
    want = paths.sum((1, 2, 3))
    assert torch.equal(want, pcost)                     # unit costs: the path cost counts its cells
    assert torch.equal(want.cpu(), torch.from_numpy(hn[np.arange(B), starts.reshape(B, -1).argmax(1)] + 1.0).float())
    with torch.no_grad():
        out = VanillaAstar(mechanism="news").to(dev).eval()(md, sm, gm)
    assert torch.equal(out.paths.sum((1, 2, 3)).float(), want)


def _four_connected(mask):
    ys, xs = np.nonzero(mask)
    cells = set(zip(ys.tolist(), xs.tolist()))
    return len(cells) == 1 or all(any((y + dy, x + dx) in cells for dy, dx in NEWS_STEPS) for y, x in cells)


def test_news_warcraft_round_trip(dev, tmp_path):
    from neural_astar.utils.data import WarCraftDataset, save_warcraft_dataset, shortest_path_maps

    B, H, W = 16, 12, 12
    rs = np.random.RandomState(12)
    images = rs.rand(B, 3, 96, 96).astype(np.float32)
    cost = _cu(rs.uniform(0.5, 9.0, size=(B, 1, H, W)).astype(np.float32), dev)
    start = torch.zeros(B, 1, H, W, device=dev)
    goal = torch.zeros(B, 1, H, W, device=dev)
    start[:, :, 0, 0] = 1
    goal[:, :, -1, -1] = 1
    paths, pcost = shortest_path_maps(cost, start, goal, mechanism="news")
    _, moore = shortest_path_maps(cost, start, goal)
    assert (moore <= pcost).all()
    save_warcraft_dataset(str(tmp_path), "train", images, paths)
    ds = WarCraftDataset(str(tmp_path), "train")
    assert len(ds) == B
    for i in range(B):
        img, s, g, traj = ds[i]
        assert np.array_equal(img, (np.rint(images[i] * 255).astype(np.uint8) / 255.0).astype(np.float32))
        assert np.array_equal(traj, paths[i].cpu().numpy())
        assert traj[0, 0, 0] == 1 and traj[0, -1, -1] == 1
        assert traj.sum() >= H + W - 1 and _four_connected(traj[0])    # no diagonal shortcut


def test_news_weighted_planning_dataset_round_trip(dev, tmp_path):
    """A NEWS weighted dataset (4-action policies) written with save_planning_dataset loads in MazeDataset, and its
    expert trajectories are the NEWS shortest_path_maps paths for the same starts, goal excluded."""
    from neural_astar.utils.data import (MazeDataset, compute_weighted_opt_labels, sample_goal_maps,
                                         save_planning_dataset, shortest_path_maps)

    B, H, W = 24, 32, 32
    rs = np.random.RandomState(19)
    maps = (rs.rand(B, 1, H, W) > 0.25).astype(np.float32)
    goals = sample_goal_maps(maps, rng=random.Random(19))
    cost = _cu(rs.uniform(0.1, 4.0, size=(B, 1, H, W)).astype(np.float32), dev)
    md, gm = _cu(maps, dev), _cu(goals, dev)
    pol, dists, _, _ = compute_weighted_opt_labels(cost, gm, passable=md, mechanism="news")
    assert pol.shape == (B, 4, 1, H, W)
    split = (maps[:, 0], goals, pol, dists)
    path = str(tmp_path / "weighted_news.npz")
    save_planning_dataset(path, split, split, split)
    ds = MazeDataset(path, "test")
    np.random.seed(0)
    for i in range(B):
        m, s, g, traj = ds[i]
        assert np.array_equal(m[0], maps[i, 0]) and np.array_equal(g, goals[i])
        p, _ = shortest_path_maps(cost[i:i + 1], _cu(s[None], dev), gm[i:i + 1], passable=md[i:i + 1],
                                  mechanism="news")
        full = p[0].cpu().numpy()
        assert _four_connected(full[0])
        assert np.array_equal(traj, full * (1 - goals[i]))
