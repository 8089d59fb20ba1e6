"""CPU tests of the NEWS (4-action) shortest-path labels: the C oracle's NEWS mode (oracle/labels_oracle.c) against the
generator's own dijkstra_dist and extract_policy and against a scipy graph search, 4-action dataset files, the dataset
tool's file names, and argument checks at the C ABI (no GPU needed)."""
import ctypes
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import labels_golden
from oracle import labels as label_oracle

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
EINVAL, EUNSUPPORTED = 1, 2
MECH_MOORE, MECH_NEWS = 0, 1


def _staged():
    return all(os.path.exists(os.path.join(label_oracle.REF_STAGE, f)) for f in label_oracle.REF_FILES)


needs_generator = pytest.mark.skipif(not _staged(), reason="the generator's dijkstra.py / mechanism.py are staged into "
                                                           "oracle/_ref by build() from a reference checkout")


@pytest.fixture(scope="module")
def built_lib():
    subprocess.check_call(["make", "-C", os.path.join(ROOT, "neural-astar_b200"), "-s", "all"])
    from neural_astar import _native

    return _native


def _random_maps(B, H, W, seed):
    """Bernoulli maps with goals; map 0 has non-binary values, map 1 a non-passable goal, map 2 a walled-in goal."""
    rs = np.random.RandomState(seed)
    maps = (rs.rand(B, H, W) >= 0.3).astype(np.float32)
    goal_idx = rs.randint(0, H * W, size=B).astype(np.int32)
    maps.reshape(B, -1)[np.arange(B), goal_idx] = 1.0
    maps[0] *= np.where(rs.rand(H, W) > 0.5, 0.25, -2.0).astype(np.float32)
    maps[1].reshape(-1)[goal_idx[1]] = 0.0
    gy, gx = divmod(int(goal_idx[2]), W)
    for y, x in ((gy - 1, gx), (gy + 1, gx), (gy, gx - 1), (gy, gx + 1)):
        if 0 <= y < H and 0 <= x < W:
            maps[2, y, x] = 0.0
    return maps, goal_idx


def _cases():
    """(maps, goal_idx) of every label fixture (the 64x64 ones cut to 40 maps: the generator's Python heap takes about
    0.08 s per map) and of random maps of several shapes."""
    for name in labels_golden.NAMES:
        maps, goal_idx, _, _ = labels_golden.load(name)
        yield name, maps[:40], goal_idx[:40]
    for H, W in ((1, 1), (1, 7), (5, 40), (12, 12), (33, 31)):
        yield f"random_{H}x{W}", *_random_maps(6, H, W, H * 100 + W)


@needs_generator
@pytest.mark.parametrize("case", [c[0] for c in _cases()])
def test_news_oracle_matches_the_generator(case):
    """Distances equal dijkstra_dist(maze, NorthEastWestSouth(), goal); masks equal extract_policy's maximal sets, whose
    lowest member is the action."""
    from labels_sweep import extract_policy_max_sets, generator_news_dists

    maps, goal_idx = next((m, g) for n, m, g in _cases() if n == case)
    d, mask, act = label_oracle.opt_labels(maps, goal_idx, mechanism="news")
    ref = generator_news_dists((maps, goal_idx, label_oracle.REF_STAGE))
    assert np.array_equal(d[:, 0], ref), f"distances differ on {int((d[:, 0] != ref).sum())} cells"
    for i in range(len(maps)):
        assert np.array_equal(mask[i, 0], extract_policy_max_sets(maps[i], ref[i], 4))
    assert (mask < 16).all() and (mask > 0).all()
    m, a = mask[:, 0].astype(np.int32), act[:, 0].astype(np.int32)
    assert ((m >> a) & 1).all() and ((m & ((1 << a) - 1)) == 0).all()


def _grid_bfs(maze, goal):
    """Unit-step distances to `goal` over 4-neighbours with scipy: a move v -> t exists when v is passable and t is
    passable or the goal (the goal is the source even when it is not passable).  Unreached: -(H*W)."""
    from scipy.sparse import coo_matrix
    from scipy.sparse.csgraph import shortest_path

    H, W = maze.shape
    N = H * W
    ok = (maze != 0).ravel()
    into = ok.copy()
    into[goal] = True
    src, dst = [], []
    idx = np.arange(N).reshape(H, W)
    for a, b in ((idx[:, :-1], idx[:, 1:]), (idx[:-1, :], idx[1:, :])):
        for u, v in ((a.ravel(), b.ravel()), (b.ravel(), a.ravel())):
            keep = ok[u] & into[v]
            src.append(v[keep])           # reversed edges: the search runs from the goal
            dst.append(u[keep])
    s, t = np.concatenate(src), np.concatenate(dst)
    g = coo_matrix((np.ones(len(s)), (s, t)), shape=(N, N)).tocsr()
    dist = shortest_path(g, unweighted=True, indices=goal)
    return np.where(np.isinf(dist), -N, -dist).reshape(H, W).astype(np.float32)


@pytest.mark.parametrize("H,W", [(1, 1), (2, 9), (5, 40), (24, 40), (64, 64)])
def test_news_oracle_matches_a_graph_search(H, W):
    """Without the generator's code: the NEWS distances equal scipy's breadth-first distances on the 4-neighbour move
    graph, and the masks equal the maximal sets of the restated extract_policy."""
    from labels_sweep import extract_policy_max_sets

    maps, goal_idx = _random_maps(8, H, W, 7 * H + W)
    d, mask, _ = label_oracle.opt_labels(maps, goal_idx, mechanism="news")
    for i in range(len(maps)):
        ref = _grid_bfs(maps[i], int(goal_idx[i]))
        assert np.array_equal(d[i, 0], ref)
        assert np.array_equal(mask[i, 0], extract_policy_max_sets(maps[i], ref, 4))
    walled = d[2, 0].ravel()
    assert walled[goal_idx[2]] == 0 and (np.delete(walled, goal_idx[2]) == -H * W).all()


def test_news_distances_are_4_connected():
    """On an open map the NEWS distance is the Manhattan distance, the Moore one the Chebyshev distance."""
    H, W, g = 9, 13, 4 * 13 + 5
    maps = np.ones((1, H, W), np.float32)
    y, x = np.mgrid[0:H, 0:W]
    news, _, _ = label_oracle.opt_labels(maps, [g], mechanism="news")
    moore, _, _ = label_oracle.opt_labels(maps, [g])
    assert np.array_equal(news[0, 0], -(np.abs(y - 4) + np.abs(x - 5)).astype(np.float32))
    assert np.array_equal(moore[0, 0], -np.maximum(np.abs(y - 4), np.abs(x - 5)).astype(np.float32))


def test_news_oracle_without_a_goal_and_with_an_obstacle_goal():
    """An index outside the grid reaches nothing; an obstacle goal is still the source of the search."""
    maps = np.ones((3, 4, 5), np.float32)
    maps[2, 1, 2] = 0.0
    d, mask, act = label_oracle.opt_labels(maps, [-1, 20, 7], mechanism="news")
    assert (d[0] == -20).all() and (d[1] == -20).all()
    assert d[2, 0, 1, 2] == 0 and d[2, 0, 0, 2] == -1 and d[2, 0, 0, 0] == -3
    assert (mask[:2] == 15).all() and (act[:2] == 0).all()     # all targets equal: every action is maximal


def test_four_action_dataset_rolls_out_in_maze_dataset(tmp_path):
    """A NEWS dataset file (policies [N,4,1,H,W]) saves, loads with num_actions 4, and MazeDataset's trajectories follow
    N/E/W/S moves to the goal in exactly -opt_dists[start] moves."""
    from neural_astar.utils.data import MazeDataset, save_planning_dataset

    maps, goal_idx, _, _ = labels_golden.load("mazes032_test")
    B, H, W = maps.shape
    goals = np.zeros((B, 1, H, W), np.float32)
    goals.reshape(B, -1)[np.arange(B), goal_idx] = 1
    d, _, act = label_oracle.opt_labels(maps, goal_idx, mechanism="news")
    pol = np.zeros((B, 4, 1, H, W), np.float32)
    np.put_along_axis(pol, act[:, None].astype(np.int64), 1.0, axis=1)
    split = (maps, goals, pol, d)
    path = str(tmp_path / "mazes_032_news_c8.npz")
    save_planning_dataset(path, split, split, split)
    ds = MazeDataset(path, "train")
    assert ds.num_actions == 4 and ds.opt_policies.shape == (B, 4, 1, H, W)
    np.random.seed(0)
    for i in range(B):
        _, start, _, traj = ds[i]
        assert traj[0].sum() == -d[i].ravel()[int(start[0].argmax())]
        ref = ds.get_opt_traj(start[0][None], goals[i], pol[i])       # the reference's own roll-out
        assert np.array_equal(ref[0], traj[0])
    with pytest.raises(ValueError):
        save_planning_dataset(str(tmp_path / "x.npz"), split, (maps, goals, np.zeros((B, 5, 1, H, W)), d), split)


def test_tool_names_news_files_and_rejects_other_mechanisms():
    import argparse

    import make_planning_dataset as mpd

    assert mpd.output_name("data/mpd/original/mazes/", 32, 1, 8, "news") == "mazes_032_news_c8.npz"
    assert mpd.output_name("data/mpd/original/*", 32, 2, 16, "news") == "all_064_news_c16.npz"
    assert mpd.output_name("data/mpd/original/mazes", 32, 1, 8) == "mazes_032_moore_c8.npz"
    args = argparse.Namespace(input_path="x", output_path="y", maze_size=32, mechanism="hex", edge_ratio=0.0,
                              train_size=1, valid_size=1, test_size=1, seed=0, tile_size=1)
    with pytest.raises(SystemExit, match="news, moore"):
        mpd.make(args)


def test_opt_labels_mech_rejects_bad_arguments_without_a_launch(built_lib):
    from neural_astar.utils.data import compute_opt_labels

    L = built_lib.lib()
    p = ctypes.c_void_p(16)          # never dereferenced: every call below fails validation before any launch
    before = L.nastar_b200_launch_count()
    f = L.nastar_b200_opt_labels_mech
    assert f(None, 64, p, 1, 8, 8, MECH_NEWS, p, p, p, None) == EINVAL
    assert f(p, 64, None, 1, 8, 8, MECH_NEWS, p, p, p, None) == EINVAL
    assert f(p, 64, p, 1, 8, 8, MECH_NEWS, None, p, p, None) == EINVAL
    assert f(p, 64, p, 1, 8, 8, MECH_NEWS, p, None, p, None) == EINVAL
    assert f(p, 64, p, 1, 8, 8, MECH_NEWS, p, p, None, None) == EINVAL
    assert f(p, 64, p, 0, 8, 8, MECH_NEWS, p, p, p, None) == EINVAL
    assert f(p, 64, p, 1, 0, 8, MECH_NEWS, p, p, p, None) == EINVAL
    assert f(p, 64, p, 1, 8, -1, MECH_NEWS, p, p, p, None) == EINVAL
    assert f(p, 63, p, 1, 8, 8, MECH_NEWS, p, p, p, None) == EINVAL            # map stride < H*W
    for mech in (-1, 2, 8):
        assert f(p, 64, p, 1, 8, 8, mech, p, p, p, None) == EINVAL
    assert f(p, 513 * 8, p, 1, 513, 8, MECH_NEWS, p, p, p, None) == EUNSUPPORTED
    assert f(p, 8 * 600, p, 1, 8, 600, MECH_MOORE, p, p, p, None) == EUNSUPPORTED
    assert f(p, 513 * 8, p, 1, 513, 8, 5, p, p, p, None) == EINVAL              # argument errors come first
    assert L.nastar_b200_launch_count() == before, "a rejected call launched something"
    maps = torch.ones(2, 1, 8, 8)
    with pytest.raises(ValueError, match="mechanism"):
        built_lib.opt_labels(maps, torch.zeros(2, dtype=torch.int32), "hex")
    with pytest.raises(RuntimeError, match="CUDA"):
        built_lib.opt_labels(maps, torch.zeros(2, dtype=torch.int32), "news")
    with pytest.raises(RuntimeError, match="CUDA"):
        compute_opt_labels(maps, torch.zeros(2, 1, 8, 8), "news")
