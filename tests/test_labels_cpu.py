"""CPU tests of the shortest-path label generator: the oracle against the shipped datasets and the fixtures, goal
sampling, the dataset writer, and argument checks at the C ABI (no GPU needed)."""
import ctypes
import os
import random
import subprocess
import sys

import numpy as np
import pytest
import torch

import labels_golden

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
SHIPPED = "/root/reference/planning-datasets/data"


@pytest.fixture(scope="module")
def built_lib():
    subprocess.check_call(["make", "-C", os.path.join(ROOT, "neural-astar_b200"), "-s", "all"])
    from neural_astar import _native

    return _native


@pytest.mark.skipif(not os.path.isdir(SHIPPED), reason="needs the planning-datasets files of a reference checkout")
def test_oracle_matches_every_shipped_map():
    """All splits of all 10 shipped .npz files (16 000 maps): distances equal opt_dists exactly, and the shipped
    policy's action is a member of the oracle's maximal-action set on every cell."""
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    from labels_sweep import sweep

    t = sweep(SHIPPED)["total"]
    print(f"maps {t['maps']}: dist mismatches {t['dist_mismatch_cells']}, "
          f"policy actions outside the max set {t['policy_not_in_max_set_cells']}")
    assert t["maps"] == 16000
    assert t["dist_mismatch_cells"] == 0
    assert t["policy_not_in_max_set_cells"] == 0


@pytest.mark.parametrize("name", labels_golden.NAMES)
def test_oracle_reproduces_fixtures(name):
    from oracle import labels as label_oracle

    maps, goal_idx, dists, action = labels_golden.load(name)
    d, mask, act = label_oracle.opt_labels(maps, goal_idx)
    assert np.array_equal(d[:, 0], dists)
    assert ((mask[:, 0] >> action.astype(np.uint8)) & 1).all()     # the fixture's action is maximal
    m, a = mask[:, 0].astype(np.int32), act[:, 0].astype(np.int32)
    assert ((m >> a) & 1).all() and ((m & ((1 << a) - 1)) == 0).all()   # the action is the lowest set bit
    if name == "synthetic":
        assert np.array_equal(act[:, 0], action)
        H, W = maps.shape[1:]
        walled = d[8, 0].ravel()
        assert walled[goal_idx[8]] == 0 and (np.delete(walled, goal_idx[8]) == -H * W).all()


def _component_sizes(maze):
    from scipy import ndimage

    lab, n = ndimage.label(maze != 0)
    return lab, np.bincount(lab.ravel())[1:]


@pytest.mark.parametrize("edge", [0, 4])
def test_sample_goal_maps_draws_from_the_largest_region(edge):
    from neural_astar.utils.data import sample_goal_maps

    rs = np.random.RandomState(3)
    maps = (rs.rand(40, 1, 32, 32) > 0.45).astype(np.float32)
    maps[:5, 0, :8, :8] = 0
    maps[:5, 0, :8, -8:] = 0
    maps[:5, 0, -8:, :] = 0        # maps 0..4: no corner square touches any passable cell
    goals = sample_goal_maps(maps, edge_size=edge, rng=random.Random(11))
    assert goals.shape == maps.shape and goals.dtype == np.float32
    assert (goals.reshape(40, -1).sum(1) == 1).all()
    corner = np.zeros((32, 32), bool)
    if edge:
        for ys in (slice(0, edge), slice(-edge, None)):
            for xs in (slice(0, edge), slice(-edge, None)):
                corner[ys, xs] = True
    n_corner = 0
    for i in range(40):
        lab, sizes = _component_sizes(maps[i, 0])
        gy, gx = np.unravel_index(goals[i, 0].argmax(), (32, 32))
        assert lab[gy, gx] != 0 and sizes[lab[gy, gx] - 1] == sizes.max()
        big = lab == (np.argmax(sizes) + 1)
        if edge and (big & corner).any():
            assert corner[gy, gx]
            n_corner += 1
    if edge:
        assert n_corner >= 20      # most of the 35 maps with open corners
    # same seed, same goals; one rng.choice per map
    again = sample_goal_maps(torch.from_numpy(maps), edge_size=edge, rng=random.Random(11))
    assert np.array_equal(goals, again)


def test_sample_goal_maps_ties_go_to_the_first_region():
    from neural_astar.utils.data import sample_goal_maps

    m = np.zeros((1, 9, 9), np.float32)
    m[0, 0:2, 0:2] = 1      # first region in raster order, 4 cells
    m[0, 6:8, 6:8] = 1      # same size
    for seed in range(8):
        g = sample_goal_maps(m, rng=random.Random(seed))[0, 0]
        assert g[0:2, 0:2].sum() == 1


def test_saved_dataset_round_trips_through_the_dataloader(tmp_path):
    """save_planning_dataset -> MazeDataset / create_dataloader: same maps and goals, starts drawn from the 55-100 %
    distance bands, and the trajectory follows the saved policy to the goal."""
    from oracle import labels as label_oracle

    from neural_astar.utils.data import MazeDataset, create_dataloader, sample_goal_maps, save_planning_dataset

    maps, *_ = labels_golden.load("mazes032_test")
    goals = sample_goal_maps(maps, rng=random.Random(5))
    B, H, W = maps.shape
    d, _, act = label_oracle.opt_labels(maps, goals.reshape(B, -1).argmax(1))
    pol = np.zeros((B, 8, 1, H, W), np.float32)
    np.put_along_axis(pol, act[:, None].astype(np.int64), 1.0, axis=1)
    split = (maps, goals, pol, d)
    path = str(tmp_path / "new_032_moore.npz")
    save_planning_dataset(path, split, (maps[:10], goals[:10], pol[:10], d[:10]), (maps[:20], goals[:20], pol[:20], d[:20]))
    ds = MazeDataset(path, "train")
    assert np.array_equal(ds.map_designs, maps) and np.array_equal(ds.goal_maps, goals)
    assert len(MazeDataset(path, "valid")) == 10 and len(MazeDataset(path, "test")) == 20
    np.random.seed(0)
    for i in range(B):
        md, start, goal, traj = ds[i]
        od = d[i].ravel()
        th = np.percentile(od[od > od.min()], 100.0 * (1 - np.array([0.55, 0.70, 0.85, 1.0])))
        s = int(start[0].argmax())
        assert th[3] <= od[s] <= th[0]
        assert traj[0].sum() == -od[s]              # one cell per move, start included, goal excluded
    batch = next(iter(create_dataloader(path, "test", batch_size=20)))
    assert batch[0].shape == (20, 1, H, W) and torch.equal(batch[2], torch.from_numpy(goals[:20]))


def test_save_planning_dataset_checks_shapes(tmp_path):
    from neural_astar.utils.data import save_planning_dataset

    m = np.ones((2, 8, 8), np.float32)
    good = (m, np.zeros((2, 1, 8, 8)), np.zeros((2, 8, 1, 8, 8)), np.zeros((2, 1, 8, 8)))
    bad = (m, np.zeros((2, 8, 8)), np.zeros((2, 8, 1, 8, 8)), np.zeros((2, 1, 8, 8)))
    with pytest.raises(ValueError):
        save_planning_dataset(str(tmp_path / "x.npz"), good, bad, good)


def test_opt_labels_rejects_bad_arguments_without_a_gpu(built_lib):
    from neural_astar.utils.data import compute_opt_labels

    L = built_lib.lib()
    p = ctypes.c_void_p(16)          # never dereferenced: every call below fails validation before any launch
    assert L.nastar_b200_opt_labels(None, 64, p, 1, 8, 8, p, p, p, None) == 1
    assert L.nastar_b200_opt_labels(p, 64, None, 1, 8, 8, p, p, p, None) == 1
    assert L.nastar_b200_opt_labels(p, 64, p, 1, 8, 8, p, p, None, None) == 1
    assert L.nastar_b200_opt_labels(p, 64, p, 0, 8, 8, p, p, p, None) == 1
    assert L.nastar_b200_opt_labels(p, 63, p, 1, 8, 8, p, p, p, None) == 1        # map stride < H*W
    assert L.nastar_b200_opt_labels(p, 513 * 8, p, 1, 513, 8, p, p, p, None) == 2  # NASTAR_EUNSUPPORTED
    assert L.nastar_b200_opt_labels(p, 8 * 600, p, 1, 8, 600, p, p, p, None) == 2
    maps = torch.ones(2, 1, 8, 8)
    goals = torch.zeros(2, 1, 8, 8)
    with pytest.raises(RuntimeError, match="CUDA"):
        built_lib.opt_labels(maps, torch.zeros(2, dtype=torch.int32))
    with pytest.raises(RuntimeError, match="CUDA"):
        compute_opt_labels(maps, goals)
