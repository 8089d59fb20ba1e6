"""GPU tests of the shortest-path label kernel (nastar_labels.cuh): bit-exact against the CPU oracle on the fixtures
and on seeded random maps, policy roll-outs, and VanillaAstar path lengths on the labelled maps."""
import os
import sys

import numpy as np
import pytest
import torch

import labels_golden

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

pytestmark = pytest.mark.gpu

_MOVES = ((-1, 0), (0, 1), (0, -1), (1, 0), (-1, 1), (-1, -1), (1, 1), (1, -1))


@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    return torch.device("cuda:0")


def _kernel(maps, goal_idx, dev):
    from neural_astar import _native

    d, m, a = _native.opt_labels(torch.from_numpy(np.ascontiguousarray(maps, np.float32)).to(dev),
                                 torch.from_numpy(np.asarray(goal_idx, np.int32)).to(dev))
    torch.cuda.synchronize()
    return d.cpu().numpy(), m.cpu().numpy(), a.cpu().numpy()


def _assert_matches_oracle(maps, goal_idx, dev):
    from oracle import labels as label_oracle

    d, m, a = _kernel(maps, goal_idx, dev)
    od, om, oa = label_oracle.opt_labels(maps, goal_idx)
    assert np.array_equal(d, od), f"distances differ on {int((d != od).sum())} cells"
    assert np.array_equal(m, om), f"max-set masks differ on {int((m != om).sum())} cells"
    assert np.array_equal(a, oa), "first-max actions differ"
    return d, m, a


def _random_maps(B, H, W, seed, density):
    rs = np.random.RandomState(seed)
    maps = (rs.rand(B, H, W) >= density).astype(np.float32)
    goal_idx = rs.randint(0, H * W, size=B).astype(np.int32)
    maps.reshape(B, -1)[np.arange(B), goal_idx] = 1.0
    return maps, goal_idx


def _rollout_check(maps, goal_idx, d, a):
    """From every reachable cell, following the first-max action reaches the goal in exactly -dist moves and never
    revisits a cell (MazeDataset.__getitem__'s assertion), rolled out for all starts at once: every move goes to a
    passable cell on the grid whose distance is one move shorter."""
    B, H, W = maps.shape
    N = H * W
    dy = np.array([m[0] for m in _MOVES])
    dx = np.array([m[1] for m in _MOVES])
    for b in range(B):
        dist = d[b, 0].ravel().astype(np.int64)
        act = a[b, 0].ravel().astype(np.int64)
        passable = maps[b].ravel() != 0
        if not passable[goal_idx[b]]:
            continue        # an obstacle goal: moves onto it stay put, so no roll-out can end there
        cur = np.flatnonzero(dist > -N)
        steps = -dist[cur]
        for k in range(int(steps.max())):
            live = steps > k
            c = cur[live]
            y, x = np.divmod(c, W)
            ty, tx = y + dy[act[c]], x + dx[act[c]]
            assert ((ty >= 0) & (ty < H) & (tx >= 0) & (tx < W)).all(), "a roll-out leaves the grid"
            nxt = ty * W + tx
            assert passable[nxt].all(), "a roll-out enters an obstacle"
            assert (dist[nxt] == dist[c] + 1).all(), "a roll-out move does not shorten the distance by one"
            cur[live] = nxt
        assert (cur == goal_idx[b]).all(), "a roll-out did not end at the goal"


@pytest.mark.parametrize("name", labels_golden.NAMES)
def test_kernel_matches_fixtures_and_oracle(dev, name):
    maps, goal_idx, dists, action = labels_golden.load(name)
    d, m, a = _assert_matches_oracle(maps, goal_idx, dev)
    assert np.array_equal(d[:, 0], dists)
    assert ((m[:, 0] >> action.astype(np.uint8)) & 1).all()
    _rollout_check(maps, goal_idx, d, a)


SHAPES = [(12, 12), (32, 32), (33, 31), (64, 64), (64, 128), (128, 128), (256, 256), (5, 300), (512, 512)]


@pytest.mark.parametrize("H,W", SHAPES)
def test_kernel_matches_oracle_on_random_maps(dev, H, W):
    B = 24 if H * W <= 128 * 128 else 6
    for density in (0.1, 0.3, 0.5):
        maps, goal_idx = _random_maps(B, H, W, seed=H * 1000 + W + int(density * 10), density=density)
        maps[0] *= np.where(np.random.RandomState(1).rand(H, W) > 0.5, 0.5, 1.0).astype(np.float32)   # non-binary
        maps[1].fill(1.0)
        goal_idx[1] = 0                                     # corner goal on an open map
        goal_idx[2] = H * W - 1
        maps[2].reshape(-1)[-1] = 1.0                       # opposite corner
        gy, gx = divmod(int(goal_idx[3]), W)
        for y in range(gy - 1, gy + 2):
            for x in range(gx - 1, gx + 2):
                if 0 <= y < H and 0 <= x < W and (y, x) != (gy, gx):
                    maps[3, y, x] = 0.0                     # every neighbour of the goal blocked
        d, m, a = _assert_matches_oracle(maps, goal_idx, dev)
        walled = d[3, 0].ravel()
        assert walled[goal_idx[3]] == 0 and (np.delete(walled, goal_idx[3]) == -H * W).all()
        if H * W <= 128 * 128:
            _rollout_check(maps, goal_idx, d, a)


def test_compute_opt_labels_public_api(dev):
    from neural_astar.utils.data import compute_opt_labels

    maps, goal_idx, dists, action = labels_golden.load("mazes032_test")
    B, H, W = maps.shape
    goals = np.zeros((B, 1, H, W), np.float32)
    goals.reshape(B, -1)[np.arange(B), goal_idx] = 1
    pol, d, mask = compute_opt_labels(torch.from_numpy(maps).to(dev)[:, None], torch.from_numpy(goals).to(dev))
    assert pol.shape == (B, 8, 1, H, W) and d.shape == (B, 1, H, W) and mask.shape == (B, 1, H, W)
    assert np.array_equal(d.cpu().numpy()[:, 0], dists)
    p = pol.cpu().numpy()
    assert (p.sum(1) == 1).all()
    first = p[:, :, 0].argmax(1)
    m = mask.cpu().numpy()[:, 0].astype(np.int32)
    assert ((m >> first) & 1).all() and ((m & ((1 << first) - 1)) == 0).all()


@pytest.mark.parametrize("H,W", [(32, 32), (64, 64), (128, 128)])
def test_vanilla_astar_paths_have_optimal_length(dev, H, W):
    """VanillaAstar on GPU-labelled binary maps finds paths of -dist[start] + 1 cells (optimal distances < 700: the
    heuristic's 0.001 * euclid term may add a step on longer paths)."""
    from neural_astar.planner import VanillaAstar
    from neural_astar.utils.data import compute_opt_labels, sample_goal_maps

    import random

    B = 32
    rs = np.random.RandomState(H)
    maps = (rs.rand(B, 1, H, W) > 0.3).astype(np.float32)
    goals = sample_goal_maps(maps, rng=random.Random(H))
    md = torch.from_numpy(maps).to(dev)
    _, d, _ = compute_opt_labels(md, torch.from_numpy(goals).to(dev))
    dn = d.cpu().numpy().reshape(B, -1)
    starts = np.zeros_like(goals)
    want = np.zeros(B, np.int64)
    for b in range(B):
        cand = np.flatnonzero((dn[b] < 0) & (dn[b] > -700) & (dn[b] > -H * W))
        s = cand[rs.randint(len(cand))]
        starts.reshape(B, -1)[b, s] = 1
        want[b] = -dn[b, s] + 1
    out = VanillaAstar().to(dev).eval()(md, torch.from_numpy(starts).to(dev), torch.from_numpy(goals).to(dev))
    got = out.paths.reshape(B, -1).sum(1).cpu().numpy()
    assert np.array_equal(got, want)
