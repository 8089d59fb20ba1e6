"""GPU tests of the NEWS (4-action) shortest-path labels (nastar_labels.cuh, kMechNews; compute_opt_labels(...,
mechanism="news")): bit-exact against the CPU oracle, policy roll-outs, policy draws, one launch per call, the Moore
default unchanged, and images -> maps -> goals -> NEWS labels -> a dataset file that MazeDataset and
DeviceMazeDataset read alike."""
import ctypes
import os
import sys

import numpy as np
import pytest
import torch

import labels_golden
from oracle import labels as label_oracle

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
GOLDEN_MAPS = os.path.join(ROOT, "tests", "golden", "maps", "sources.npz")

pytestmark = pytest.mark.gpu

_NEWS_MOVES = ((-1, 0), (0, 1), (0, -1), (1, 0))


@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    return torch.device("cuda:0")


def _kernel(maps, goal_idx, dev, mechanism="news"):
    from neural_astar import _native

    d, m, a = _native.opt_labels(torch.from_numpy(np.ascontiguousarray(maps, np.float32)).to(dev),
                                 torch.from_numpy(np.asarray(goal_idx, np.int32)).to(dev), mechanism)
    torch.cuda.synchronize()
    return d.cpu().numpy(), m.cpu().numpy(), a.cpu().numpy()


def _assert_matches_oracle(maps, goal_idx, dev):
    d, m, a = _kernel(maps, goal_idx, dev)
    od, om, oa = label_oracle.opt_labels(maps, goal_idx, mechanism="news")
    assert np.array_equal(d, od), f"distances differ on {int((d != od).sum())} cells"
    assert np.array_equal(m, om), f"max-set masks differ on {int((m != om).sum())} cells"
    assert np.array_equal(a, oa), "first-max actions differ"
    assert (m < 16).all() and (a < 4).all()
    return d, m, a


def _rollout_check(maps, goal_idx, d, a):
    """From every reachable cell, following the first-max action (one of N, E, W, S) reaches the goal in exactly -dist
    moves: every move goes to a passable 4-neighbour on the grid whose distance is one move shorter."""
    B, H, W = maps.shape
    N = H * W
    dy = np.array([m[0] for m in _NEWS_MOVES])
    dx = np.array([m[1] for m in _NEWS_MOVES])
    for b in range(B):
        dist = d[b, 0].ravel().astype(np.int64)
        act = a[b, 0].ravel().astype(np.int64)
        assert ((act >= 0) & (act < 4)).all()
        passable = maps[b].ravel() != 0
        if not 0 <= goal_idx[b] < N or not passable[goal_idx[b]]:
            continue        # no goal, or an obstacle goal: moves onto it stay put, so no roll-out can end there
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
def test_news_kernel_matches_oracle_on_fixtures(dev, name):
    maps, goal_idx, _, _ = labels_golden.load(name)
    d, m, a = _assert_matches_oracle(maps, goal_idx, dev)
    _rollout_check(maps, goal_idx, d, a)


SHAPES = [(1, 1), (1, 33), (40, 1), (5, 40), (12, 12), (32, 32), (33, 31), (64, 128), (128, 128), (256, 256),
          (5, 300), (512, 512)]


@pytest.mark.parametrize("H,W", SHAPES)
def test_news_kernel_matches_oracle_on_random_maps(dev, H, W):
    B = 24 if H * W <= 128 * 128 else 6
    for density in (0.1, 0.3, 0.5):
        rs = np.random.RandomState(H * 1000 + W + int(density * 10))
        maps = (rs.rand(B, H, W) >= density).astype(np.float32)
        goal_idx = rs.randint(0, H * W, size=B).astype(np.int32)
        maps.reshape(B, -1)[np.arange(B), goal_idx] = 1.0
        maps[0] *= np.where(rs.rand(H, W) > 0.5, 0.5, -3.0).astype(np.float32)      # non-binary
        maps[1].fill(1.0)
        goal_idx[1] = 0                                                             # corner goal on an open map
        maps[2].reshape(-1)[goal_idx[2]] = 0.0                                      # non-passable goal
        gy, gx = divmod(int(goal_idx[3]), W)
        for y, x in ((gy - 1, gx), (gy + 1, gx), (gy, gx - 1), (gy, gx + 1)):
            if 0 <= y < H and 0 <= x < W:
                maps[3, y, x] = 0.0                                                 # 4-neighbours of the goal blocked
        goal_idx[4] = -1                                                            # no goal
        d, m, a = _assert_matches_oracle(maps, goal_idx, dev)
        walled = d[3, 0].ravel()
        assert walled[goal_idx[3]] == 0 and (np.delete(walled, goal_idx[3]) == -H * W).all()
        assert (d[4] == -H * W).all()
        y, x = np.mgrid[0:H, 0:W]
        assert np.array_equal(d[1, 0], -(y + x).astype(np.float32))                # Manhattan on the open map
        if H * W <= 128 * 128:
            _rollout_check(maps, goal_idx, d, a)


def test_news_call_is_one_launch_and_moore_default_is_unchanged(dev):
    """compute_opt_labels(..., "news") is one label launch; the default still gives what nastar_b200_opt_labels, the
    Moore-only entry point, writes, bit for bit."""
    from neural_astar import _native
    from neural_astar.utils.data import compute_opt_labels

    maps_np, goal_idx, dists, _ = labels_golden.load("all064_test")
    B, H, W = maps_np.shape
    maps = torch.from_numpy(maps_np).to(dev)
    gi = torch.from_numpy(goal_idx.astype(np.int32)).to(dev)
    goals = torch.zeros(B, H * W, device=dev).scatter_(1, gi.long()[:, None], 1.0).view(B, 1, H, W)
    n0 = _native.launch_count()
    _native.opt_labels(maps, gi, "news")
    assert _native.launch_count() - n0 == 1
    pol, d, mask = compute_opt_labels(maps, goals, "news")
    assert pol.shape == (B, 4, 1, H, W) and (pol.sum(1) == 1).all()

    L = _native.lib()
    ref = (torch.empty(B, 1, H, W, device=dev), torch.empty(B, 1, H, W, dtype=torch.uint8, device=dev),
           torch.empty(B, 1, H, W, dtype=torch.int8, device=dev))
    stream = ctypes.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
    assert L.nastar_b200_opt_labels(maps.data_ptr(), H * W, gi.data_ptr(), B, H, W, *(t.data_ptr() for t in ref),
                                    stream) == 0
    ref_pol = torch.zeros(B, 8, 1, H, W, device=dev).scatter_(1, ref[2].long().view(B, 1, 1, H, W), 1.0)
    for out in (compute_opt_labels(maps, goals), compute_opt_labels(maps[:, None], goals, "moore")):
        p8, d8, m8 = out
        assert torch.equal(p8, ref_pol) and torch.equal(d8, ref[0]) and torch.equal(m8, ref[1])
    assert np.array_equal(ref[0].cpu().numpy()[:, 0], dists)
    with pytest.raises(ValueError, match="mechanism"):
        compute_opt_labels(maps, goals, "hex")


def test_draw_opt_policies_with_four_actions_follows_the_bit_rule(dev):
    from neural_astar import _native
    from neural_astar.utils.data import compute_opt_labels, draw_opt_policies

    maps, goal_idx, _, _ = labels_golden.load("mixed064_test")
    B, H, W = maps.shape
    goals = np.zeros((B, 1, H, W), np.float32)
    goals.reshape(B, -1)[np.arange(B), goal_idx] = 1
    _, _, mask = compute_opt_labels(torch.from_numpy(maps).to(dev), torch.from_numpy(goals).to(dev), "news")
    m = mask.cpu().numpy()[:, 0].astype(np.int64)
    assert (m > 0).all() and (m < 16).all()
    n = np.array([bin(v).count("1") for v in range(256)])[m]
    reached = np.zeros_like(m)
    for k in range(4):
        kk = np.minimum(k, n - 1)
        d = -((-kk << 32) // n)        # ceil(k * 2^32 / n): the first draw that picks member k
        draws = torch.from_numpy(d.astype(np.uint32).view(np.int32)).to(dev)
        pol = draw_opt_policies(mask, draws=draws, num_actions=4)
        assert pol.shape == (B, 4, 1, H, W) and pol.is_contiguous()
        assert torch.equal(pol, draw_opt_policies(mask, draws=draws)[:, :4])
        p = pol.cpu().numpy()[:, :, 0]
        assert (p.sum(1) == 1).all()
        act = p.argmax(1)
        assert ((m >> act) & 1).all(), "a drawn action outside the maximal set"
        reached |= 1 << act
    assert np.array_equal(reached, m), "enumerated draws miss a member of the maximal set"
    g = torch.Generator(dev)
    n0 = _native.launch_count()
    a = draw_opt_policies(mask, generator=g.manual_seed(3), num_actions=4)
    assert _native.launch_count() - n0 == 1
    assert torch.equal(a, draw_opt_policies(mask, generator=g.manual_seed(3), num_actions=4))
    with pytest.raises(ValueError, match="num_actions"):
        draw_opt_policies(mask, num_actions=5)


def test_news_end_to_end_dataset(dev, tmp_path):
    """Images -> maps -> goals -> NEWS labels -> drawn policies -> a 4-action file.  MazeDataset and DeviceMazeDataset
    (from the file and from the labels) read it; the device trajectories are the reference roll-outs of the same starts,
    with -opt_dists[start] cells; VanillaAstar (8-connected) paths are no longer than the NEWS optimum."""
    from neural_astar.planner import VanillaAstar
    from neural_astar.utils.data import (DeviceMazeDataset, MazeDataset, compute_opt_labels, draw_opt_policies,
                                         maps_from_images, sample_device_goal_maps, save_planning_dataset)

    with np.load(GOLDEN_MAPS) as z:
        images = z["mp_images"]
    g = torch.Generator(dev).manual_seed(5)
    maps = maps_from_images(torch.from_numpy(images).to(dev), 32)
    goals = sample_device_goal_maps(maps, 8, generator=g)
    _, dists, mask = compute_opt_labels(maps, goals, "news")
    pol = draw_opt_policies(mask, generator=g, num_actions=4)
    n = 80
    split = (maps[:n], goals[:n], pol[:n], dists[:n])
    path = str(tmp_path / "mazes_032_news_c8.npz")
    save_planning_dataset(path, split, (maps[80:100], goals[80:100], pol[80:100], dists[80:100]),
                          (maps[100:], goals[100:], pol[100:], dists[100:]))
    ds = MazeDataset(path, "train")
    assert ds.num_actions == 4 and len(ds) == n
    np.random.seed(0)
    for i in range(0, n, 7):
        _, start, _, traj = ds[i]
        assert traj.sum() == -dists[i].reshape(-1)[int(start.reshape(-1).argmax())].item()

    for dds in (DeviceMazeDataset(path, "train"), DeviceMazeDataset.from_labels(*split)):
        bm, bs, bg, bt = dds.sample(torch.arange(n), generator=g)
        want = -dists[:n].reshape(n, -1).gather(1, bs.reshape(n, -1).argmax(1, keepdim=True))[:, 0]
        assert torch.equal(bt.reshape(n, -1).sum(1), want)
        bs_np, bt_np = bs.cpu().numpy(), bt.cpu().numpy()
        for i in range(n):
            ref = ds.get_opt_traj(bs_np[i][None, 0], ds.goal_maps[i], ds.opt_policies[i])
            assert np.array_equal(ref[0], bt_np[i, 0]), f"map {i}: device and MazeDataset trajectories differ"
        out = VanillaAstar().to(dev).eval()(bm, bs, bg)
        assert (out.paths.reshape(n, -1).sum(1).float() - 1 <= want).all()
