"""GPU tests of the goal sampler (csrc/nastar_goals.cuh, utils.data.sample_device_goal_maps): goal index, goal plane and
status bit for bit against the NumPy oracle (tests/goals_oracle.py) with explicit draws, coverage of every candidate,
determinism, one launch per call, and goals -> labels -> training batches on Config-5 maps."""
import os
import sys

import numpy as np
import pytest
import torch
from scipy import ndimage

import goals_oracle as go
import labels_golden

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    return torch.device("cuda:0")


def _draws(rs, B):
    d = rs.randint(0, 2 ** 32, size=B, dtype=np.uint64).astype(np.uint32)
    d[0] = 0
    d[-1] = 2 ** 32 - 1   # first and last candidate
    return d


def _assert_equals_oracle(maps, e, draws, dev, maps_t=None):
    """maps: float32 [B,H,W]; maps_t: the same maps as a CUDA tensor (default: a dense copy)"""
    from neural_astar import _native

    maps_t = torch.from_numpy(maps).to(dev) if maps_t is None else maps_t
    d = torch.from_numpy(np.asarray(draws, np.uint32).view(np.int32)).to(dev)
    gi, gm, st = (x.cpu().numpy() for x in _native.sample_goals(maps_t, d, e))
    ref_gi, ref_gm, ref_st = go.sample(maps, e, draws)
    assert np.array_equal(st, ref_st)
    assert np.array_equal(gi, ref_gi), np.flatnonzero(gi != ref_gi)[:10]
    assert gm.tobytes() == ref_gm.tobytes()
    return gi, st


@pytest.mark.parametrize("name", labels_golden.NAMES)
def test_equals_oracle_on_label_fixtures(dev, name):
    maps = labels_golden.load(name)[0]
    B, H, W = maps.shape
    rs = np.random.RandomState(B)
    for e in (0, H // 4, (max(H, W) + 1) // 2, max(H, W) + 1):
        _assert_equals_oracle(maps, e, _draws(rs, B), dev)


SHAPES = [(1, 1), (1, 512), (5, 40), (33, 31), (32, 32), (64, 64), (100, 72), (128, 128), (256, 256), (300, 5),
          (512, 512)]


@pytest.mark.parametrize("p", [0.2, 0.4, 0.5])
@pytest.mark.parametrize("H,W", SHAPES)
def test_equals_oracle_on_bernoulli_maps(dev, H, W, p):
    """p = 0.4 and 0.5 lie near 4-connected percolation: many regions of similar size"""
    B = 4 if H * W >= 256 * 256 else 24
    rs = np.random.RandomState(H * 1000 + W + int(100 * p))
    maps = (rs.rand(B, H, W) >= p).astype(np.float32)
    maps[1] = 1.0
    for e in (0, max(1, H // 4)):
        gi, st = _assert_equals_oracle(maps, e, _draws(rs, B), dev)
        assert (st == 0).all() or H * W == 1


def test_strided_maps_equal_oracle(dev):
    rs = np.random.RandomState(3)
    both = (rs.rand(16, 2, 40, 24) >= 0.4).astype(np.float32)
    t = torch.from_numpy(both).to(dev)[:, 1]    # map stride 2*H*W
    assert t.stride(0) == 2 * 40 * 24
    _assert_equals_oracle(np.ascontiguousarray(both[:, 1]), 6, _draws(rs, 16), dev, maps_t=t)


def _spiral(n):
    """one 1-wide corridor spiralling inwards: a single region whose union chains are long"""
    m = np.zeros((n, n), np.float32)
    y = x = 0
    m[0, 0] = 1
    lengths = [n - 1, n - 1, n - 1] + [L for k in range(n - 3, 0, -2) for L in (k, k)]
    for i, L in enumerate(lengths):
        dy, dx = ((0, 1), (1, 0), (0, -1), (-1, 0))[i % 4]
        for _ in range(L):
            y, x = y + dy, x + dx
            m[y, x] = 1
    return m


def _special_maps():
    H = W = 64
    checker = (np.indices((H, W)).sum(0) % 2).astype(np.float32)
    two = np.ones((H, 2 * 32 + 1), np.float32)
    two[:, 32] = 0      # two 64x32 regions: the left one starts first
    ring = np.zeros((H, W), np.float32)
    ring[12:52, 12:52] = 1
    ring[:3, :3] = ring[-2:, -3:] = 1      # small corner blobs; the largest region reaches no corner square
    nonbin = np.where(np.random.RandomState(2).rand(H, W) < 0.35, 0.0,
                      np.random.RandomState(3).choice([0.5, -1.0, 2.0, 1e-30], size=(H, W))).astype(np.float32)
    return {"checkerboard": checker, "two_equal_regions": two, "ring_no_corner": ring, "non_binary": nonbin,
            "all_passable": np.ones((H, W), np.float32), "spiral_512": _spiral(512)}


@pytest.mark.parametrize("name", ["checkerboard", "two_equal_regions", "ring_no_corner", "non_binary", "all_passable",
                                  "spiral_512"])
def test_equals_oracle_on_special_maps(dev, name):
    m = _special_maps()[name]
    H, W = m.shape
    maps = np.repeat(m[None], 8, axis=0)
    rs = np.random.RandomState(5)
    for e in (0, 3, 8, H // 4, max(H, W) + 1):
        gi, _ = _assert_equals_oracle(maps, e, _draws(rs, 8), dev)
    if name == "checkerboard":
        assert (gi == gi[0]).all() and gi[0] == 1   # every region is one cell: the first passable cell wins the tie
    if name == "two_equal_regions":
        assert (gi % m.shape[1] < 32).all()
    if name == "ring_no_corner":
        assert all(12 <= g // W < 52 for g in gi)
    if name == "spiral_512":
        assert len(go.candidates(m, 0)) == int(m.sum())   # one region


def test_no_passable_cell(dev):
    from neural_astar.utils.data import sample_device_goal_maps

    maps = np.ones((5, 20, 30), np.float32)
    maps[1] = 0
    maps[3] = 0
    gi, st = _assert_equals_oracle(maps, 4, np.arange(5, dtype=np.uint32) * 7 ** 9, dev)
    assert st.tolist() == [0, 1, 0, 1, 0] and gi[1] == gi[3] == -1
    with pytest.raises(ValueError, match=r"maps \[1, 3\]"):
        sample_device_goal_maps(torch.from_numpy(maps).to(dev))


@pytest.mark.parametrize("e", [0, 3])
def test_enumerated_draws_reach_every_candidate(dev, e):
    from neural_astar import _native

    m = (np.random.RandomState(8).rand(12, 12) >= 0.3).astype(np.float32)
    cand = go.candidates(m, e)
    n = len(cand)
    assert n > 1
    draws = np.array([go.draw_for(k, n) for k in range(n)] + [go.draw_for(k + 1, n) - 1 for k in range(n - 1)],
                     np.uint64).astype(np.uint32)
    maps = torch.from_numpy(np.repeat(m[None], len(draws), axis=0)).to(dev)
    gi, _, _ = _native.sample_goals(maps, torch.from_numpy(draws.view(np.int32)).to(dev), e)
    gi = gi.cpu().numpy()
    assert np.array_equal(gi[:n], cand)                 # the smallest draw of each candidate
    assert np.array_equal(gi[n:], cand[:-1])            # the largest draw of each candidate
    assert set(gi.tolist()) == set(cand.tolist())


def test_determinism_generator_and_one_launch(dev):
    from neural_astar import _native
    from neural_astar.utils.data import sample_device_goal_maps

    rs = np.random.RandomState(4)
    maps = torch.from_numpy((rs.rand(64, 1, 300, 200) >= 0.45).astype(np.float32)).to(dev)
    d = torch.from_numpy(_draws(rs, 64).view(np.int32)).to(dev)
    a, b = sample_device_goal_maps(maps, 50, draws=d), sample_device_goal_maps(maps, 50, draws=d)
    assert torch.equal(a, b)

    def seeded(seed):
        g = torch.Generator(device=dev)
        g.manual_seed(seed)
        return sample_device_goal_maps(maps, 50, generator=g)

    x, y, z = seeded(1), seeded(1), seeded(2)
    assert torch.equal(x, y) and not torch.equal(x, z)
    assert (x.view(64, -1).sum(1) == 1).all() and x.shape == (64, 1, 300, 200) and x.dtype == torch.float32
    n0 = _native.launch_count()
    sample_device_goal_maps(maps, 50)
    assert _native.launch_count() - n0 == 1
    n0 = _native.launch_count()
    sample_device_goal_maps(maps[:, 0], draws=d)
    assert _native.launch_count() - n0 == 1


def test_config5_goals_labels_and_batches(dev):
    from c5_data import c5_maps
    from neural_astar.utils.data import DeviceMazeDataset, compute_opt_labels, sample_device_goal_maps

    obst = c5_maps(1024, 256, 256, 77)[0]
    md = torch.from_numpy(obst).to(dev)
    g = torch.Generator(device=dev)
    g.manual_seed(0)
    goals = sample_device_goal_maps(md, 64, generator=g)
    pol, dists, _ = compute_opt_labels(md, goals)
    ds = DeviceMazeDataset.from_labels(md, goals, pol, dists, num_starts=2)
    batch = ds.sample(torch.arange(0, 1024, 4, device=dev), generator=g)
    torch.cuda.synchronize()
    assert batch[1].shape == (256, 2, 256, 256) and (batch[1].view(256, 2, -1).sum(-1) == 1).all()
    gi = goals.view(1024, -1).argmax(1).cpu().numpy()
    assert (goals.view(1024, -1).sum(1) == 1).all()
    for i in range(1024):
        lab, _ = ndimage.label(obst[i, 0] != 0)
        counts = np.bincount(lab.ravel())
        counts[0] = 0
        assert lab.ravel()[gi[i]] == np.argmax(counts), i   # the goal lies in the largest region
