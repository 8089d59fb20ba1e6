"""GPU tests of the map kernel (csrc/nastar_maps.cuh, utils.data.maps_from_images) and the policy draw
(utils.data.draw_opt_policies): resized image, threshold, status and map bit for bit against the NumPy oracle
(tests/maps_oracle.py), the shipped planning-datasets maps and tiles, one launch per call, and fixture images -> maps
-> goals -> labels -> policies -> a dataset file that MazeDataset and DeviceMazeDataset read."""
import os

import numpy as np
import pytest
import torch

import maps_oracle as mo

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "maps", "sources.npz")

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    return torch.device("cuda:0")


@pytest.fixture(scope="module")
def golden():
    with np.load(GOLDEN) as z:
        return {k: z[k] for k in z.files}


def _assert_equals_oracle(images, H, W, dev):
    from neural_astar import _native

    maps, resized, th, status = _native.maps_from_images(torch.from_numpy(images).to(dev), H, W, want_resized=True)
    maps, resized = maps.cpu().numpy()[:, 0], resized.cpu().numpy()
    th, status = th.cpu().numpy(), status.cpu().numpy()
    for i, img in enumerate(images):
        m, r, t, s = mo.make_map(img, H, W)
        assert np.array_equal(resized[i], r), f"image {i}: resized levels differ"
        assert th[i] == t and status[i] == s, f"image {i}: threshold {th[i]} / {t}, status {status[i]} / {s}"
        assert np.array_equal(maps[i], m), f"image {i}: map differs"
    return maps


def test_fixture_images_equal_oracle_and_shipped_maps(dev, golden):
    imgs = golden["mp_images"]
    maps = _assert_equals_oracle(imgs, 32, 32, dev)
    ship = np.unpackbits(golden["mp_maps"], axis=1)[:, :1024].reshape(-1, 32, 32)
    assert np.array_equal(maps, ship)
    _assert_equals_oracle(golden["tiled_images"], 32, 32, dev)


def test_tiles_replay_shipped_tiled_mp(dev, golden):
    from neural_astar.utils.data import maps_from_images, tile_maps

    pos, count = golden["tiled_pos"], int(golden["tiled_count"])
    maps = maps_from_images(torch.from_numpy(golden["tiled_images"]).to(dev), 32)
    ship = np.unpackbits(golden["tiled_maps"], axis=1).reshape(-1, 64, 64)
    rng = np.random.RandomState(1372)
    idx = np.stack([np.searchsorted(pos, rng.choice(count, 4)) for _ in range(len(ship))])
    tiles = tile_maps(maps, 2, indices=idx)
    assert tiles.shape == (len(ship), 1, 64, 64) and tiles.is_cuda
    assert np.array_equal(tiles.cpu().numpy()[:, 0], ship)


def _random_images(rs, B, h, w):
    imgs = rs.randint(0, 256, (B, h, w)).astype(np.uint8)
    imgs[1] = ((rs.rand(h, w) > 0.4) * 255).astype(np.uint8)
    return imgs


@pytest.mark.parametrize("H0,W0,H,W", [(201, 201, 32, 32), (201, 201, 64, 64), (201, 201, 128, 128),
                                       (201, 201, 256, 256), (201, 201, 512, 512), (1024, 1024, 64, 64),
                                       (5, 700, 300, 3), (2048, 2048, 512, 512), (2048, 3, 1, 7)])
def test_random_images_equal_oracle(dev, H0, W0, H, W):
    _assert_equals_oracle(_random_images(np.random.RandomState(H0 + W), 3, H0, W0), H, W, dev)


def test_special_images_equal_oracle(dev):
    rs = np.random.RandomState(5)
    one = np.array([[[7]], [[0]], [[255]]], np.uint8)
    _assert_equals_oracle(one, 1, 1, dev)
    _assert_equals_oracle(one, 4, 3, dev)
    _assert_equals_oracle(_random_images(rs, 3, 7, 9), 1, 1, dev)
    uniform = np.stack([np.full((201, 201), v, np.uint8) for v in (0, 128, 255)])
    _assert_equals_oracle(uniform, 32, 32, dev)
    two = np.where(rs.rand(4, 60, 50) > 0.5, 40, 200).astype(np.uint8)
    two[1] = 3
    two[1, 0, 0] = 4          # two adjacent levels
    two[2] = 0
    two[2, 30:, :] = 255      # a vertical step: the resize overshoots and clips
    maps = _assert_equals_oracle(two, 60, 50, dev)    # same size: no resize pass
    assert maps[1].sum() == 1
    _assert_equals_oracle(two, 17, 50, dev)           # vertical pass only
    _assert_equals_oracle(two, 60, 23, dev)           # horizontal pass only


def test_groups_restore_file_order_and_one_launch(dev, golden):
    from neural_astar import _native
    from neural_astar.utils.data import maps_from_images

    rs = np.random.RandomState(9)
    small = _random_images(rs, 3, 50, 70)
    groups = [(np.array([4, 0, 2]), golden["mp_images"][:3]), (np.array([1, 3, 5]), small)]
    got = maps_from_images(groups, (24, 40), device=dev).cpu().numpy()[:, 0]
    order = {4: golden["mp_images"][0], 0: golden["mp_images"][1], 2: golden["mp_images"][2], 1: small[0],
             3: small[1], 5: small[2]}
    for p, img in order.items():
        assert np.array_equal(got[p], mo.make_map(img, 24, 40)[0])
    x = torch.from_numpy(golden["mp_images"]).to(dev)
    torch.cuda.synchronize()
    n0 = _native.launch_count()
    maps_from_images(x, 32)
    assert _native.launch_count() - n0 == 1


def _kth_set_bit(mask, k):
    for a in range(8):
        if (mask >> a) & 1:
            if k == 0:
                return a
            k -= 1
    return -1


def test_draw_policies_exact_on_every_mask(dev):
    from neural_astar.utils.data import draw_opt_policies

    masks = np.tile(np.arange(256, dtype=np.uint8), 4).reshape(4, 1, 16, 16)
    draws = np.random.RandomState(1).randint(0, 2 ** 32, masks.shape, dtype=np.uint64).astype(np.uint32)
    draws[0] = 0
    draws[1] = 2 ** 32 - 1
    pol = draw_opt_policies(torch.from_numpy(masks).to(dev),
                            draws=torch.from_numpy(draws.view(np.int32)).to(dev)).cpu().numpy()
    assert pol.shape == (4, 8, 1, 16, 16)
    for b in range(4):
        for c in range(256):
            m, d = int(masks[b, 0].flat[c]), int(draws[b, 0].flat[c])
            col = pol[b, :, 0].reshape(8, -1)[:, c]
            a = _kth_set_bit(m, (d * bin(m).count("1")) >> 32)
            assert np.array_equal(col, np.eye(8, dtype=np.float32)[a] if a >= 0 else np.zeros(8, np.float32))


def test_draw_policies_reach_every_member_and_seeds_reproduce(dev, golden):
    from neural_astar import _native
    from neural_astar.utils.data import (compute_opt_labels, draw_opt_policies, maps_from_images,
                                         sample_device_goal_maps)

    maps = maps_from_images(torch.from_numpy(golden["mp_images"][:16]).to(dev), 32)
    goals = sample_device_goal_maps(maps, 8, generator=torch.Generator(dev).manual_seed(0))
    _, _, mask = compute_opt_labels(maps, goals)
    m = mask.cpu().numpy()[:, 0].astype(np.int64)
    n = np.array([bin(v).count("1") for v in range(256)])[m]
    assert (n > 0).all()
    reached = np.zeros_like(m)
    for k in range(8):
        kk = np.minimum(k, n - 1)
        d = -((-kk << 32) // n)        # ceil(k * 2^32 / n): the first draw that picks member k
        pol = draw_opt_policies(mask, draws=torch.from_numpy(d.astype(np.uint32).view(np.int32)).to(dev))
        p = pol.cpu().numpy()[:, :, 0]
        assert (p.sum(1) == 1).all()
        act = p.argmax(1)
        assert ((m >> act) & 1).all(), "a drawn action outside the maximal set"
        reached |= 1 << act
    assert np.array_equal(reached, m), "enumerated draws miss a member of the maximal set"
    g = torch.Generator(dev)
    a = draw_opt_policies(mask, generator=g.manual_seed(3))
    n0 = _native.launch_count()
    b = draw_opt_policies(mask, generator=g.manual_seed(3))
    assert _native.launch_count() - n0 == 1
    assert torch.equal(a, b)
    assert not torch.equal(a, draw_opt_policies(mask, generator=g.manual_seed(4)))


def test_end_to_end_dataset(dev, golden, tmp_path):
    from neural_astar.planner import VanillaAstar
    from neural_astar.utils.data import (DeviceMazeDataset, MazeDataset, compute_opt_labels, draw_opt_policies,
                                         maps_from_images, sample_device_goal_maps, save_planning_dataset, tile_maps)

    g = torch.Generator(dev).manual_seed(11)
    maps = maps_from_images(torch.from_numpy(golden["mp_images"]).to(dev), 32)
    goals = sample_device_goal_maps(maps, 8, generator=g)
    _, dists, mask = compute_opt_labels(maps, goals)
    pol = draw_opt_policies(mask, generator=g)
    tiles = tile_maps(maps, 2, indices=np.random.RandomState(0).choice(len(maps), (20, 4)))
    tgoals = sample_device_goal_maps(tiles, 16, generator=g)
    _, tdists, tmask = compute_opt_labels(tiles, tgoals)
    split = (maps[:80], goals[:80], pol[:80], dists[:80])
    path = str(tmp_path / "mazes_032_moore_c8.npz")
    save_planning_dataset(path, split, (maps[80:100], goals[80:100], pol[80:100], dists[80:100]),
                          (maps[100:], goals[100:], pol[100:], dists[100:]))
    ds = MazeDataset(path, "train")
    assert len(ds) == 80
    md, start, goal, traj = ds[5]
    od = dists[5, 0].cpu().numpy()
    assert traj.sum() == -od.reshape(-1)[start.reshape(-1).argmax()]
    dds = DeviceMazeDataset.from_labels(*split)
    bm, bs, bg, bt = dds.sample(torch.arange(80), generator=g)
    out = VanillaAstar().to(dev).eval()(bm, bs, bg)
    want = -dists[:80].reshape(80, -1).gather(1, bs.reshape(80, -1).argmax(1, keepdim=True))[:, 0] + 1
    assert torch.equal(out.paths.reshape(80, -1).sum(1).float(), want)
    assert torch.equal(bt.reshape(80, -1).sum(1), want - 1)
    tpol = draw_opt_policies(tmask, generator=g)
    DeviceMazeDataset.from_labels(tiles, tgoals, tpol, tdists)


def test_make_planning_dataset_tool(dev, golden, tmp_path):
    """tools/make_planning_dataset.py on PNGs of the fixture's mazes test images: the test split's maps are the shipped
    ones, every split loads in MazeDataset, and --tile-size 2 makes split-size tiled maps."""
    import argparse
    import sys

    from PIL import Image

    sys.path.insert(0, os.path.join(ROOT, "tools"))
    import make_planning_dataset as mpd
    from neural_astar.utils.data import MazeDataset

    src = tmp_path / "mazes"
    for split, idx in (("train", range(20)), ("validation", range(20, 30)), ("test", range(100))):
        os.makedirs(src / split)
        for i in idx:
            Image.fromarray(golden["mp_images"][i], "L").save(src / split / f"{900 + i}.png")
    args = argparse.Namespace(input_path=str(src) + "/", output_path=str(tmp_path / "out"), maze_size=32,
                              mechanism="moore", edge_ratio=0.25, train_size=6, valid_size=4, test_size=5, seed=1372,
                              tile_size=1)
    path = mpd.make(args)
    assert os.path.basename(path) == "mazes_032_moore_c8.npz"
    ship = np.unpackbits(golden["mp_maps"], axis=1)[:100, :1024].reshape(-1, 32, 32)
    assert np.array_equal(MazeDataset(path, "test").map_designs, ship)
    assert len(MazeDataset(path, "train")) == 20 and len(MazeDataset(path, "valid")) == 10
    args.tile_size = 2
    path = mpd.make(args)
    assert os.path.basename(path) == "mazes_064_moore_c16.npz"
    for split, n in (("train", 6), ("valid", 4), ("test", 5)):
        ds = MazeDataset(path, split)
        assert ds.map_designs.shape == (n, 64, 64)
        ds[0]
