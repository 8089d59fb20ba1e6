"""GPU tests of Neural A* training on the Stanford Drone samples (DESIGN.md §23): chamfer_distances
(nastar_b200_chamfer) against the scipy oracle (tests/chamfer_oracle.py) and bit-identical from run to run, with every
square root correctly rounded; DeviceSDDDataset and sdd_leave_one_scene_out on the fixture tree against a host
construction from np.load; GraphedTrainStep on rgb+ / learn_obstacles batches against the eager step; and
tools/train_sdd.py end to end.  The pipeline is checked, not the quality of what it learns."""
import glob
import json
import os
import sys
from types import SimpleNamespace

import numpy as np
import pytest
import torch

import chamfer_oracle as co

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SDD = os.path.join(ROOT, "tests", "golden", "sdd", "original")


@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    return torch.device("cuda:0")


@pytest.fixture(scope="module")
def tree(dev, tmp_path_factory):
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    import make_sdd_dataset

    return make_sdd_dataset.main(["--input-path", SDD, "--save-dir", str(tmp_path_factory.mktemp("sdd"))])


def masks(kind, B, H, W, rng):
    if kind == "random":
        return rng.rand(B, H, W) < 0.2, rng.rand(B, H, W) < 0.05
    if kind == "single":
        a, b = np.zeros((B, H, W), bool), np.zeros((B, H, W), bool)
        a[np.arange(B), rng.randint(0, H, B), rng.randint(0, W, B)] = True
        b[np.arange(B), rng.randint(0, H, B), rng.randint(0, W, B)] = True
        return a, b
    if kind == "full":
        return np.ones((B, H, W), bool), rng.rand(B, H, W) < 0.1
    a, b = rng.rand(B, H, W) < 0.3, rng.rand(B, H, W) < 0.3   # "empty": one set empty in every other map
    a[::2] = False
    return a, b


def as_dtype(x, dtype, rng, dev):
    t = torch.from_numpy(x)
    if dtype == torch.bool:
        return t.to(dev)
    vals = torch.from_numpy(rng.randint(1, 9, x.shape)) * (1 if dtype == torch.int64 else -0.5)
    return torch.where(t, vals, torch.zeros_like(vals)).to(dtype).to(dev)


@pytest.mark.parametrize("H,W", [(1, 1), (7, 13), (64, 64), (200, 37), (1024, 1024)])
@pytest.mark.parametrize("kind", ["random", "single", "full", "empty"])
def test_chamfer_equals_scipy_and_repeats_bit_for_bit(dev, H, W, kind):
    from neural_astar.utils.training import chamfer_distance, chamfer_distances

    rng = np.random.RandomState(H * 7 + W + len(kind))
    B = 2 if H * W > 100000 else 6
    a, b = masks(kind, B, H, W, rng)
    want = co.chamfer(a, b)
    for dtype in (torch.float32, torch.float64, torch.int64, torch.bool):
        ta, tb = as_dtype(a, dtype, rng, dev), as_dtype(b, dtype, rng, dev)
        got = chamfer_distances(ta[:, None], tb[:, None])
        assert got.dtype == torch.float64 and tuple(got.shape) == (B, 2)
        np.testing.assert_allclose(got.cpu().numpy(), want, rtol=1e-12, atol=0, equal_nan=True)
        again = chamfer_distances(ta, tb)
        assert torch.equal(got.nan_to_num(-1.0), again.nan_to_num(-1.0)), "results differ between two calls"
        swapped = chamfer_distances(tb, ta)
        assert torch.equal(swapped.flip(1).nan_to_num(-1.0), got.nan_to_num(-1.0))
        s = chamfer_distance(ta, tb)
        assert torch.equal(s.nan_to_num(-1.0), got.sum(1).nan_to_num(-1.0))
    same = chamfer_distances(ta, ta).cpu()
    filled = torch.from_numpy(a.reshape(B, -1).any(1))
    assert (same[filled] == 0).all() and same[~filled].isnan().all()


@pytest.mark.parametrize("H,W", [(64, 64), (8, 1024)])
def test_every_square_root_is_correctly_rounded(dev, H, W):
    """One cell in each set: d(A -> B) is one square root, which must equal NumPy's (IEEE, correctly rounded)."""
    from neural_astar.utils.training import chamfer_distances

    dy, dx = np.divmod(np.arange(H * W), W)
    a = np.zeros((H * W, H, W), bool)
    b = np.zeros((H * W, H, W), bool)
    a[:, 0, 0] = True
    b[np.arange(H * W), dy, dx] = True
    got = chamfer_distances(torch.from_numpy(a).to(dev), torch.from_numpy(b).to(dev)).cpu().numpy()
    want = np.sqrt((dy * dy + dx * dx).astype(np.float64))
    assert np.array_equal(got[:, 0], want) and np.array_equal(got[:, 1], want)


def test_chamfer_of_planner_paths_against_fixture_trajectories(dev, tree):
    from neural_astar.planner import VanillaAstar
    from neural_astar.utils.data import DeviceSDDDataset
    from neural_astar.utils.training import chamfer_distances

    ds = DeviceSDDDataset(tree, device=dev)
    paths = VanillaAstar().to(dev)(torch.ones_like(ds.start_maps), ds.start_maps, ds.goal_maps).paths
    got = chamfer_distances(paths, ds.traj_images)
    want = co.chamfer(paths.cpu().numpy(), ds.traj_images.cpu().numpy())
    np.testing.assert_allclose(got.cpu().numpy(), want, rtol=1e-12, atol=0)
    assert torch.isfinite(got).all()


def host_dataset(files):
    zs = [np.load(f) for f in files]
    return dict(
        map_designs=np.stack([(z["image"].transpose(2, 0, 1) / 255.0).astype(np.float32) for z in zs]),
        start_maps=np.stack([z["start_image"] for z in zs])[:, None].astype(np.float32),
        goal_maps=np.stack([z["goal_image"] for z in zs])[:, None].astype(np.float32),
        traj_images=np.stack([z["traj_image"] for z in zs])[:, None].astype(np.float32),
        label=np.stack([z["label"] for z in zs]), length_ratio=np.stack([z["length_ratio"] for z in zs]),
        traj=np.concatenate([z["traj"] for z in zs]),
        traj_offsets=np.concatenate([[0], np.cumsum([len(z["traj"]) for z in zs])]))


def test_dataset_equals_host_construction(dev, tree):
    from neural_astar import _native
    from neural_astar.utils.data import DeviceSDDDataset

    n0 = _native.launch_count()
    ds = DeviceSDDDataset(tree, device=dev)
    assert _native.launch_count() - n0 == 1
    files = sorted(glob.glob(os.path.join(tree, "*", "*", "*.npz")))
    assert len(ds) == len(files) == 21
    assert [os.path.join(tree, s, n) for s, n in zip(ds.scene, ds.name)] == files
    want = host_dataset(files)
    for k, w in want.items():
        t = getattr(ds, k)
        assert t.is_cuda and torch.equal(t.cpu(), torch.from_numpy(w)), k
    assert ds.map_designs.shape[1:] == (3, 64, 64)


def test_leave_one_scene_out_partitions_the_scenes(dev, tree):
    from neural_astar.utils.data import DeviceSDDDataset, sdd_leave_one_scene_out

    everything = DeviceSDDDataset(tree, device=dev)
    scenes = sorted(set(everything.scene))
    assert len(scenes) == 3
    for s in scenes:
        train, test = sdd_leave_one_scene_out(tree, s, dev)
        assert set(test.scene) == {s} and s not in set(train.scene)
        assert len(train) + len(test) == len(everything)
        assert sorted(zip(train.scene + test.scene, train.name + test.name)) == \
            sorted(zip(everything.scene, everything.name))
    with pytest.raises(ValueError, match="no scene"):
        sdd_leave_one_scene_out(tree, "nowhere", dev)
    with pytest.raises(ValueError, match="no scene"):
        DeviceSDDDataset(tree, ["nowhere"], dev)


def test_device_dataloader_batches_equal_sample(dev, tree):
    from neural_astar.utils.data import DeviceDataLoader, DeviceSDDDataset

    ds = DeviceSDDDataset(tree, device=dev)
    g1 = torch.Generator(device=dev).manual_seed(5)
    batches = list(DeviceDataLoader(ds, 8, shuffle=True, generator=g1))
    order = torch.randperm(len(ds), device=dev, generator=torch.Generator(device=dev).manual_seed(5))
    assert [b[0].shape[0] for b in batches] == [8, 8, 5]
    for i, batch in enumerate(batches):
        want = ds.sample(order[8 * i:8 * i + 8])
        assert all(torch.equal(x, y) for x, y in zip(batch, want))
    assert ds.sample([0, 3])[0].shape == (2, 3, 64, 64)


@pytest.mark.parametrize("arch", ["CNN", "Unet"])
def test_graphed_train_step_equals_eager_on_sdd_batches(dev, tree, arch):
    from neural_astar.planner import NeuralAstar
    from neural_astar.utils.data import DeviceSDDDataset
    from neural_astar.utils.training import GraphedTrainStep, PlannerModule

    ds = DeviceSDDDataset(tree, device=dev)
    batches = [ds.sample(range(0, 8)), ds.sample(range(8, 16)), ds.sample(range(13, 21))]

    def make():
        torch.manual_seed(1234)
        planner = NeuralAstar(encoder_input="rgb+", encoder_arch=arch, learn_obstacles=True, Tmax=0.25)
        return PlannerModule(planner, SimpleNamespace(params=SimpleNamespace(lr=1e-3))).to(dev).train()

    eager = make()
    opt = eager.configure_optimizers()
    eager_losses = []
    for i, batch in enumerate(batches):
        opt.zero_grad()
        loss = eager.training_step(batch, i)
        loss.backward()
        opt.step()
        eager_losses.append(float(loss))
    graphed = make()
    step = GraphedTrainStep(graphed, batches[0])
    graph_losses = [float(step(b)) for b in batches]
    assert step.replays == 3
    np.testing.assert_allclose(graph_losses, eager_losses, rtol=2e-3)
    pe = float(sum(p.detach().abs().sum() for p in eager.planner.parameters()))
    pg = float(sum(p.detach().abs().sum() for p in graphed.planner.parameters()))
    assert pg == pytest.approx(pe, rel=1e-3)


def test_train_tool_prints_one_json_line_per_scene(dev, tree, capsys):
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    import train_sdd

    train_sdd.main(["--data-dir", tree, "--all-scenes", "--epochs", "1", "--batch-size", "4"])
    out = capsys.readouterr()
    recs = [json.loads(line) for line in out.out.splitlines() if line.startswith("{")]
    assert [r["test_scene"] for r in recs] == sorted(os.listdir(tree))
    for r in recs:
        assert r["train_samples"] + r["test_samples"] == 21 and r["epochs"] == 1
        assert np.isfinite(r["chamfer_neural_astar"]) and np.isfinite(r["chamfer_vanilla_astar"])
        assert np.isfinite(r["final_train_loss"]) and r["seconds"] > 0
    assert "dropped" in out.err
