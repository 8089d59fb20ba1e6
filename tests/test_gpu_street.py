"""GPU test of tools/make_street_dataset.py on the street fixture's sources (tests/golden/street/) with the small Ns, in
the glob order the reference saw: every crop file decodes to the crop the reference saved, under the same names and
counts; the .npz maps are the maps oracle's of those crops in natural-sort order; MazeDataset loads the file, and
VanillaAstar's paths on a sample have -opt_dists[start] + 1 cells."""
import os
import sys

import numpy as np
import pytest
import torch
from PIL import Image

import maps_oracle as mo

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
STREET = os.path.join(ROOT, "tests", "golden", "street")
SPLITS = ("train", "validation", "test")


@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    return torch.device("cuda:0")


@pytest.fixture(scope="module")
def built(dev, tmp_path_factory):
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    import make_street_dataset as msd

    golden = dict(np.load(os.path.join(STREET, "street.npz")))
    src = os.path.join(STREET, "sources")
    train = [os.path.join(src, f) for f in golden["glob_train"]]
    test = [os.path.join(src, f) for f in golden["glob_test"]]
    tmp = tmp_path_factory.mktemp("street")
    path = msd.make(train, test, str(tmp / "mixed"), str(tmp / "out"), counts=(8, 2, 4))
    return golden, tmp / "mixed", path


def test_crops_equal_the_reference(built):
    golden, mixed, _ = built
    for s in SPLITS:
        names = list(golden[f"small_names_{s}"])
        assert sorted(os.listdir(mixed / s)) == sorted(names), s
        for name, want in zip(names, golden[f"small_crops_{s}"]):
            with Image.open(mixed / s / name) as im:
                im.load()
                assert im.mode == "L" and im.size == (128, 128)
                assert np.array_equal(np.asarray(im), want), (s, name)


def test_dataset_maps_and_paths(built, dev):
    from neural_astar.planner import VanillaAstar
    from neural_astar.utils.data import MazeDataset

    golden, _, path = built
    assert os.path.basename(path) == "mixed_064_moore_c16.npz"
    z = np.load(path)
    for s, k in zip(SPLITS, (0, 4, 8)):
        names = list(golden[f"small_names_{s}"])
        order = sorted(range(len(names)), key=lambda i: mo.natural_key(names[i]))
        want = np.stack([mo.make_map(golden[f"small_crops_{s}"][i], 64, 64)[0] for i in order])
        assert np.array_equal(z[f"arr_{k}"], want), s
        assert z[f"arr_{k + 2}"].shape == (len(names), 8, 1, 64, 64)
    ds = MazeDataset(path, "test")
    assert len(ds) == 8 and len(MazeDataset(path, "train")) == 32 and len(MazeDataset(path, "valid")) == 8
    maps, goals, dists = z["arr_8"], z["arr_9"], z["arr_11"]
    B = len(maps)
    rs = np.random.RandomState(0)
    starts = np.zeros_like(goals)
    want, keep = np.zeros(B, np.int64), np.zeros(B, bool)
    for b in range(B):
        d = dists[b].reshape(-1)
        cand = np.flatnonzero((d < 0) & (d > -700) & (d > -64 * 64))
        if len(cand):
            s = cand[rs.randint(len(cand))]
            starts.reshape(B, -1)[b, s] = 1
            want[b], keep[b] = -d[s] + 1, True
        else:
            starts.reshape(B, -1)[b] = goals.reshape(B, -1)[b]
    assert keep.sum() >= B // 2
    out = VanillaAstar().to(dev).eval()(torch.from_numpy(maps[:, None]).to(dev), torch.from_numpy(starts).to(dev),
                                        torch.from_numpy(goals).to(dev))
    got = out.paths.reshape(B, -1).sum(1).cpu().numpy()
    assert np.array_equal(got[keep], want[keep])
