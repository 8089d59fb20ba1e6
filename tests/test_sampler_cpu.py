"""CPU tests of the GPU batch sampler's specification (no GPU needed): the NumPy oracle (tests/sampler_oracle.py)
against MazeDataset's own bands, thresholds and walks on the label fixtures, and argument checks at the C ABI."""
import ctypes
import os
import subprocess
import sys

import numpy as np
import pytest

import labels_golden
import sampler_oracle as so

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


@pytest.fixture(scope="module")
def built_lib():
    subprocess.check_call(["make", "-C", os.path.join(ROOT, "neural-astar_b200"), "-s", "all"])
    from neural_astar import _native

    return _native


def fixture_dataset(name, tmp_path):
    """The fixture as a planning .npz (train split) and its MazeDataset."""
    from neural_astar.utils.data import MazeDataset, save_planning_dataset

    maps, goal_idx, dists, action = labels_golden.load(name)
    B, H, W = maps.shape
    goals = np.zeros((B, 1, H, W), np.float32)
    goals.reshape(B, -1)[np.arange(B), goal_idx] = 1
    pol = np.zeros((B, 8, 1, H, W), np.float32)
    np.put_along_axis(pol, action[:, None, None].astype(np.int64), 1.0, axis=1)
    split = (maps, goals, pol, dists[:, None])
    path = str(tmp_path / f"{name}.npz")
    save_planning_dataset(path, split, split, split)
    return path, MazeDataset(path, "train")


@pytest.mark.parametrize("name", labels_golden.NAMES)
def test_oracle_bands_equal_maze_dataset(name, tmp_path):
    """Thresholds equal np.percentile bit for bit and bands equal MazeDataset._prepared's on every fixture map."""
    _, ds = fixture_dataset(name, tmp_path)
    q = so.fractions()
    overlaps = non_integer = 0
    for i in range(len(ds)):
        od = ds.opt_dists[i].ravel()
        th = so.thresholds(od, q)
        ref = np.percentile(od[od > od.min()], 100.0 * (1 - ds.pcts))
        assert th.dtype == ref.dtype and th.tobytes() == ref.tobytes(), (i, th, ref)
        masks = so.band_masks(od, th)
        bands, _ = ds._prepared(i)
        for r in range(3):
            assert np.array_equal(np.flatnonzero(masks[r]), bands[r]), (i, r)
        overlaps += int((masks.sum(0) > 1).any())
        non_integer += int((th != np.round(th)).any())
    if name != "synthetic":
        assert overlaps > 0 and non_integer > 0      # both cases the kernel must get right occur in the data


@pytest.mark.parametrize("name", labels_golden.NAMES)
def test_oracle_draws_and_walks_equal_maze_dataset(name, tmp_path):
    """MazeDataset.__getitem__'s start, replayed through the u32 draw mapping, gives the same start and trajectory;
    maps the sampler rejects (status != 0) are exactly the ones whose walk MazeDataset cannot finish."""
    _, ds = fixture_dataset(name, tmp_path)
    q = so.fractions()
    H, W = ds.map_designs.shape[1:]
    np.random.seed(7)
    accepted = 0
    for i in range(len(ds)):
        od = ds.opt_dists[i].ravel()
        act = so.first_max_actions(ds.opt_policies[i])
        goal = int(np.argmax(ds.goal_maps[i].ravel()))
        if so.status(od, act, goal, H, W, q):
            continue
        accepted += 1
        _, starts, _, trajs = ds[i]
        s = int(starts[0].argmax())
        masks = so.band_masks(od, so.thresholds(od, q))
        r = [rr for rr in range(3) if masks[rr, s]][0]
        k = int(np.searchsorted(np.flatnonzero(masks[r]), s))
        d0, d1 = so.draws_for(r, k, int(masks[r].sum()))
        assert (d0 * 3) >> 32 == r and 0 <= d0 < 2 ** 32 and 0 <= d1 < 2 ** 32
        s2, t2 = so.sample(ds.opt_dists[i], ds.opt_policies[i], ds.goal_maps[i], [(d0, d1)])
        assert s2[0].argmax() == s and np.array_equal(t2[0], trajs[0].ravel())
        assert t2[0].sum() == -od[s]
    assert accepted >= len(ds) - 1      # the synthetic fixture has one map whose goal is an obstacle


def test_draw_mapping_extremes():
    m = np.zeros((3, 10), bool)
    m[0, [1, 4]] = m[1, [2]] = m[2, [0, 5, 9]] = True
    assert so.start_from_draws(m, 0, 0) == 1
    assert so.start_from_draws(m, 2 ** 32 - 1, 2 ** 32 - 1) == 9
    for r in range(3):
        cells = np.flatnonzero(m[r])
        for k, c in enumerate(cells):
            assert so.start_from_draws(m, *so.draws_for(r, k, len(cells))) == c


def test_sampler_abi_rejects_bad_arguments_without_a_gpu(built_lib):
    L = built_lib.lib()
    p = ctypes.c_void_p(256)         # never dereferenced: every call below fails validation before any launch
    n0 = built_lib.launch_count()
    q = (0.45, 0.3, 0.15, 0.0)

    def prep(*, d=p, pol=p, g=p, B=2, H=8, W=8, qs=q, out=(p,) * 6):
        return L.nastar_b200_sampler_prepare(d, pol, g, B, H, W, *qs, *out, None)

    assert prep(d=None) == 1 and prep(pol=None) == 1 and prep(g=None) == 1
    for k in range(6):
        out = [p] * 6
        out[k] = None
        assert prep(out=tuple(out)) == 1
    assert prep(B=0) == 1 and prep(H=0) == 1 and prep(W=-3) == 1
    assert prep(qs=(0.45, 0.3, 0.15, -0.1)) == 1 and prep(qs=(1.5, 0.3, 0.15, 0.0)) == 1
    assert prep(qs=(float("nan"), 0.3, 0.15, 0.0)) == 1
    assert prep(H=513) == 2 and prep(W=600) == 2      # NASTAR_EUNSUPPORTED

    def samp(*, ptrs=(p,) * 8, n=4, H=8, W=8, B=2, S=1, outs=(p,) * 4):
        m, g, bits, cnt, gi, act, idx, dr = ptrs
        return L.nastar_b200_sampler_sample(m, g, n, H, W, bits, cnt, gi, act, idx, dr, B, S, *outs, None)

    for k in range(8):
        ptrs = [p] * 8
        ptrs[k] = None
        assert samp(ptrs=tuple(ptrs)) == 1
    for k in range(4):
        outs = [p] * 4
        outs[k] = None
        assert samp(outs=tuple(outs)) == 1
    assert samp(B=0) == 1 and samp(B=-1) == 1 and samp(S=0) == 1 and samp(S=-2) == 1 and samp(n=0) == 1
    assert samp(H=0) == 1 and samp(W=0) == 1
    assert samp(outs=(ctypes.c_void_p(260), p, p, p)) == 1     # float4 stores need 16-B aligned planes
    assert samp(H=513) == 2 and samp(W=1024) == 2
    assert built_lib.launch_count() == n0, "a rejected call must not launch"


def test_device_dataset_needs_cuda_tensors():
    import torch

    from neural_astar.utils.data import DeviceMazeDataset

    maps = torch.ones(2, 1, 8, 8)
    with pytest.raises(RuntimeError, match="CUDA"):
        DeviceMazeDataset.from_labels(maps, torch.zeros(2, 1, 8, 8), torch.zeros(2, 8, 1, 8, 8), torch.zeros(2, 1, 8, 8))
