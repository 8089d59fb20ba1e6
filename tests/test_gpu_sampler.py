"""GPU tests of the batch sampler (csrc/nastar_sampler.cuh, utils.data.DeviceMazeDataset): bands bit for bit against
MazeDataset, starts and trajectories bit for bit against the NumPy oracle, coverage, determinism, one launch per
batch, rejection of bad labels, from_labels, and training steps fed by create_device_dataloader."""
import os
import random
import sys
from types import SimpleNamespace

import numpy as np
import pytest
import torch

import labels_golden
import sampler_oracle as so

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    return torch.device("cuda:0")


def _fixture(name):
    """(maps [B,1,H,W], goals [B,1,H,W], one-hot policies [B,8,1,H,W], dists [B,1,H,W]) as float32 NumPy arrays."""
    maps, goal_idx, dists, action = labels_golden.load(name)
    B, H, W = maps.shape
    goals = np.zeros((B, 1, H, W), np.float32)
    goals.reshape(B, -1)[np.arange(B), goal_idx] = 1
    pol = np.zeros((B, 8, 1, H, W), np.float32)
    np.put_along_axis(pol, action[:, None, None].astype(np.int64), 1.0, axis=1)
    return maps[:, None], goals, pol, dists[:, None]


def _random_labelled(B, H, W, seed, dev):
    from neural_astar.utils.data import compute_opt_labels, sample_goal_maps

    rs = np.random.RandomState(seed)
    maps = (rs.rand(B, 1, H, W) > 0.3).astype(np.float32)
    goals = sample_goal_maps(maps, rng=random.Random(seed))
    md, gm = torch.from_numpy(maps).to(dev), torch.from_numpy(goals).to(dev)
    pol, d, _ = compute_opt_labels(md, gm)
    return md, gm, pol, d


def _maze_dataset(pol, dists):
    """MazeDataset over in-memory labels (its _prepared reads only these attributes)."""
    from neural_astar.utils.data import MazeDataset

    ds = MazeDataset.__new__(MazeDataset)
    ds.opt_policies, ds.opt_dists = pol, dists
    ds.pcts = np.array([0.55, 0.70, 0.85, 1.0])
    return ds


def _unpack_bits(bits, N):
    b = bits.cpu().numpy().view(np.uint32)
    return np.unpackbits(b.view(np.uint8), axis=-1, bitorder="little")[..., :N].astype(bool)


def _check_tables(maps, goals, pol, dists, dev):
    """Kernel tables equal MazeDataset._prepared's bands, np.percentile's thresholds and the oracle's status."""
    from neural_astar import _native

    B, _, H, W = maps.shape
    N = H * W
    t = lambda x: torch.as_tensor(x).to(dev)
    bits, counts, goal_idx, actions, th, status = _native.sampler_prepare(t(dists), t(pol), t(goals), so.fractions())
    torch.cuda.synchronize()
    masks = _unpack_bits(bits, N)
    counts, goal_idx, th, status = (x.cpu().numpy() for x in (counts, goal_idx, th, status))
    acts = actions.cpu().numpy().view(np.uint32)
    acts = ((acts[:, :, None] >> (4 * np.arange(8, dtype=np.uint32))) & 15).reshape(B, -1)[:, :N]
    pol_np, d_np, g_np = (np.asarray(x.cpu() if torch.is_tensor(x) else x) for x in (pol, dists, goals))
    ds = _maze_dataset(pol_np, d_np)
    overlaps = non_integer = 0
    for i in range(B):
        od = d_np[i].ravel()
        ref_th = np.percentile(od[od > od.min()], 100.0 * (1 - ds.pcts))
        assert th[i].tobytes() == ref_th.tobytes(), (i, th[i], ref_th)
        bands, _ = ds._prepared(i)
        for r in range(3):
            assert np.array_equal(np.flatnonzero(masks[i, r]), bands[r]), (i, r)
            assert counts[i, r] == len(bands[r])
        act = so.first_max_actions(pol_np[i])
        assert np.array_equal(acts[i], act)
        assert goal_idx[i] == int(np.argmax(g_np[i].ravel()))
        assert status[i] == so.status(od, act, goal_idx[i], H, W, so.fractions()), i
        overlaps += int((masks[i].sum(0) > 1).any())
        non_integer += int((ref_th != np.round(ref_th)).any())
    return overlaps, non_integer, status


@pytest.mark.parametrize("name", labels_golden.NAMES)
def test_bands_equal_maze_dataset_on_fixtures(dev, name):
    overlaps, non_integer, status = _check_tables(*_fixture(name), dev)
    if name != "synthetic":
        assert overlaps > 0 and non_integer > 0
        assert (status == 0).all()


@pytest.mark.parametrize("H,W", [(12, 12), (24, 40), (32, 32), (64, 64), (128, 128), (256, 256), (5, 300), (512, 512)])
def test_bands_equal_maze_dataset_on_labelled_random_maps(dev, H, W):
    B = 16 if H * W <= 128 * 128 else 3
    overlaps, _, status = _check_tables(*_random_labelled(B, H, W, H * 7 + W, dev), dev)
    assert (status == 0).all()
    if H * W >= 32 * 32:
        assert overlaps > 0


def _dataset(arrays, dev, num_starts):
    from neural_astar.utils.data import DeviceMazeDataset

    return DeviceMazeDataset.from_labels(*(torch.as_tensor(x).to(dev) for x in arrays), num_starts=num_starts)


def _assert_batch_equals_oracle(ds, arrays, idx, draws):
    maps, goals, pol, dists = (np.asarray(x.cpu() if torch.is_tensor(x) else x) for x in arrays)
    out = ds.sample(torch.as_tensor(idx), draws=torch.from_numpy(draws.view(np.int32)).to(ds.device))
    md, st, gm, tr = (x.cpu().numpy() for x in out)
    B, S = draws.shape[:2]
    H, W = maps.shape[-2:]
    assert md.shape == (B, 1, H, W) and st.shape == (B, S, H, W) and gm.shape == (B, 1, H, W) and tr.shape == st.shape
    for j, i in enumerate(idx):
        assert np.array_equal(md[j], maps[i]) and np.array_equal(gm[j], goals[i])
        s_ref, t_ref = so.sample(dists[i], pol[i], goals[i], draws[j])
        assert np.array_equal(st[j].reshape(S, -1), s_ref), j
        assert np.array_equal(tr[j].reshape(S, -1), t_ref), j
        od = dists[i].ravel()
        goal = int(goals[i].argmax())
        for s in range(S):
            start = int(s_ref[s].argmax())
            t = tr[j, s].ravel()
            assert t.sum() == -od[start] and t[goal] == 0 and (t[start] == 1 or start == goal)


@pytest.mark.parametrize("S", [1, 3])
@pytest.mark.parametrize("shape", ["synthetic", "mazes032_test", "all064_test", "512x512"])
def test_starts_and_trajectories_equal_oracle(dev, shape, S):
    if shape == "512x512":
        md, gm, pol, d = _random_labelled(3, 512, 512, 11, dev)
        arrays = (md, gm, pol, d)
    else:
        arrays = _fixture(shape)
        if shape == "synthetic":   # map 8's goal is walled in (start == goal, empty trajectory); drop rejected maps
            keep = [i for i in range(len(arrays[0]))
                    if so.status(arrays[3][i].ravel(), so.first_max_actions(arrays[2][i]), int(arrays[1][i].argmax()),
                                 24, 40, so.fractions()) == 0]
            arrays = tuple(x[keep] for x in arrays)
    ds = _dataset(arrays, dev, S)
    n = len(ds)
    rs = np.random.RandomState(S * 100 + n)
    idx = rs.randint(0, n, size=min(64, 4 * n))
    draws = rs.randint(0, 2 ** 32, size=(len(idx), S, 2), dtype=np.uint64).astype(np.uint32)
    draws[0] = 0
    draws[-1] = 2 ** 32 - 1        # first candidate of band 0, last candidate of band 2
    _assert_batch_equals_oracle(ds, arrays, idx, draws)


def test_enumerated_draws_cover_every_candidate(dev):
    arrays = _random_labelled(4, 12, 12, 5, dev)
    ds = _dataset(arrays, dev, 1)
    bits, counts = ds._tables[0], ds._tables[1].cpu().numpy()
    masks = _unpack_bits(bits, 144)
    idx, draws = [], []
    for i in range(4):
        for r in range(3):
            for k in range(int(counts[i, r])):
                idx.append(i)
                draws.append([so.draws_for(r, k, int(counts[i, r]))])
    draws = np.array(draws, np.uint64).astype(np.uint32)
    _, st, _, _ = ds.sample(torch.tensor(idx), draws=torch.from_numpy(draws.view(np.int32)).to(dev))
    got = st[:, 0].reshape(len(idx), -1).argmax(1).cpu().numpy()
    pos = 0
    for i in range(4):
        for r in range(3):
            c = int(counts[i, r])
            assert np.array_equal(got[pos:pos + c], np.flatnonzero(masks[i, r]))   # every candidate, in order
            pos += c


def test_generator_determinism_and_one_launch(dev):
    from neural_astar import _native

    ds = _dataset(_fixture("mazes032_test"), dev, 2)
    idx = torch.arange(100, device=dev)

    def draw(seed):
        g = torch.Generator(device=dev)
        g.manual_seed(seed)
        return ds.sample(idx, generator=g)

    a, b, c = draw(1), draw(1), draw(2)
    assert all(torch.equal(x, y) for x, y in zip(a, b))
    assert not torch.equal(a[1], c[1])
    n0 = _native.launch_count()
    out = ds.sample(idx)
    assert _native.launch_count() - n0 == 1
    torch.cuda.synchronize()
    st = out[1].reshape(100, 2, -1)
    assert (st.sum(-1) == 1).all()
    tr = out[3].reshape(100, 2, -1)
    assert ((tr * st).sum(-1) == 1).all()          # every trajectory contains its start (no start is a goal here)


def test_bad_labels_are_rejected(dev):
    from neural_astar.utils.data import DeviceMazeDataset

    maps, goals, pol, dists = _fixture("mazes032_test")
    B, _, H, W = maps.shape
    t = lambda x: torch.from_numpy(np.ascontiguousarray(x)).to(dev)

    bad_d = dists.copy()
    bad_d[3, 0, 5, 7] += 0.5
    with pytest.raises(ValueError, match=r"integers.*maps \[3\]"):
        DeviceMazeDataset.from_labels(t(maps), t(goals), t(pol), t(bad_d))

    bad_p = pol.copy()
    od = dists[6].ravel()
    goal = int(goals[6].argmax())
    c = int(np.flatnonzero((od > -H * W) & (od < 0))[0])
    y, x = divmod(c, W)
    for a, (dy, dx) in enumerate(so.MOVES):      # an action that does not lead one step closer
        ty, tx = y + dy, x + dx
        if not (0 <= ty < H and 0 <= tx < W) or od[ty * W + tx] != od[c] + 1:
            break
    bad_p[6, :, 0, y, x] = 0
    bad_p[6, a, 0, y, x] = 1
    assert c != goal
    with pytest.raises(ValueError, match=r"policy action.*maps \[6\]"):
        DeviceMazeDataset.from_labels(t(maps), t(goals), t(bad_p), t(dists))

    # pct1 == pct2 makes band 0 the cells at exactly the 45th percentile: empty where that is not an integer
    q = 100.0 * (1 - np.array([0.55, 0.55, 0.85, 1.0]))
    empty = [i for i in range(B) if (lambda th: th[0] != np.round(th[0]))(
        np.percentile(dists[i].ravel()[dists[i].ravel() > dists[i].min()], q))]
    assert empty
    with pytest.raises(ValueError, match="empty percentile band"):
        DeviceMazeDataset.from_labels(t(maps), t(goals), t(pol), t(dists), pct1=0.55, pct2=0.55)


def test_from_labels_equals_file(dev, tmp_path):
    from neural_astar.utils.data import DeviceMazeDataset, save_planning_dataset

    arrays = _fixture("all064_test")
    path = str(tmp_path / "all064.npz")
    save_planning_dataset(path, arrays, arrays, arrays)
    a = DeviceMazeDataset(path, "valid", num_starts=2)
    b = _dataset(arrays, dev, 2)
    for x, y in zip(a._tables, b._tables):
        assert torch.equal(x, y)
    idx = torch.arange(0, 400, 3, device=dev)
    g1, g2 = torch.Generator(device=dev), torch.Generator(device=dev)
    g1.manual_seed(9)
    g2.manual_seed(9)
    assert all(torch.equal(x, y) for x, y in zip(a.sample(idx, g1), b.sample(idx, g2)))


def test_graphed_training_on_device_batches(dev, tmp_path):
    """create_device_dataloader feeds GraphedTrainStep directly; its losses equal eager steps on the same batches, and
    PlannerModule.fit takes the loader as it is."""
    from neural_astar.planner import NeuralAstar
    from neural_astar.utils.data import create_device_dataloader, save_planning_dataset
    from neural_astar.utils.training import GraphedTrainStep, PlannerModule

    arrays = _fixture("mazes032_test")
    path = str(tmp_path / "mazes032.npz")
    save_planning_dataset(path, arrays, arrays, arrays)
    g = torch.Generator(device=dev)
    g.manual_seed(3)
    loader = create_device_dataloader(path, "train", 25, shuffle=True, generator=g)
    batches = list(loader)
    assert len(batches) == len(loader) == 4 and all(b[0].is_cuda and b[1].shape == (25, 1, 32, 32) for b in batches)

    def make():
        torch.manual_seed(1234)
        planner = NeuralAstar(encoder_input="m+", encoder_arch="CNN", encoder_depth=4, Tmax=0.25)
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
    step = GraphedTrainStep(make(), batches[0])
    graph_losses = [float(step(batch)) for batch in batches]
    np.testing.assert_allclose(graph_losses, eager_losses, rtol=2e-3)
    curve = make().fit(create_device_dataloader(path, "test", 50), device=dev)
    assert len(curve) == 2 and all(np.isfinite(curve))
