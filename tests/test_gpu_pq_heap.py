"""The reference heap A* on the GPU (csrc/nastar_pq.cuh; pq_astar(semantics="reference"), the planners'
pq_semantics="reference"): bit-equal to the reference's goldens and to the C oracle (oracle/pq_oracle.c)."""
import os
import sys

import numpy as np
import pytest
import torch

import pq_golden
from golden_util import Golden

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tools")]
from oracle import pq as pq_oracle  # noqa: E402

pytestmark = pytest.mark.gpu


def _cuda(*xs):
    return [torch.from_numpy(np.ascontiguousarray(x, dtype=np.float32)).cuda() for x in xs]


def _kernel(cost, start, goal, obst, g_ratio):
    from neural_astar import _native

    out = _native.pq_astar(*_cuda(cost, start, goal, obst), g_ratio)
    return [t.cpu().numpy() for t in out]


def _assert_equal_oracle(cost, start, goal, obst, g_ratio, out=None):
    got = out if out is not None else _kernel(cost, start, goal, obst, g_ratio)
    want = pq_oracle.pq_astar(cost, start, goal, obst, g_ratio)
    for name, a, b in zip(("histories", "paths", "status", "expansions"), got, want):
        np.testing.assert_array_equal(a, b, err_msg=name)
    return want


@pytest.mark.parametrize("name", pq_golden.NAMES)
def test_kernel_equals_golden(name):
    g = pq_golden.PqGolden(name)
    hist, paths, status, exp = _kernel(g.cost, g.start, g.goal, g.obst, g.g_ratio)
    eh, ep, es, ee = g.expected
    np.testing.assert_array_equal(status, es)
    np.testing.assert_array_equal(hist, eh)
    np.testing.assert_array_equal(paths, ep)
    np.testing.assert_array_equal(exp[es == 0], ee[es == 0])


def _ckpt_planner():
    from neural_astar.planner import NeuralAstar

    state = np.load(os.path.join(ROOT, "tests", "golden", "mazes032_ckpt_planner_state.npz"))
    na = NeuralAstar(encoder_arch="CNN", use_differentiable_astar=False, pq_semantics="reference")
    na.load_state_dict({k: torch.from_numpy(state[k]) for k in state.files})
    return na.cuda().eval()


def test_neural_astar_reference_mode_on_all_1000_mazes():
    g = Golden("inputs_mazes032_all1000")
    na = _ckpt_planner()
    maps, start, goal = _cuda(g.obst, g.start, g.goal)
    with torch.no_grad():
        cost = na.encode(maps, start, goal)
        out = na.perform_astar(cost, start, goal, maps)
    c = cost.cpu().numpy()
    want = pq_oracle.pq_astar(c, g.start, g.goal, g.obst, 0.5)
    assert out.histories.dtype == torch.float32 and out.paths.dtype == torch.int64 and out.histories.is_cuda
    np.testing.assert_array_equal(out.histories.cpu().numpy(), want[0])
    np.testing.assert_array_equal(out.paths.cpu().numpy(), want[1])
    assert (want[2] == 0).all()


def test_all064_400_maps():
    g = Golden("inputs_all064_test400")
    rng = np.random.RandomState(64)
    cost = rng.rand(g.B, 1, g.H, g.W).astype(np.float32)
    _assert_equal_oracle(g.obst, g.start, g.goal, g.obst, 0.5)
    _assert_equal_oracle(cost, g.start, g.goal, g.obst, 0.5)


def test_64_maps_of_256x256_binary_and_random_cost():
    from c5_data import c5_maps

    obst, start, goal = c5_maps(64, 256, 256, seed=17)
    cost = np.random.RandomState(17).rand(64, 1, 256, 256).astype(np.float32)
    _assert_equal_oracle(obst, start, goal, obst, 0.5)
    _assert_equal_oracle(cost, start, goal, obst, 0.5)


@pytest.mark.parametrize("H,W", [(32, 32), (64, 64), (100, 100), (128, 128)])
def test_batch_of_one_each_state_placement(H, W):
    from c5_data import c5_maps

    obst, start, goal = c5_maps(1, H, W, seed=H)
    cost = np.random.RandomState(H).rand(1, 1, H, W).astype(np.float32)
    _assert_equal_oracle(cost, start, goal, obst, 0.5)


def test_4096_maps_beyond_the_resident_ctas():
    g = Golden("inputs_mazes032_all1000")
    idx = np.arange(4096) % g.B
    rng = np.random.RandomState(4096)
    cost = (rng.rand(4096, 1, 32, 32) * 0.9 + 0.1).astype(np.float32)
    want = _assert_equal_oracle(cost, g.start[idx], g.goal[idx], g.obst[idx], 0.6)
    assert (want[2] == 0).all()


@pytest.mark.parametrize("B,H,W", [(8, 41, 41), (8, 45, 45), (6, 255, 255), (4, 1, 2001), (4, 2001, 1)])
def test_global_state_with_odd_cell_counts(B, H, W):
    """An odd H*W above the shared-memory threshold on several CTAs: each workspace slot must keep its fp64 array
    8-byte aligned."""
    from c5_data import c5_maps

    if H > 1 and W > 1:
        obst, start, goal = c5_maps(B, H, W, seed=H)
    else:
        obst = np.ones((B, 1, H, W), np.float32)
        start, goal = np.zeros_like(obst), np.zeros_like(obst)
        start.reshape(B, -1)[:, 0] = 1
        goal.reshape(B, -1)[np.arange(B), H * W - 1 - 7 * np.arange(B)] = 1
    cost = np.random.RandomState(H * W).rand(B, 1, H, W).astype(np.float32)
    want = _assert_equal_oracle(cost, start, goal, obst, 0.5)
    assert (want[2] == 0).all()


def test_global_slots_reused_by_many_maps():
    """More maps than resident CTAs on the global-workspace path (an odd side), so every slot serves several maps and
    stale state from an earlier map would show."""
    from c5_data import c5_maps

    obst, start, goal = c5_maps(1500, 45, 45, seed=1500, min_cheb=10)
    cost = np.random.RandomState(1500).rand(1500, 1, 45, 45).astype(np.float32)
    _assert_equal_oracle(cost, start, goal, obst, 0.5)
    _assert_equal_oracle(obst, start, goal, obst, 0.7)


def test_mixed_batch_solved_unreachable_start_is_goal():
    rng = np.random.RandomState(5)
    B, H, W = 24, 48, 40
    obst = (rng.rand(B, 1, H, W) > 0.2).astype(np.float32)
    start = np.zeros_like(obst)
    goal = np.zeros_like(obst)
    start[:, 0, 1, 1] = 1
    goal[:, 0, -2, -2] = 1
    obst[:, 0, 1, 1] = obst[:, 0, -2, -2] = 1
    obst[0::3, 0, :, W // 2] = 0            # a wall: unreachable
    goal[1::3] = start[1::3]                 # start == goal
    cost = rng.rand(B, 1, H, W).astype(np.float32)
    want = _assert_equal_oracle(cost, start, goal, obst, 0.5)
    assert set(want[2][0::3]) == {1} and set(want[2][1::3]) == {0} and (want[3][1::3] == 1).all()
    assert not want[0][0::3].any() and not want[1][0::3].any()


def _fixture():
    maps = torch.ones((8, 1, 64, 64))
    maps[:, :, 24:48, 24:48] = 0
    start = torch.zeros((8, 1, 64, 64))
    start[:, :, 0, 0] = 1
    goal = torch.zeros((8, 1, 64, 64))
    goal[:, :, -1, -1] = 1
    return maps, start, goal


def test_reference_fixture_equals_differentiable_search():
    """The reference's own test_pq_astar assertion (tests/astar_test.py:33-42), with its heap semantics."""
    from neural_astar.planner import VanillaAstar

    maps, start, goal = _fixture()
    out = VanillaAstar().cuda()(maps.cuda(), start.cuda(), goal.cuda())
    out_pq = VanillaAstar(use_differentiable_astar=False, pq_semantics="reference")(maps, start, goal)
    assert not out_pq.histories.is_cuda and out_pq.histories.dtype == torch.float32
    assert out_pq.paths.dtype == torch.int64
    assert torch.equal(out.histories.cpu(), out_pq.histories) and torch.equal(out.paths.cpu(), out_pq.paths)
    g = Golden("fixture64_vanilla")
    np.testing.assert_array_equal(out_pq.histories[:2].numpy(), g.bits("hist_bits"))
    np.testing.assert_array_equal(out_pq.paths[:2].numpy(), g.bits("path_bits"))
    assert int(out_pq.histories[0].sum()) == 1169 and int(out_pq.paths[0].sum()) == 88


def test_invalid_start_or_goal_raises():
    from neural_astar.planner.pq_astar import pq_astar

    maps, start, goal = _fixture()
    start[3, 0, 5, 5] = 1
    goal[6] = 0
    with pytest.raises(ValueError, match=r"\[3, 6\]"):
        pq_astar(maps, start, goal, maps, semantics="reference")


def test_devices_and_dtypes():
    from neural_astar.planner.pq_astar import pq_astar

    maps, start, goal = _fixture()
    ref = pq_astar(maps, start, goal, maps, semantics="reference")
    out = pq_astar(maps.cuda(), start.cuda(), goal.cuda(), maps.cuda(), semantics="reference")
    assert out.histories.is_cuda and out.paths.is_cuda and out.paths.dtype == torch.int64
    assert torch.equal(out.histories.cpu(), ref.histories) and torch.equal(out.paths.cpu(), ref.paths)
    o64 = pq_astar(maps.double(), start.double(), goal.double(), maps.double(), semantics="reference")
    assert o64.histories.dtype == torch.float64 and o64.paths.dtype == torch.int64 and not o64.histories.is_cuda
    assert torch.equal(o64.histories.float(), ref.histories)
    m2 = torch.cat((maps, maps), 1)   # channel 0 is searched; the outputs have the goal maps' shape
    o2 = pq_astar(m2, torch.cat((start, start), 1), torch.cat((goal, goal), 1), m2, semantics="reference")
    assert o2.histories.shape == (8, 2, 64, 64) and not o2.histories[:, 1].any() and not o2.paths[:, 1].any()
    assert torch.equal(o2.histories[:, :1], ref.histories) and torch.equal(o2.paths[:, :1], ref.paths)


def test_one_launch_per_call():
    from neural_astar import _native
    from neural_astar.planner.pq_astar import pq_astar

    maps, start, goal = (t.cuda() for t in _fixture())
    for side in (64, 128):   # shared-memory and global-workspace state
        m = torch.nn.functional.pad(maps, (0, side - 64, 0, side - 64), value=1.0)
        s = torch.nn.functional.pad(start, (0, side - 64, 0, side - 64))
        g = torch.nn.functional.pad(goal, (0, side - 64, 0, side - 64))
        pq_astar(m, s, g, m, semantics="reference")
        torch.cuda.synchronize()
        before = _native.launch_count()
        pq_astar(m, s, g, m, semantics="reference")
        assert _native.launch_count() - before == 1
