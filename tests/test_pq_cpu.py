"""CPU checks of the reference heap A* (pq_astar, use_differentiable_astar=False, pq_semantics="reference"):
the pqdict shim against heapq, the C oracle against the goldens and the staged reference, the C ABI's rejections and
the planners' keyword validation."""
import ctypes
import heapq
import os
import random
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import pq as pq_oracle  # noqa: E402

import pq_golden  # noqa: E402
from pqdict_shim import pqdict  # noqa: E402

EINVAL, EUNSUPPORTED, EWORKSPACE = 1, 2, 4


class _Item:
    """Compares by priority only, like heapq's entries would without a tie-breaker."""

    def __init__(self, key, prio):
        self.key, self.prio = key, prio

    def __lt__(self, other):
        return self.prio < other.prio


@pytest.mark.parametrize("seed", range(6))
def test_shim_heap_moves_equal_heapq(seed):
    rng = random.Random(seed)
    q, h = pqdict(), []
    next_key = 0
    for _ in range(3000):
        op = rng.random()
        if op < 0.45 or not h:
            prio = rng.randint(0, 6)   # few values: many equal priorities
            q.additem(next_key, prio)
            heapq.heappush(h, _Item(next_key, prio))
            next_key += 1
        elif op < 0.8:
            k, v = q.popitem()
            it = heapq.heappop(h)
            assert (k, v) == (it.key, it.prio)
        else:
            pos = rng.randrange(len(h))
            it = h[pos]
            new = it.prio - rng.randint(0, 3)   # a lowered or equal key, as the reference only lowers keys
            it.prio = new
            heapq._siftdown(h, 0, pos)
            q[it.key] = new
        assert [n.key for n in q._heap] == [it.key for it in h]
        assert len(q) == len(h) and all(q[it.key] == it.prio and it.key in q for it in h)


@pytest.mark.parametrize("name", pq_golden.NAMES)
def test_oracle_equals_golden(name):
    g = pq_golden.PqGolden(name)
    hist, paths, status, exp = pq_oracle.pq_astar(g.cost, g.start, g.goal, g.obst, g.g_ratio)
    eh, ep, es, ee = g.expected
    np.testing.assert_array_equal(status, es)
    np.testing.assert_array_equal(hist, eh)
    np.testing.assert_array_equal(paths, ep)
    solved = es == 0
    np.testing.assert_array_equal(exp[solved], ee[solved])


def test_golden_set_covers_the_cases():
    assert {"fixture64", "mazes032_ckpt_g05", "mazes032_ckpt_g02", "mazes032_ckpt_g08", "ties32_g10", "ties32_g00",
            "ties32_costs", "edge32", "line1x40", "line40x1", "large128", "large256"} <= set(pq_golden.NAMES)
    fx = pq_golden.PqGolden("fixture64")
    eh, ep, es, ee = fx.expected
    assert list(ee) == [1169, 1169] and list(ep.sum((1, 2, 3))) == [88, 88]
    assert list(pq_golden.PqGolden("edge32").z["status"]) == [0, 1, 0, 1, 0, 0, 0]


def _random_maps(rng, B, H, W, quantised):
    obst = (rng.rand(B, 1, H, W) > rng.uniform(0.05, 0.4)).astype(np.float32)
    s, t = rng.randint(0, H * W, B), rng.randint(0, H * W, B)
    start = np.zeros((B, 1, H * W), np.float32)
    goal = np.zeros((B, 1, H * W), np.float32)
    start[np.arange(B), 0, s] = 1
    goal[np.arange(B), 0, t] = 1
    obst.reshape(B, -1)[np.arange(B), t] = 1
    cost = rng.rand(B, 1, H, W).astype(np.float32)
    if quantised:
        cost = np.round(cost * 4) / 4
    return cost, start.reshape(B, 1, H, W), goal.reshape(B, 1, H, W), obst


@pytest.mark.parametrize("seed,H,W,g_ratio", [(0, 16, 16, 0.5), (1, 24, 17, 0.3), (2, 9, 30, 0.9), (3, 20, 20, 1.0),
                                              (4, 20, 20, 0.0)])
def test_oracle_equals_staged_reference(seed, H, W, g_ratio):
    solve = pq_golden.staged_solve_single()
    if solve is None:
        pytest.skip("the reference is not staged in oracle/_ref/")
    rng = np.random.RandomState(1000 + seed)
    cost, start, goal, obst = _random_maps(rng, 12, H, W, quantised=seed % 2 == 1)
    hist, paths, status, _ = pq_oracle.pq_astar(cost, start, goal, obst, g_ratio)
    import contextlib
    import io

    for b in range(len(cost)):
        with contextlib.redirect_stdout(io.StringIO()):
            rh, rp = solve(cost[b, 0].astype(np.float64), start[b, 0], goal[b, 0], obst[b, 0], g_ratio)
        np.testing.assert_array_equal(hist[b, 0], rh)
        np.testing.assert_array_equal(paths[b, 0], rp)
        assert status[b] == (0 if rh.any() else 1)


def test_oracle_status_two_for_bad_ends():
    cost = np.ones((3, 1, 8, 8), np.float32)
    start = np.zeros_like(cost)
    goal = np.zeros_like(cost)
    start[:, 0, 0, 0] = 1
    goal[:, 0, 7, 7] = 1
    start[1, 0, 3, 3] = 1      # two starts
    goal[2] = 0                # no goal
    hist, paths, status, _ = pq_oracle.pq_astar(cost, start, goal, cost, 0.5)
    assert list(status) == [0, 2, 2]
    assert not hist[1:].any() and not paths[1:].any()


# ---- C ABI ----------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def native():
    subprocess.check_call(["make", "-C", os.path.join(ROOT, "neural-astar_b200"), "-s", "all"])
    from neural_astar import _native

    return _native


def _call(native, **kw):
    a = dict(cost=0x10000, cs=32 * 32, start=0x20000, ss=32 * 32, goal=0x30000, gs=32 * 32, map=0x40000, ms=32 * 32,
             B=4, H=32, W=32, g=0.5, hist=0x50000, paths=0x60000, status=0x70000, exp=0x80000, ws=0x90000,
             ws_bytes=1 << 20)
    a.update(kw)
    return native.lib().nastar_b200_pq_astar(a["cost"], a["cs"], a["start"], a["ss"], a["goal"], a["gs"], a["map"],
                                             a["ms"], a["B"], a["H"], a["W"], a["g"], a["hist"], a["paths"],
                                             a["status"], a["exp"], a["ws"], a["ws_bytes"], None)


@pytest.mark.parametrize("kw,status", [
    (dict(cost=0), EINVAL), (dict(start=0), EINVAL), (dict(goal=0), EINVAL), (dict(map=0), EINVAL),
    (dict(hist=0), EINVAL), (dict(paths=0), EINVAL), (dict(status=0), EINVAL), (dict(exp=0), EINVAL),
    (dict(B=0), EINVAL), (dict(H=0), EINVAL), (dict(W=-1), EINVAL),
    (dict(cs=32 * 31), EINVAL), (dict(ms=0), EINVAL),
    (dict(H=1025, W=1024, cs=1 << 21, ss=1 << 21, gs=1 << 21, ms=1 << 21), EUNSUPPORTED),
    (dict(ws=0x90004), EINVAL),   # the workspace slots hold fp64 arrays
    (dict(ws=0), EWORKSPACE), (dict(ws_bytes=255), EWORKSPACE),
    (dict(H=256, W=256, cs=1 << 16, ss=1 << 16, gs=1 << 16, ms=1 << 16, ws_bytes=1 << 20), EWORKSPACE),
])
def test_pq_abi_rejects_without_launch(native, kw, status):
    L = native.lib()
    before = L.nastar_b200_launch_count()
    assert _call(native, **kw) == status
    assert L.nastar_b200_launch_count() == before, "a rejected call launched something"


def test_pq_workspace_bytes(native):
    L = native.lib()
    assert L.nastar_b200_pq_astar_workspace_bytes(0, 32, 32) == 0
    assert L.nastar_b200_pq_astar_workspace_bytes(4, 1025, 1024) == 0
    assert L.nastar_b200_pq_astar_workspace_bytes(1000, 32, 32) == 256      # state in shared memory
    one = L.nastar_b200_pq_astar_workspace_bytes(1, 256, 256)
    many = L.nastar_b200_pq_astar_workspace_bytes(100000, 256, 256)
    assert one == 256 + 20 * 65536
    assert many < 3 << 30   # sized to the resident CTAs, not to B
    assert L.nastar_b200_pq_astar_workspace_bytes(100000, 1024, 1024) <= 256 + max(2 << 30, 132 * 20 << 20)


# ---- planners ---------------------------------------------------------------------------------------------------------
def test_planner_pq_semantics_keyword():
    from neural_astar.planner import NeuralAstar, VanillaAstar

    for cls in (VanillaAstar, NeuralAstar):
        assert cls(use_differentiable_astar=False).pq_semantics == "engine"
        assert cls(use_differentiable_astar=False, pq_semantics="reference").pq_semantics == "reference"
        assert cls().pq_semantics == "engine"
        with pytest.raises(ValueError):
            cls(use_differentiable_astar=False, pq_semantics="exact")
        with pytest.raises(ValueError):
            cls(pq_semantics="reference")   # the differentiable search has no heap semantics
        with pytest.raises(NotImplementedError):
            cls(use_differentiable_astar=False, mechanism="news", pq_semantics="reference")
    with pytest.raises(TypeError):
        VanillaAstar(0.5, False, "reference")
    with pytest.raises(TypeError):
        NeuralAstar(0.5, 1.0, "m+", "CNN", 4, False, None, False, "reference")


def test_pq_astar_function_semantics_validation():
    import torch

    from neural_astar.planner.pq_astar import pq_astar

    x = torch.zeros(1, 1, 4, 4)
    with pytest.raises(ValueError):
        pq_astar(x, x, x, x, semantics="exact")
    with pytest.raises(AssertionError):
        pq_astar(x, x, x, x, True, semantics="reference")
    with pytest.raises(TypeError):
        pq_astar(x, x, x, x, False, 0.5, "reference")
