"""The backward of every engine (1, 4, 2, 3) cell by cell against the oracle's fp64 closed form, within the rounding
bound M (tests/grad_bound.py, oracle/astar_oracle.c nastar_oracle_backward_bound), where incremental sums drift:

  * S growing: at g_ratio 0 and 0.2 f falls as the search nears the goal, so S = sum exp(-f / sqrt(W)) grows by up to
    e^45 over a corner-to-corner search 2 048 wide, and the prefix sums A = sum 1/S, B = sum D/S^2 are dominated by
    their early terms (the engines rebase them, nastar_common.cuh bwd_rebase);
  * S decaying: exhaustive searches (unreachable goals, cost x 10) that resum S and D many times;
  * mixed magnitudes: one map's upstream gradient 1e-6 of the other's in one batch;
  * large x = f / sqrt(W): open numerators near the bottom of fp32's normal range and in its subnormal range;
  * every open numerator underflowing at one step: the map's gradient is NaN on every engine (DESIGN.md section 8);
  * boundaries: g_ratio 0.49 / 0.5 / 0.51, T_batch 1 and 2, start == goal, the goal clamp, the step cap.

The same search reaches several engines by padding a map with rows of obstacles, which changes neither the search nor
its gradient.  Each case prints its GPU and oracle time.
"""
import time

import numpy as np
import pytest
import torch

from grad_bound import assert_within_bound, open_x_range
from oracle import oracle
from test_engine_limits_cpu import engine_for

pytestmark = pytest.mark.gpu
CLOCK = {"gpu": 0.0, "oracle": 0.0}


@pytest.fixture(scope="module")
def native():
    from neural_astar import _native

    _native.lib()
    yield _native
    print(f"\ntest_gpu_backward_bound: gpu {CLOCK['gpu']:.2f} s, oracle {CLOCK['oracle']:.2f} s")


def _dev(x):
    return torch.from_numpy(np.ascontiguousarray(x)).cuda()


def _timed(key, fn):
    if key == "gpu":
        torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = fn()
    if key == "gpu":
        torch.cuda.synchronize()
    CLOCK[key] += time.perf_counter() - t0
    return out, time.perf_counter() - t0


def _gpu_grad(native, planes, G, g_ratio, T, mechanism="moore", T_batch=None):
    """forward (early exit), then the backward for the forward's T_batch or a given one; (grad, T_batch, t_solve)"""
    def run():
        dev = [_dev(x) for x in planes]
        hist, paths, ts, ns, _ = native.forward(*dev, g_ratio, T, mechanism=mechanism)
        Tb = native.batch_steps(ts, ns, T) if T_batch is None else torch.full((1,), T_batch, dtype=torch.int32,
                                                                               device="cuda")
        gc = native.backward(*dev, _dev(G), Tb, ts, g_ratio, mechanism=mechanism)
        return gc.cpu().numpy(), int(Tb.item()), ts.cpu().numpy()
    out, _ = _timed("gpu", run)
    return out


def _check(native, planes, G, g_ratio, T, what, mechanism="moore", T_batch=None, engine=None):
    """The engine's gradient within M of the oracle's on every cell; returns (worst ratio, T_batch, t_solve)."""
    H, W = planes[0].shape[-2:]
    if engine is not None:
        assert engine_for(H, W) == engine, (H, W)
    gc, Tb, ts = _gpu_grad(native, planes, G, g_ratio, T, mechanism, T_batch)
    (want, M), t_or = _timed("oracle", lambda: oracle.backward_with_bound(*planes, G, Tb, g_ratio=g_ratio,
                                                                         mechanism=mechanism))
    worst = assert_within_bound(gc, want, M, what, mechanism=mechanism)
    print(f"{what}: {H}x{W} engine {engine_for(H, W)} T_batch {Tb} t_solve {ts.tolist()[:4]}: worst {worst:.3g}, "
          f"oracle {t_or:.2f} s")
    return worst, Tb, ts


def _corner(rng, H, W, p_obst, cost_lo=0.1, cost_hi=1.0):
    """One map, start at the top-left corner, goal at the bottom-right, learned-style costs."""
    obst = (rng.rand(1, 1, H, W) > p_obst).astype(np.float32)
    start = np.zeros_like(obst)
    goal = np.zeros_like(obst)
    obst[0, 0, 0, 0] = obst[0, 0, -1, -1] = 1
    start[0, 0, 0, 0] = goal[0, 0, -1, -1] = 1
    cost = rng.uniform(cost_lo, cost_hi, obst.shape).astype(np.float32)
    return cost, start, goal, obst


def _pad_rows(planes, G, H2):
    """The planes with rows of obstacles (zero cost, start, goal and upstream gradient) added below, up to H2 rows."""
    def pad(x):
        out = np.zeros(x.shape[:2] + (H2, x.shape[3]), np.float32)
        out[:, :, :x.shape[2]] = x
        return out
    return tuple(pad(x) for x in planes), pad(G)


# -------------------------------------------------------------------------------------------------------- S growing
GROWING = [(32, 32, 1), (64, 64, 4), (16, 128, 2), (16, 256, 2), (16, 512, 2), (16, 1024, 2), (16, 2048, 3)]


@pytest.mark.parametrize("g_ratio", [0.0, 0.2])
@pytest.mark.parametrize("p_obst", [0.0, 0.1], ids=["open", "sparse"])
@pytest.mark.parametrize("H,W,engine", GROWING, ids=[f"{h}x{w}" for h, w, _ in GROWING])
def test_s_growing_corner_to_corner(native, H, W, engine, p_obst, g_ratio):
    """Corner to corner with learned costs at low g_ratio: f falls by about 0.7 (g_ratio 0.2) or 1 (g_ratio 0) per
    step, so the last steps' S is e^(0.7 W / sqrt(W)) times the first's.  Solved within T = W * W."""
    rng = np.random.RandomState(H * 31 + W + int(10 * g_ratio) + int(100 * p_obst))
    planes = _corner(rng, H, W, p_obst)
    planes[3][0, 0, 0, :] = planes[3][0, 0, :, -1] = 1   # the top row and the right column stay open: solvable
    G = rng.randn(*planes[0].shape).astype(np.float32)
    _, Tb, ts = _check(native, planes, G, g_ratio, W * W, f"growing gr={g_ratio} p={p_obst}", engine=engine)
    assert (ts >= 0).all() and Tb >= W - 1


# -------------------------------------------------------------------------------------------------------- S decaying
DECAYING = [(64, 64, 4), (128, 128, 2), (131, 132, 3)]


@pytest.mark.parametrize("H,W,engine", DECAYING, ids=[f"{h}x{w}" for h, w, _ in DECAYING])
def test_s_decaying_exhaustive_search(native, H, W, engine):
    """The goal walled in, costs x 10: the search closes every reachable cell (t_solve -2) while S shrinks by many
    orders of magnitude, which makes the engines resum S and D again and again."""
    rng = np.random.RandomState(H + 7 * W)
    cost, start, goal, obst = _corner(rng, H, W, 0.15)
    cost *= np.float32(10.0)
    obst[0, 0, -3:, -3:] = 0
    obst[0, 0, -1, -1] = 1
    G = rng.randn(*cost.shape).astype(np.float32)
    planes = (cost, start, goal, obst)
    _, _, ts = _check(native, planes, G, 0.5, W * W, "decaying", engine=engine)
    assert ts.tolist() == [-2]


# ----------------------------------------------------------------------------------------------- mixed magnitudes
@pytest.mark.parametrize("H,W,engine", [(32, 32, 1), (64, 64, 4), (100, 72, 2), (131, 132, 3)])
def test_mixed_magnitudes_in_one_batch(native, H, W, engine):
    """Two maps whose upstream gradients differ by 1e-6: the small map is held to its own M, not the batch's."""
    rng = np.random.RandomState(H * 5 + W)
    maps = [_corner(rng, H, W, 0.15) for _ in range(2)]
    planes = tuple(np.concatenate(x) for x in zip(*maps))
    G = rng.randn(*planes[0].shape).astype(np.float32)
    G[1] *= np.float32(1e-6)
    _check(native, planes, G, 0.5, W * W, "mixed 1e-6", engine=engine)


# ---------------------------------------------------------------------------------------------------------- large x
ENGINE_ROWS = {1: 16, 4: 48, 2: 100, 3: 4000}   # 16 columns: the rows that take each engine


def _large_x_problem(seed, wall_cost):
    """16 x 16, costs uniform(0.1, 1) with 30 % of the cells costing `wall_cost`: those cells' f / sqrt(W) is large
    once opened, while the cheap cells the search selects keep exp(-f / sqrt(W)) normal."""
    rng = np.random.RandomState(seed)
    cost, start, goal, obst = _corner(rng, 16, 16, 0.0)
    walls = rng.rand(*cost.shape) < 0.3
    walls[0, 0, 0, 0] = walls[0, 0, -1, -1] = False
    cost[walls] = np.float32(wall_cost)
    G = rng.randn(*cost.shape).astype(np.float32)
    return (cost, start, goal, obst), G


@pytest.mark.parametrize("target,wall_cost", [(40, 300.0), (80, 620.0), (86, 668.0), (100, 780.0)],
                         ids=["x40", "x80", "x86", "subnormal"])
def test_large_x_on_every_engine(native, target, wall_cost):
    """The largest open x = f / sqrt(W) near 40, 80 and 86 (the bottom of fp32's normal range is 87.3), and in 88..103
    where the open numerators are subnormal, while the selected cell's stays normal.  The same search on engines 1, 4,
    2 and 3 (rows of obstacles below), each within M."""
    planes, G = _large_x_problem(7, wall_cost)
    T = 256
    ref = oracle.forward(*planes, mode="spec", T=T)
    x_max, x_min = open_x_range(*planes, 0.5, int(ref.n_steps.max()))
    print(f"large x {target}: open x up to {x_max:.1f}, smallest open x at most {x_min:.1f}")
    assert abs(x_max - target) < 4 and x_min < 87
    for engine, H2 in ENGINE_ROWS.items():
        p2, G2 = _pad_rows(planes, G, H2)
        _check(native, p2, G2, 0.5, T, f"large x {target}", engine=engine)


# ------------------------------------------------------------------------------------------- every open v underflows
def test_all_open_numerators_underflow_gives_nan_on_every_engine(native):
    """Costs of 900 on a 16-wide map: the start's x = f / sqrt(W) is about 114, so exp(-x) is 0 in fp32 and S is 0 at
    the first step.  The reference's own softmax is 0/0 there.  Every engine writes NaN on every cell of that map and
    leaves the other map of the batch within M."""
    rng = np.random.RandomState(11)
    bad = _corner(rng, 16, 16, 0.0, 900.0, 900.0)
    good = _corner(rng, 16, 16, 0.1)
    planes = tuple(np.concatenate(x) for x in zip(bad, good))
    G = rng.randn(*planes[0].shape).astype(np.float32)
    x_max, x_min = open_x_range(*bad, 0.5, 1)
    assert x_min > 103.3, x_min
    for engine, H2 in ENGINE_ROWS.items():
        p2, G2 = _pad_rows(planes, G, H2)
        assert engine_for(H2, 16) == engine
        gc, Tb, ts = _gpu_grad(native, p2, G2, 0.5, 256)
        assert np.isnan(gc[0]).all(), engine
        want, M = oracle.backward_with_bound(*(x[1:] for x in p2), G2[1:], Tb, g_ratio=0.5)
        assert_within_bound(gc[1:], want, M, ("beside the NaN map", engine))


# ------------------------------------------------------------------------------------------------------- boundaries
@pytest.mark.parametrize("g_ratio", [0.49, 0.5, 0.51])
@pytest.mark.parametrize("H,W,engine", [(32, 32, 1), (64, 64, 4), (100, 72, 2), (131, 132, 3)])
def test_g_ratio_either_side_of_the_fold(native, H, W, engine, g_ratio):
    """Through DifferentiableAstar, a batch of a short and a long search: the short map's post-solve steps are folded
    analytically at 0.5 and above and replayed one by one below (the batch-coupled stop), and its goal is clamped.
    Against the oracle run for the LITERAL form's T_batch."""
    from neural_astar.planner.differentiable_astar import DifferentiableAstar

    assert engine_for(H, W) == engine
    rng = np.random.RandomState(H + W + int(100 * g_ratio))
    long_map = _corner(rng, H, W, 0.15)
    short_map = tuple(x.copy() for x in _corner(rng, H, W, 0.15))
    short_map[2][:] = 0
    short_map[2][0, 0, 2, 2] = short_map[3][0, 0, 2, 2] = 1
    planes = tuple(np.concatenate(x) for x in zip(short_map, long_map))
    G = rng.randn(*planes[0].shape).astype(np.float32)
    lit = oracle.forward(*planes, g_ratio=g_ratio, mode="literal", T=W * W)
    assert lit.t_solve[0] >= 0 and lit.t_solve[0] + 1 < lit.T_batch
    astar = DifferentiableAstar(g_ratio=g_ratio).cuda().eval()

    def run():
        c = _dev(planes[0]).requires_grad_(True)
        out = astar(c, *(_dev(x) for x in planes[1:]))
        (out.histories * _dev(G)).sum().backward()
        return out.histories.detach().cpu().numpy(), c.grad.cpu().numpy()
    (hist, gc), _ = _timed("gpu", run)
    np.testing.assert_array_equal(hist, lit.histories)
    (want, M), t_or = _timed("oracle", lambda: oracle.backward_with_bound(*planes, G, lit.T_batch, g_ratio=g_ratio))
    worst = assert_within_bound(gc, want, M, ("fold", g_ratio))
    print(f"fold gr={g_ratio}: {H}x{W} T_batch {lit.T_batch}: worst {worst:.3g}, oracle {t_or:.2f} s")


@pytest.mark.parametrize("H,W,engine", [(32, 32, 1), (64, 64, 4), (100, 72, 2), (131, 132, 3)])
def test_short_and_edge_batches(native, H, W, engine):
    """T_batch 1 and 2; start == goal; the goal clamped (solved long before T_batch); the step cap."""
    rng = np.random.RandomState(3 * H + W)
    planes = _corner(rng, H, W, 0.15)
    G = rng.randn(*planes[0].shape).astype(np.float32)
    for Tb in (1, 2):
        _check(native, planes, G, 0.5, W * W, f"T_batch {Tb}", T_batch=Tb, engine=engine)
    same = tuple(x.copy() for x in planes)
    same[2][:] = same[1]
    _, _, ts = _check(native, same, G, 0.5, W * W, "start == goal", T_batch=10, engine=engine)
    assert ts.tolist() == [0]
    ref = oracle.forward(*planes, mode="spec", T=W * W)
    _check(native, planes, G, 0.5, W * W, "clamped goal", T_batch=int(ref.t_solve[0]) + 50, engine=engine)
    _, Tb, ts = _check(native, planes, G, 0.5, W // 2, "step cap", engine=engine)
    assert ts.tolist() == [-1] and Tb == W // 2
