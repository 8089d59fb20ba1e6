"""The oracle's rounding bound M (oracle/astar_oracle.c, nastar_oracle_backward_bound) checked on the CPU.

The oracle's model mode rounds the softmax numerators as the engines do, v = expf(fl32(-f / sqrt(W))) in fp32, and
keeps everything else in fp64.  On a matrix of shapes, g_ratio, cost scales and both mechanisms, including open
numerators deep in fp32's subnormal range, |model - want| <= M on every cell, and the worst ratio stays above a floor,
so that M is not vacuous.  Mutations that max|got - want| / max|want| < 1e-5 over a batch lets through must fall
outside M.
"""
import numpy as np
import pytest

from grad_bound import assert_within_bound, open_x_range, relerr_to_max

WORST_FLOOR = 0.1   # the matrix's worst ratio measured 0.63 (12 x 12, walls of 500); M 6x looser would fail here


def _corner(rng, B, H, W, p_obst, cost_scale=1.0, wall_cost=None):
    """B maps, start top-left and goal bottom-right, learned-style costs x cost_scale; with wall_cost, 30 % of the cells
    off a free band around the diagonal cost that much (their f / sqrt(W) is large once opened, while the search walks
    the band and every step keeps a normal numerator)."""
    obst = (rng.rand(B, 1, H, W) > p_obst).astype(np.float32)
    start = np.zeros_like(obst)
    goal = np.zeros_like(obst)
    obst[:, 0, 0, 0] = obst[:, 0, -1, -1] = 1
    start[:, 0, 0, 0] = goal[:, 0, -1, -1] = 1
    cost = (cost_scale / (1.0 + np.exp(-rng.randn(B, 1, H, W)))).astype(np.float32)
    if wall_cost is not None:
        walls = rng.rand(B, 1, H, W) < 0.3
        ys, xs = np.mgrid[:H, :W]
        band = np.abs(ys * (W - 1) - xs * (H - 1)) <= max(H, W)
        walls[:, 0, band] = False
        obst[:, 0, band] = 1
        cost[walls] = np.float32(wall_cost)
    G = rng.randn(B, 1, H, W).astype(np.float32)
    return (cost, start, goal, obst), G


CASES = [
    # H, W, g_ratio, cost_scale, wall_cost
    (16, 16, 0.5, 1.0, None), (32, 32, 0.5, 1.0, None), (24, 40, 0.8, 1.0, None), (32, 32, 0.2, 1.0, None),
    (40, 40, 0.0, 1.0, None), (64, 64, 0.5, 10.0, None), (31, 29, 0.3, 10.0, None), (8, 200, 0.2, 1.0, None),
    (16, 16, 0.5, 1.0, 620.0), (16, 16, 0.5, 1.0, 780.0), (16, 16, 0.2, 1.0, 900.0), (12, 12, 0.5, 1.0, 500.0),
]
RESULTS = {}


@pytest.mark.parametrize("mechanism", ["moore", "news"])
@pytest.mark.parametrize("H,W,g_ratio,cost_scale,wall_cost", CASES)
def test_engine_rounding_model_within_bound(oracle, H, W, g_ratio, cost_scale, wall_cost, mechanism):
    rng = np.random.RandomState(H * 1000 + W + int(100 * g_ratio) + int(cost_scale) + int(wall_cost or 0))
    planes, G = _corner(rng, 3, H, W, 0.15, cost_scale, wall_cost)
    lit = oracle.forward(*planes, g_ratio=g_ratio, mode="literal", T=W * W, mechanism=mechanism)
    Tb = lit.T_batch
    want, M = oracle.backward_with_bound(*planes, G, Tb, g_ratio=g_ratio, mechanism=mechanism)
    model, _ = oracle.backward_with_bound(*planes, G, Tb, g_ratio=g_ratio, mechanism=mechanism, model=True)
    assert np.array_equal(want, oracle.backward(*planes, G, Tb, g_ratio=g_ratio, dtype=np.float64,
                                                mechanism=mechanism))
    x_max, x_min = open_x_range(*planes, g_ratio, Tb, mechanism)
    assert x_min < 103.0
    worst = assert_within_bound(model, want, M, (H, W, g_ratio, cost_scale, wall_cost), mechanism=mechanism,
                                engine="cpu model")
    RESULTS[(H, W, g_ratio, cost_scale, wall_cost, mechanism)] = worst
    print(f"{H}x{W} gr={g_ratio} cost x{cost_scale} walls {wall_cost} {mechanism}: T_batch {Tb}, open x up to "
          f"{x_max:.1f}, worst |model - want| / M = {worst:.3g}")


def test_bound_is_not_vacuous(oracle):
    """Run after the matrix: its worst ratio over every case is above WORST_FLOOR."""
    if len(RESULTS) < 2 * len(CASES):
        for mech in ("moore", "news"):
            for case in CASES:
                if case + (mech,) not in RESULTS:
                    test_engine_rounding_model_within_bound(oracle, *case, mech)
    worst = max(RESULTS.values())
    print(f"worst |model - want| / M over {len(RESULTS)} cases: {worst:.3g}")
    assert worst > WORST_FLOOR


def test_subnormal_numerators_are_covered(oracle):
    """A case of the matrix whose open numerators go below fp32's normal range (x > 87.3) and to zero (x > 103.3)
    while the selected cell's stays normal."""
    for g_ratio, wall_cost, lo, hi in ((0.5, 780.0, 88.0, 103.3), (0.2, 900.0, 103.3, np.inf)):
        rng = np.random.RandomState(16 * 1000 + 16 + int(100 * g_ratio) + 1 + int(wall_cost))
        planes, G = _corner(rng, 3, 16, 16, 0.15, 1.0, wall_cost)
        Tb = oracle.forward(*planes, g_ratio=g_ratio, mode="literal", T=256).T_batch
        x_max, x_min = open_x_range(*planes, g_ratio, Tb)
        assert lo < x_max < hi and x_min < 87


def _old_check(got, want):
    return relerr_to_max(got, want) < 1e-5


def test_mutations_fall_outside_the_bound(oracle):
    """Three wrong gradients, each rejected by M on some cell.  Printed beside each: whether the batch-max check
    max|got - want| / max|want| < 1e-5 accepts it."""
    rng = np.random.RandomState(5)
    table = []

    # the gradient for T_batch - 1 steps: the last step dropped, in a batch where one map solved long before T_batch
    # and re-selects its goal (so its last step moves few cells) and the other is capped
    planes, G = _corner(rng, 2, 32, 32, 0.15)
    planes[2][1] = 0
    planes[2][1, 0, 31, 2] = planes[3][1, 0, 31, 2] = 1
    T = int(oracle.forward(*planes, mode="spec", T=1024).t_solve[0]) + 50
    want, M = oracle.backward_with_bound(*planes, G, T)
    got, _ = oracle.backward_with_bound(*planes, G, T - 1, model=True)
    table.append(("T_batch - 1", got, want, M))

    # the goal clamp flipped: a map solved at its last step (not clamped) treated as clamped, G at the goal zeroed
    planes, G = _corner(rng, 1, 32, 32, 0.15)
    Tb = int(oracle.forward(*planes, mode="spec", T=1024).t_solve[0]) + 1
    want, M = oracle.backward_with_bound(*planes, G, Tb)
    G2 = G.copy()
    G2[0, 0, -1, -1] = 0
    got, _ = oracle.backward_with_bound(*planes, G2, Tb, model=True)
    table.append(("goal clamp flipped", got, want, M))

    # one map of a batch with its upstream gradient x 1e-6, its engine gradient then perturbed by 1 %
    planes, G = _corner(rng, 2, 32, 32, 0.15)
    G[1] *= np.float32(1e-6)
    want, M = oracle.backward_with_bound(*planes, G, 1024)
    got, _ = oracle.backward_with_bound(*planes, G, 1024, model=True)
    got[1] *= 1.01
    table.append(("small map x 1.01", got, want, M))

    print("\nmutation              old check     worst |got - want| / M")
    for name, got, want, M in table:
        old = _old_check(got, want)
        worst = float((np.abs(got - want) / M).max())
        print(f"{name:<20}  {'accepts' if old else 'rejects':<12}  {worst:.3g}")
        assert worst > 1.0, name
