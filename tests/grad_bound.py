"""Cell-by-cell check of an engine's backward against the oracle's fp64 closed form, within the oracle's rounding bound.

`oracle.backward_with_bound` returns the fp64 gradient `want` and, per cell, the bound M on |engine - want| that the
fp32 rounding of the softmax numerators allows (derivation in oracle/astar_oracle.c, nastar_oracle_backward_bound).
Unlike max|got - want| / max|want| over a batch, the check sees a map of small gradients beside one of large gradients
and the cells whose gradients are far below the batch's largest.

Every check records its worst |got - want| / M under (engine, mechanism); the table is printed when the test process
ends.
"""
import atexit

import numpy as np

WORST = {}   # (engine, mechanism) -> [worst ratio, checks, cells]


def relerr_to_max(a, b) -> float:
    """max|a - b| / max|b|: for references that are fp32 themselves (the reference's autograd goldens)."""
    return float(np.abs(a - b).max() / (np.abs(b).max() + 1e-30))


def engine_of(H: int, W: int) -> str:
    """The engine the library's backward takes at H x W (nastar_b200_engine_for)."""
    from neural_astar import _native

    return f"engine {int(_native.lib().nastar_b200_engine_for(int(H), int(W)))}"


def assert_within_bound(got, want, M, what, *, mechanism="moore", engine=None) -> float:
    """Assert that every value of `got` is finite and |got - want| <= M on every cell; returns the worst ratio
    |got - want| / M.  got, want and M have one shape ([B,1,H,W]); `engine` defaults to the one the library takes at
    that H x W."""
    got = np.asarray(got, np.float64)
    want = np.asarray(want, np.float64)
    M = np.asarray(M, np.float64)
    assert got.shape == want.shape == M.shape, (got.shape, want.shape, M.shape, what)
    assert np.isfinite(got).all(), ("non-finite gradient", what)
    assert (M > 0).all(), what
    ratio = np.abs(got - want) / M
    worst = float(ratio.max()) if ratio.size else 0.0
    key = (engine if engine is not None else engine_of(*got.shape[-2:]), mechanism)
    rec = WORST.setdefault(key, [0.0, 0, 0])
    rec[0] = max(rec[0], worst)
    rec[1] += 1
    rec[2] += ratio.size
    if worst > 1.0:
        i = np.unravel_index(int(ratio.argmax()), ratio.shape)
        raise AssertionError(f"{what}: |got - want| > M at {tuple(int(k) for k in i)}: got {got[i]!r}, want "
                             f"{want[i]!r}, M {M[i]!r} (ratio {worst:.3g}; {int((ratio > 1).sum())} cells outside)")
    return worst


def report() -> str:
    lines = ["worst |got - want| / M per (engine, mechanism):"]
    for (eng, mech), (worst, n, cells) in sorted(WORST.items()):
        lines.append(f"  {eng:>14} {mech:>5}: {worst:.3g}  ({n} checks, {cells} cells)")
    return "\n".join(lines)


@atexit.register
def _print_report():
    if WORST:
        print("\n" + report())


def open_x_range(cost, start, goal, obst, g_ratio, T_batch, mechanism="moore"):
    """Over the first T_batch steps of every map's backward replay (the goal stays open once selected; no early exit):
    (largest x = f / sqrt(W) of any open cell, largest over steps of the step's smallest open x), in the engines' fp32
    quotient.  The first says how far into fp32's subnormal range the softmax numerators exp(-x) go; the second
    whether a step's every numerator underflows (above 103.28 expf returns 0)."""
    from oracle import oracle
    from search_steps import machines

    gr, omg, sqw = oracle.scalars(g_ratio, cost.shape[-1])
    x_max = x_min_max = 0.0
    for m in machines(cost, start, goal, obst, mechanism):
        for _ in range(T_batch):
            ind = m.select(gr, omg)
            if ind < 0:
                break
            x = (-m.f(gr, omg)[m.open]) / sqw
            x_max = max(x_max, float(-x.min()))
            x_min_max = max(x_min_max, float(-x.max()))
            m.close_and_expand(ind)
    return x_max, x_min_max
