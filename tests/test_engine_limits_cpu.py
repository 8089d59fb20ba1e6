"""The largest shapes each search engine takes, asked of the library, and the step bound that has to fit 32 bits.

Engine 5 (nastar_bin16.cuh, binary aliased planes) and the generic engine with its state in HBM (engine 3,
nastar_generic.cuh) are limited by shared memory: 232 448 B of dynamic shared memory per CTA on sm_90 (nastar_api.cu
kMaxDynSmem).  The edges below are found by asking nastar_b200_bin16_supported / nastar_b200_engine_for, checked to be
real edges (one more row or column flips the answer), and checked against the two layouts restated here, so a change of
either layout moves the shapes that tests/test_gpu_engine_limits.py searches along with the edge.

The loop bound T = int(Tmax * W * W) reaches the library and the CPU oracle as a 32-bit int; above 2**31 - 1 ctypes
would truncate it silently into a wrong bound (W = 92 682: 18 532 steps), so both refuse it with a ValueError.
"""
import functools
import os
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MAX_DYN_SMEM = 232448          # nastar_api.cu kMaxDynSmem: the sm_90 opt-in limit per CTA
MAX_STEPS = 2**31 - 1


# ------------------------------------------------------------------------------------------- the library's answer
@functools.lru_cache(maxsize=None)
def _lib():
    subprocess.check_call(["make", "-C", os.path.join(ROOT, "neural-astar_b200"), "-s", "all"])
    from neural_astar import _native

    return _native.lib()


def engine_for(H: int, W: int) -> int:
    return int(_lib().nastar_b200_engine_for(H, W))


def bin16_supported(H: int, W: int) -> bool:
    return _lib().nastar_b200_bin16_supported(H, W) == 1


def _largest(ok, lo: int, hi: int) -> int:
    """The largest x in [lo, hi] with ok(x), for an ok that holds up to some edge and not beyond; ok(lo) must hold."""
    assert ok(lo), lo
    while lo < hi:
        mid = (lo + hi + 1) // 2
        lo, hi = (mid, hi) if ok(mid) else (lo, mid - 1)
    return lo


def bin16_max_h(W: int) -> int:
    """The most rows engine 5 takes at width W."""
    return _largest(lambda h: bin16_supported(h, W), 1, 4096)


def bin16_max_w(H: int) -> int:
    """The widest map engine 5 takes with H rows."""
    return _largest(lambda w: bin16_supported(H, w), 65, 4096)


def generic_max_h(W: int) -> int:
    """The most rows any engine takes at width W: the generic engine's edge wherever these tests ask for one."""
    return _largest(lambda h: engine_for(h, W) != 0, 1, 1 << 20)


# ----------------------------------------------------------------------------------------- the layouts restated
def _a16(n: int) -> int:
    return (n + 15) & ~15


def bin16_layout_ok(H: int, W: int) -> bool:
    """Bin16Layout (nastar_bin16.cuh) and bin16_shape_ok (nastar_api.cu): segment minima (8 B per 32-column segment),
    32 x kRows row keys (kRows = 8 up to 256 rows, else 16), a column per row, g (2 B), parent (1 B) and the closed
    bits per cell, 64 B of barriers; at most 32 segments and 512 rows, not a shape of engines 1 / 4, and a shape the
    generic engine takes too (its redo pass)."""
    Wd, N = (W + 31) // 32, H * W
    if H <= 0 or W <= 0 or (H <= 64 and W <= 64) or generic_layout_engine(H, W) == 0:
        return False
    krows = 8 if H <= 256 else 16
    smem = (_a16(H * Wd * 8) + 32 * krows * 4 + _a16(H * 4) + _a16(N * 2) + _a16(N) + _a16(H * Wd * 4) + 64)
    return Wd <= 32 and H <= 512 and W < 65536 and N < (1 << 30) and smem <= MAX_DYN_SMEM


def generic_layout_engine(H: int, W: int) -> int:
    """GenericLayout (nastar_generic.cuh) and generic_engine_for (nastar_api.cu): three bit planes of H x ceil(W/32)
    words, a row-min cache of 8 B per row and 16 B of barrier always in shared memory; cost, g, f and parent (13 B per
    cell) too when they fit (engine 2), else in the HBM workspace (engine 3); 0 above 2**30 cells or that."""
    if H <= 0 or W <= 0 or H * W > (1 << 30):
        return 0
    Wd = (W + 31) // 32
    common = 12 * H * Wd + 8 * H + 16
    planes = ((H * W + 3) & ~3) * 13
    if common + planes <= MAX_DYN_SMEM:
        return 2
    return 3 if common <= MAX_DYN_SMEM else 0


def _model_engine(H: int, W: int) -> int:
    if H <= 32 and W <= 32:
        return 1
    if H <= 64 and W <= 64:
        return 4
    return generic_layout_engine(H, W)


BIN16_H_AT_W = (1024, 993, 261, 128)
BIN16_W_AT_H = (512, 300, 257)
GENERIC_H_AT_W = (1, 32, 33, 1024, 2048, 46340)


# ------------------------------------------------------------------------------------------------------ edges
@pytest.mark.parametrize("W", BIN16_H_AT_W)
def test_bin16_largest_rows_is_an_edge(W):
    H = bin16_max_h(W)
    assert engine_for(H, W) == 3 and bin16_supported(H, W)
    assert not bin16_supported(H + 1, W) and engine_for(H + 1, W) == 3
    assert bin16_layout_ok(H, W) and not bin16_layout_ok(H + 1, W)


@pytest.mark.parametrize("H", BIN16_W_AT_H)
def test_bin16_largest_width_is_an_edge(H):
    W = bin16_max_w(H)
    assert bin16_supported(H, W) and not bin16_supported(H, W + 1)
    assert engine_for(H, W + 1) == 3
    assert bin16_layout_ok(H, W) and not bin16_layout_ok(H, W + 1)


@pytest.mark.parametrize("W", GENERIC_H_AT_W)
def test_generic_largest_rows_is_an_edge(W):
    H = generic_max_h(W)
    assert engine_for(H, W) == 3 and engine_for(H + 1, W) == 0
    assert generic_layout_engine(H, W) == 3 and generic_layout_engine(H + 1, W) == 0


def test_limits_reach_the_widest_segments_and_rows():
    """The edges exercise what the kernels size by them: engine 5 with 32 segments of a row (W = 1024) and 16 rows
    per lane (H > 256), and the generic engine's bit planes at thousands of words per row."""
    assert (bin16_max_h(1024) > 64) and bin16_max_w(512) >= 128
    assert bin16_max_w(257) > 256 and bin16_max_w(300) > 200
    assert generic_max_h(1024) > 512 and generic_max_h(46340) >= 1
    assert engine_for(1, 46340) == 3 and engine_for(generic_max_h(46340), 46340) == 3


def test_layouts_restated_match_the_library_on_a_sweep():
    """Every shape of a coarse sweep, and the rows around each edge, get the same answer from the restated layouts as
    from the library."""
    rng = np.random.RandomState(0)
    shapes = [(int(h), int(w)) for h, w in zip(rng.randint(1, 1200, 400), rng.randint(1, 2100, 400))]
    shapes += [(h, w) for w in BIN16_H_AT_W for h in range(bin16_max_h(w) - 2, bin16_max_h(w) + 3)]
    shapes += [(h, w) for h in BIN16_W_AT_H for w in range(bin16_max_w(h) - 2, bin16_max_w(h) + 3)]
    shapes += [(h, w) for w in GENERIC_H_AT_W for h in range(generic_max_h(w) - 2, generic_max_h(w) + 3)]
    for H, W in shapes:
        assert engine_for(H, W) == _model_engine(H, W), (H, W)
        assert bin16_supported(H, W) == bin16_layout_ok(H, W), (H, W)


# ------------------------------------------------------------------------------------------------ the step bound
def _strip(W: int):
    plane = np.ones((1, 1, 1, W), np.float32)
    start = np.zeros_like(plane)
    goal = np.zeros_like(plane)
    start[0, 0, 0, 0] = goal[0, 0, 0, -1] = 1
    return plane, start, goal


@pytest.mark.parametrize("W", [46341, 65536, 65537, 92682])
def test_oracle_refuses_a_step_bound_above_int32(oracle, W):
    """The evaluation bound W * W of these widths does not fit a C int: the oracle refuses it, for the forward and
    for the backward's T_batch, instead of searching with the truncated value."""
    plane, start, goal = _strip(W)
    assert W * W > MAX_STEPS
    with pytest.raises(ValueError, match=r"2\*\*31 - 1"):
        oracle.forward(plane, start, goal, plane, mode="spec")
    with pytest.raises(ValueError, match=r"2\*\*31 - 1"):
        oracle.forward(plane, start, goal, plane, mode="literal")
    with pytest.raises(ValueError, match=r"2\*\*31 - 1"):
        oracle.backward(plane, start, goal, plane, np.ones_like(plane), W * W)


def test_oracle_takes_the_largest_bound(oracle):
    """T = 2**31 - 1 itself is taken: a 1 x 40 strip is solved at step W - 1."""
    plane, start, goal = _strip(40)
    out = oracle.forward(plane, start, goal, plane, mode="spec", T=MAX_STEPS)
    assert out.t_solve.tolist() == [39] and out.n_steps.tolist() == [40]


def test_oracle_guard_is_what_refuses(oracle, monkeypatch):
    """Mutation check: with the guard removed, the refusal test fails on the 1 x 92 682 strip, because ctypes
    truncates the bound W * W to 18 532 and the oracle searches with it: the goal at x = W - 1 is reported as not
    found (t_solve -1) after 18 532 steps."""
    W = 92682
    plane, start, goal = _strip(W)
    monkeypatch.setattr(oracle, "check_steps", int)
    with pytest.raises(pytest.fail.Exception):
        test_oracle_refuses_a_step_bound_above_int32(oracle, W)
    out = oracle.forward(plane, start, goal, plane, mode="spec")
    assert out.t_solve.tolist() == [-1] and out.n_steps.tolist() == [18532]


# ------------------------------------------------- the same refusal in the package, before it touches the library
@pytest.mark.parametrize("W", [46341, 92682])
def test_search_refuses_a_step_bound_above_int32(W):
    """DifferentiableAstar, _native.forward / forward_coupled, batch_steps and backward refuse a bound above
    2**31 - 1 with a ValueError; the module's message names the map width.  Raised before the device or the library
    is looked at, so it holds on the host as it does on the GPU (tests/test_gpu_engine_limits.py)."""
    import torch

    from neural_astar import _native
    from neural_astar.planner.differentiable_astar import DifferentiableAstar

    plane, start, goal = (torch.from_numpy(x) for x in _strip(W))
    with pytest.raises(ValueError, match=f"width W = {W}"):
        DifferentiableAstar()(plane, start, goal, plane)
    with pytest.raises(ValueError, match=r"W <= 46340"):
        _native.forward(plane, start, goal, plane, 0.5, W * W)
    with pytest.raises(ValueError, match=r"W <= 46340"):
        _native.forward_coupled(plane, start, goal, plane, 0.3, W * W)
    ts = torch.zeros(1, dtype=torch.int32)
    with pytest.raises(ValueError, match=r"W <= 46340"):
        _native.batch_steps(ts, ts, W * W)
    with pytest.raises(ValueError, match=r"W <= 46340"):
        _native.backward(plane, start, goal, plane, plane, W * W, ts, 0.5)
    # training with a small Tmax brings the bound back under the limit: only the bound is refused, not the width
    assert DifferentiableAstar(Tmax=0.01).train().num_steps(W) <= MAX_STEPS
