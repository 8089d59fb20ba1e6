"""The search engines at the edges of the shapes they accept, against the SPEC oracle (oracle/astar_oracle.c, either
mechanism), and the shapes just outside them.

The edges are asked of the library (tests/test_engine_limits_cpu.py, which checks them against the layouts), so these
shapes follow a layout change:
  * engine 5 (nastar_bin16.cuh): 16 row keys per lane above 256 rows, 32 segments per row at W = 1024, a partial last
    segment at W = 1000, the work queue handing out maps beyond the resident grid, an exhausted open set;
  * engine 3 (nastar_generic.cuh, state in HBM): the largest shared-memory bit planes and row-min cache, with and
    without W % 32 == 0, 11 621 rows, 46 340 columns (the widest map whose bound W * W fits 32 bits), the backward's
    workspace slots at 600 k cells, and the batch-coupled forward;
  * one row or column more: the next engine, or the library's "unsupported" error before any launch;
  * a step bound above 2**31 - 1: a ValueError before any launch.
Every forward is bit-exact (histories, paths, t_solve, n_steps and the per-map counts) and asserts its engine and its
launch count; backwards are within the oracle's rounding bound of its closed form, cell by cell (tests/grad_bound.py).  Each case prints its GPU and oracle time.
"""
import time

import numpy as np
import pytest
import torch

from grad_bound import assert_within_bound
from test_engine_limits_cpu import bin16_max_h, bin16_max_w, bin16_supported, engine_for, generic_max_h

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def native():
    from neural_astar import _native

    _native.lib()
    return _native


def _dev(x):
    return torch.from_numpy(np.ascontiguousarray(x)).cuda()


def _clock(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return out, time.perf_counter() - t0


def _place(obst, b, y, x):
    obst[b, 0, y, x] = 1
    m = np.zeros(obst.shape[2:], np.float32)
    m[y, x] = 1
    return m


def _corner_problem(rng, B, H, W, p_obst):
    """Binary planes with 1 - p_obst passable, start in the top-left quarter and goal in the bottom-right one."""
    obst = (rng.rand(B, 1, H, W) > p_obst).astype(np.float32)
    start = np.zeros_like(obst)
    goal = np.zeros_like(obst)
    for b in range(B):
        start[b, 0] = _place(obst, b, rng.randint(max(1, H // 4)), rng.randint(max(1, W // 4)))
        goal[b, 0] = _place(obst, b, H - 1 - rng.randint(max(1, H // 4)), W - 1 - rng.randint(max(1, W // 4)))
    return obst, start, goal


def _near_problem(rng, B, H, W, p_obst, dist):
    """Start anywhere, goal `dist` cells away along the longer side, joined by an open L-shaped corridor (4- and
    8-connected): a short search on a large map, never one that exhausts it."""
    obst = (rng.rand(B, 1, H, W) > p_obst).astype(np.float32)
    start = np.zeros_like(obst)
    goal = np.zeros_like(obst)
    for b in range(B):
        if W >= H:
            sy, sx = rng.randint(H), rng.randint(W - dist)
            gy, gx = rng.randint(H), sx + dist
        else:
            sy, sx = rng.randint(H - dist), rng.randint(W)
            gy, gx = sy + dist, rng.randint(W)
        obst[b, 0, sy, min(sx, gx):max(sx, gx) + 1] = 1
        obst[b, 0, min(sy, gy):max(sy, gy) + 1, gx] = 1
        start[b, 0] = _place(obst, b, sy, sx)
        goal[b, 0] = _place(obst, b, gy, gx)
    return obst, start, goal


def _search_exact(native, oracle, planes, T, launches, *, aliased=False, g_ratio=0.5, mechanism="moore", label=""):
    """native.forward against the SPEC oracle, bit for bit with the per-map counts, and its launch count.  `aliased`
    passes one device tensor as cost and obstacles (what sends a binary map to engine 5).  Returns the device outputs
    (histories, t_solve, n_steps) and the oracle's output."""
    cost, start, goal, obst = planes
    if aliased:
        c = _dev(obst)
        dev = (c, _dev(start), _dev(goal), c)
    else:
        dev = tuple(_dev(x) for x in planes)
    before = native.launch_count()
    (hist, paths, ts, ns, _, (ncl, plen)), t_gpu = _clock(lambda: native.forward(
        *dev, g_ratio, T, want_counts=True, mechanism=mechanism))
    assert native.launch_count() - before == launches
    t0 = time.perf_counter()
    ref = oracle.forward(cost, start, goal, obst, g_ratio=g_ratio, mode="spec", T=T, mechanism=mechanism)
    print(f"{label} {mechanism} T={T}: gpu {t_gpu:.3f} s, oracle {time.perf_counter() - t0:.2f} s, "
          f"t_solve {ref.t_solve.tolist()[:4]}")
    np.testing.assert_array_equal(ts.cpu().numpy(), ref.t_solve)
    np.testing.assert_array_equal(ns.cpu().numpy(), ref.n_steps)
    np.testing.assert_array_equal(hist.cpu().numpy(), ref.histories)
    np.testing.assert_array_equal(paths.cpu().numpy(), ref.paths)
    np.testing.assert_array_equal(ncl.cpu().numpy(), ref.histories.sum((1, 2, 3)).astype(np.int64))
    np.testing.assert_array_equal(plen.cpu().numpy(), ref.paths.sum((1, 2, 3)))
    return (hist, paths, ts, ns), dev, ref


# ------------------------------------------------------------------------------------------------------ engine 5
BIN16_SHAPES = {
    "512xmaxW": lambda: (512, bin16_max_w(512)),       # 512 x 128: 16 rows per lane, every lane's rows in use
    "257x256": lambda: (257, 256),                      # the first H with kRows = 16
    "257xmaxW": lambda: (257, bin16_max_w(257)),       # 257 x 261: 9 segments, the last one of 5 columns
    "300xmaxW": lambda: (300, bin16_max_w(300)),       # 300 x 224
    "400x160": lambda: (400, 160),
    "maxHx1024": lambda: (bin16_max_h(1024), 1024),    # 66 x 1024: 32 full segments per row
    "maxHx1000": lambda: (bin16_max_h(1000), 1000),    # 68 x 1000: 32 segments, the last one of 8 columns
    "64x1024": lambda: (64, 1024),                      # H <= 64 but W > 64
}


@pytest.mark.parametrize("case", list(BIN16_SHAPES))
def test_bin16_at_its_edges_vs_oracle(native, oracle, case):
    """Binary aliased planes with 25 % obstacles and far starts and goals: engine 5 then its redo pass (two launches),
    bit-exact against the oracle; the same planes passed as separate tensors take the generic engine alone (one
    launch) and give the same bits."""
    H, W = BIN16_SHAPES[case]()
    assert bin16_supported(H, W) and engine_for(H, W) == 3
    rng = np.random.RandomState(H * 7919 + W)
    obst, start, goal = _corner_problem(rng, 2, H, W, p_obst=0.25)
    planes = (obst, start, goal, obst)
    (hist, paths, ts, ns), _, _ = _search_exact(native, oracle, planes, W * W, 2, aliased=True, label=f"{H}x{W} bin16")
    before = native.launch_count()
    h2, p2, ts2, ns2, _ = native.forward(*(_dev(x) for x in planes), 0.5, W * W)
    assert native.launch_count() - before == 1
    for a, b in ((h2, hist), (p2, paths), (ts2, ts), (ns2, ns)):
        assert torch.equal(a, b)


def test_bin16_exhausted_open_set(native, oracle):
    """The goal walled in on a map at engine 5's widest 257-row shape: the open set empties (t_solve -2) and every
    cell reachable from the start, and no other, is closed."""
    from scipy import ndimage

    H, W = 257, bin16_max_w(257)
    assert bin16_supported(H, W) and W * W > H * W
    rng = np.random.RandomState(5)
    obst, start, goal = _corner_problem(rng, 1, H, W, p_obst=0.3)
    gy, gx = np.argwhere(goal[0, 0])[0]
    obst[0, 0, gy - 1:gy + 2, gx - 1:gx + 2] = 0
    obst[0, 0, gy, gx] = 1
    (hist, _, ts, _), _, ref = _search_exact(native, oracle, (obst, start, goal, obst), W * W, 2, aliased=True,
                                             label="walled bin16")
    assert ref.t_solve.tolist() == [-2]
    labels, _ = ndimage.label(obst[0, 0] > 0, structure=np.ones((3, 3)))
    sy, sx = np.argwhere(start[0, 0])[0]
    np.testing.assert_array_equal(hist.cpu().numpy()[0, 0], (labels == labels[sy, sx]).astype(np.float32))


def test_bin16_queue_hands_out_later_maps_at_512_rows(native, oracle):
    """B = 2 x SMs + 3 maps at 512 x 128, where one CTA per SM is resident: the work queue hands out the maps beyond
    the grid.  Short problems (start and goal about 20 cells apart) keep the oracle cheap."""
    H, W = 512, bin16_max_w(512)
    L = native.lib()
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    B = 2 * sms + 3
    rng = np.random.RandomState(17)
    obst, start, goal = _near_problem(rng, B, H, W, 0.25, 20)
    assert L.nastar_b200_bin16_supported(H, W) == 1
    _search_exact(native, oracle, (obst, start, goal, obst), W * W, 2, aliased=True, label=f"queue B={B}")


OUTSIDE_BIN16 = {
    "512xmaxW+1": lambda: (512, bin16_max_w(512) + 1),   # 512 x 129
    "513x64": lambda: (513, 64),                         # more than 512 rows
    "maxH+1x1000": lambda: (bin16_max_h(1000) + 1, 1000),  # 69 x 1000
}


@pytest.mark.parametrize("case", list(OUTSIDE_BIN16))
def test_just_outside_bin16_takes_the_generic_engine(native, oracle, case):
    """One row or column past engine 5's edge: bin16_supported is 0, and binary aliased planes are searched by the
    generic engine alone (one launch), bit-exact."""
    H, W = OUTSIDE_BIN16[case]()
    assert native.lib().nastar_b200_bin16_supported(H, W) == 0 and engine_for(H, W) in (2, 3)
    rng = np.random.RandomState(H + 3 * W)
    obst, start, goal = _corner_problem(rng, 1, H, W, p_obst=0.25)
    _search_exact(native, oracle, (obst, start, goal, obst), W * W, 1, aliased=True, label=f"{H}x{W} generic")


# ------------------------------------------------------------------------------------------------------ engine 3
ENGINE3_SHAPES = {
    "maxHx1024": lambda: (generic_max_h(1024), 1024),    # 592 x 1024: the largest smem_common, W % 32 == 0
    "maxHx2048": lambda: (generic_max_h(2048), 2048),    # 299 x 2048
    "maxHx32": lambda: (generic_max_h(32), 32),          # 11 621 x 32
    "maxHx46340": lambda: (generic_max_h(46340), 46340),  # 13 x 46 340: W % 32 != 0, the widest bound that fits
}


def _learned_problem(rng, H, W, dist):
    obst, start, goal = (_near_problem(rng, 1, H, W, 0.1, dist) if dist else _corner_problem(rng, 1, H, W, 0.1))
    cost = rng.uniform(0.1, 1.0, obst.shape).astype(np.float32)
    return cost, start, goal, obst


@pytest.mark.parametrize("mechanism", ["moore", "news"])
@pytest.mark.parametrize("case", list(ENGINE3_SHAPES))
def test_engine3_at_its_edges_vs_oracle(native, oracle, case, mechanism):
    """Learned-style costs (uniform(0.1, 1), 10 % obstacles) on engine 3's largest shapes.  Evaluation (T = W * W,
    start and goal a short way apart, or at 11 621 x 32 far apart with the bound capping it) bit-exact; training with
    a small Tmax (T = 256) with start and goal 400 cells apart, capped, bit-exact, and its backward within the oracle's
    bound."""
    from neural_astar.planner.differentiable_astar import DifferentiableAstar

    H, W = ENGINE3_SHAPES[case]()
    assert engine_for(H, W) == 3 and not bin16_supported(H, W)
    rng = np.random.RandomState(H + W + (mechanism == "news"))
    far = W < 64
    dist = 0 if far else (3000 if mechanism == "moore" else 500) if W > 40000 else 20
    planes = _learned_problem(rng, H, W, dist)
    _, _, ref = _search_exact(native, oracle, planes, W * W, 1, mechanism=mechanism, label=f"{H}x{W} eval")
    assert (ref.t_solve == -1).all() if far else (ref.t_solve >= 0).all()   # capped by W * W = 1024, or solved

    astar = DifferentiableAstar(Tmax=0.25 if far else 256.5 / (W * W), mechanism=mechanism).train()
    T = astar.num_steps(W)
    assert T in (256, 257)
    # 400 cells apart: more than T steps from the goal, and f / sqrt(W) small enough that the softmax numerators
    # exp(-f / sqrt(W)) stay representable in fp32, as in the reference
    planes = _learned_problem(rng, H, W, 400)
    (hist, _, ts, ns), dev, ref = _search_exact(native, oracle, planes, T, 1, mechanism=mechanism,
                                                label=f"{H}x{W} train")
    assert (ref.t_solve == -1).all()
    G = rng.randn(*planes[0].shape).astype(np.float32)
    Tb = native.batch_steps(ts, ns, T)
    assert int(Tb.item()) == T
    before = native.launch_count()
    gc, t_gpu = _clock(lambda: native.backward(*dev, _dev(G), Tb, ts, 0.5, mechanism=mechanism))
    assert native.launch_count() - before == 1
    t0 = time.perf_counter()
    want, M = oracle.backward_with_bound(*planes, G, T, mechanism=mechanism)
    print(f"{H}x{W} backward {mechanism}: gpu {t_gpu:.3f} s, oracle {time.perf_counter() - t0:.2f} s")
    gc = gc.cpu().numpy()
    assert_within_bound(gc, want, M, (H, W), mechanism=mechanism)
    # the module's route gives the same histories and gradient
    c = _dev(planes[0]).requires_grad_(True)
    out = astar.cuda()(c, *dev[1:])
    assert torch.equal(out.histories.detach(), hist)
    (out.histories * _dev(G)).sum().backward()
    assert torch.equal(c.grad.cpu(), torch.from_numpy(gc))


def test_engine3_coupled_low_g_ratio_at_2048(native, oracle):
    """The batch-coupled search (g_ratio 0.3, B = 2) at 299 x 2048, in training with a cap of about 300 steps: the
    module's host-coupled route and the device-decided forward_coupled route both equal the oracle run for exactly
    T_batch steps, and both gradients its closed form within its bound."""
    from neural_astar.planner.differentiable_astar import DifferentiableAstar, _AstarSearch

    H, W, B, g_ratio = generic_max_h(2048), 2048, 2, 0.3
    assert engine_for(H, W) == 3
    rng = np.random.RandomState(29)
    obst, start, goal = _near_problem(rng, B, H, W, 0.1, 12)
    cost = rng.uniform(0.1, 1.0, obst.shape).astype(np.float32)
    G = rng.randn(B, 1, H, W).astype(np.float32)
    astar = DifferentiableAstar(g_ratio=g_ratio, Tmax=300.5 / (W * W)).cuda().train()
    T = astar.num_steps(W)
    assert T == 300
    t0 = time.perf_counter()
    full = oracle.forward(cost, start, goal, obst, g_ratio=g_ratio, mode="spec", want_trace=True, T=T,
                          no_early_exit=True)
    gidx = goal.reshape(B, -1).argmax(1)
    every = (full.trace == gidx[:, None]).all(0)
    T_batch = int(every.argmax()) + 1 if every.any() else T
    ref = oracle.forward(cost, start, goal, obst, g_ratio=g_ratio, mode="spec", T=T_batch, no_early_exit=True)
    want, M = oracle.backward_with_bound(cost, start, goal, obst, G, T_batch, g_ratio=g_ratio)
    print(f"coupled 299x2048: T_batch {T_batch}, oracle {time.perf_counter() - t0:.2f} s")
    dev = [_dev(x) for x in (cost, start, goal, obst)]
    for device_coupled in (False, True):
        c = dev[0].clone().requires_grad_(True)
        if device_coupled:
            hist, paths = _AstarSearch.apply(c, *dev[1:], g_ratio, T, False, None, "moore", True)[:2]
        else:
            hist, paths = astar(c, *dev[1:])[:2]
        np.testing.assert_array_equal(hist.detach().cpu().numpy(), ref.histories)
        np.testing.assert_array_equal(paths.cpu().numpy(), ref.paths)
        (hist * _dev(G)).sum().backward()
        assert_within_bound(c.grad.cpu().numpy(), want, M, ("coupled 299x2048", device_coupled))


def _strip(W):
    plane = np.ones((1, 1, 1, W), np.float32)
    start = np.zeros_like(plane)
    goal = np.zeros_like(plane)
    start[0, 0, 0, 0] = goal[0, 0, 0, W - 1] = 1
    return plane, start, goal


def test_open_strip_rule_vs_oracle(native, oracle):
    """A 1 x W open strip with the start at x = 0 and the goal at x = W - 1: the cells close in order, the goal is
    selected at step W - 1 and every cell is on the path.  Checked against the oracle at W = 200, the rule that the
    46 340-wide case below relies on."""
    W = 200
    plane, start, goal = _strip(W)
    _, _, ref = _search_exact(native, oracle, (plane, start, goal, plane), W * W, 1, label="strip 200")
    assert ref.t_solve.tolist() == [W - 1] and ref.n_steps.tolist() == [W]
    assert (ref.histories == 1).all() and (ref.paths == 1).all()


@pytest.mark.parametrize("mechanism", ["moore", "news"])
def test_open_strip_at_the_widest_bound(native, oracle, mechanism):
    """1 x 46 340: the evaluation bound W * W = 2 147 395 600 just fits.  The search runs W steps and the answer is the
    strip rule.  In training (T = 2 147 steps) toward a goal at x = 3 000 it is capped, bit-exact against the oracle,
    and its gradient, zero in closed form on one row, is zero to within the oracle's bound on every cell."""
    from neural_astar.planner.differentiable_astar import DifferentiableAstar

    W = native.MAX_EVAL_WIDTH
    assert W * W <= native.MAX_STEPS < (W + 1) * (W + 1) and engine_for(1, W) == 3
    plane, start, goal = _strip(W)
    dev = [_dev(x) for x in (plane, start, goal)]
    before = native.launch_count()
    (hist, paths, ts, ns, _), t_gpu = _clock(lambda: native.forward(dev[0], dev[1], dev[2], dev[0], 0.5, W * W,
                                                                    mechanism=mechanism))
    assert native.launch_count() - before == 1
    print(f"strip {W} eval {mechanism}: gpu {t_gpu:.3f} s")
    assert ts.tolist() == [W - 1] and ns.tolist() == [W]
    assert bool((hist == 1).all()) and bool((paths == 1).all())
    astar = DifferentiableAstar(Tmax=1e-6, mechanism=mechanism).cuda().train()
    T = astar.num_steps(W)
    assert T == 2147
    cost = np.random.RandomState(3).uniform(0.1, 1.0, plane.shape).astype(np.float32)
    goal = np.zeros_like(plane)
    goal[0, 0, 0, 3000] = 1   # beyond the T steps, near enough that exp(-f / sqrt(W)) stays an fp32 number
    planes = (cost, start, goal, plane)
    (_, _, ts, ns), devp, ref = _search_exact(native, oracle, planes, T, 1, mechanism=mechanism, label="strip train")
    assert ref.t_solve.tolist() == [-1]
    G = np.random.RandomState(4).randn(*plane.shape).astype(np.float32)
    gc = native.backward(*devp, _dev(G), native.batch_steps(ts, ns, T), ts, 0.5, mechanism=mechanism).cpu().numpy()
    want, M = oracle.backward_with_bound(*planes, G, T, mechanism=mechanism)
    # one row: the one open cell takes the whole softmax at every step, so each step's term y * (G - <G, y>) is zero
    # and so is the gradient; the engine's running sums leave rounding residue, which must stay within M
    assert not want.any()
    assert_within_bound(gc, want, M, "strip train", mechanism=mechanism)


def test_heuristic_beyond_4096_cells_rounds_like_the_reference(native, oracle):
    """get_heuristic squares and adds dy and dx in fp32, so beyond 4 096 cells (dx * dx > 2**24) the sum is rounded
    twice.  At (dy, dx) = (7, 4 281) that gives 4 285.281, where the exactly rounded integer sum gives the next float
    up, the value of dy = 8 and 9.  With the goal at (12, 0) and the start at (4, 4 282), the three neighbours in
    column 4 281 then tie or not: the reference selects (5, 4 281) first, and a heuristic from the integer sum the
    lowest index of the tie, (3, 4 281).  Generic engine (13 x 4 400: engine 3), Moore."""
    H, W = 13, 4400
    assert engine_for(H, W) == 3
    plane = np.ones((1, 1, H, W), np.float32)
    start = np.zeros_like(plane)
    goal = np.zeros_like(plane)
    start[0, 0, 4, 4282] = goal[0, 0, 12, 0] = 1
    planes = (plane, start, goal, plane)
    T = 8192
    hist, paths, ts, ns, tr = native.forward(*(_dev(x) for x in planes), 0.5, T, True)
    ref = oracle.forward(*planes, mode="spec", want_trace=True, T=T)
    assert ref.trace[0, 1] == 5 * W + 4281
    np.testing.assert_array_equal(tr.cpu().numpy(), ref.trace)
    np.testing.assert_array_equal(hist.cpu().numpy(), ref.histories)
    np.testing.assert_array_equal(paths.cpu().numpy(), ref.paths)
    assert ts.tolist() == ref.t_solve.tolist()


# ---------------------------------------------------------------------------------------------- outside engine 3
@pytest.mark.parametrize("shape", [lambda: (generic_max_h(1024) + 1, 1024), lambda: (generic_max_h(46340) + 1, 46340)],
                         ids=["593x1024", "14x46340"])
def test_just_outside_engine3_is_unsupported(native, shape):
    """One row past the generic engine's edge (593 x 1024, 14 x 46 340): _native.forward and DifferentiableAstar
    raise the library's "unsupported" error, and nothing is launched."""
    from neural_astar.planner.differentiable_astar import DifferentiableAstar

    H, W = shape()
    assert engine_for(H, W) == 0 and W * W <= native.MAX_STEPS
    x = torch.ones((1, 1, H, W), device="cuda")
    s = torch.zeros_like(x)
    s[0, 0, 0, 0] = 1
    before = native.launch_count()
    with pytest.raises(RuntimeError, match="unsupported"):
        native.forward(x, s, s, x, 0.5, W * W)
    with pytest.raises(RuntimeError, match="unsupported"):
        DifferentiableAstar()(x, s, s, x)
    assert native.launch_count() == before


@pytest.mark.parametrize("W", [46341, 92682])
def test_step_bound_above_int32_is_refused(native, W):
    """1 x 46 341 and 1 x 92 682 strips take the generic engine, but their evaluation bound W * W does not fit the
    library's int32: a ValueError from DifferentiableAstar, forward, forward_coupled, batch_steps and backward, and
    no launch.  (Truncated, 92 682 would search 18 532 steps and report the goal at x = W - 1 as not found.)"""
    from neural_astar.planner.differentiable_astar import DifferentiableAstar

    assert engine_for(1, W) == 3
    plane, start, goal = (_dev(x) for x in _strip(W))
    ts = torch.zeros(1, dtype=torch.int32, device="cuda")
    before = native.launch_count()
    with pytest.raises(ValueError, match=f"W = {W}"):
        DifferentiableAstar()(plane, start, goal, plane)
    with pytest.raises(ValueError, match="2\\*\\*31 - 1"):
        native.forward(plane, start, goal, plane, 0.5, W * W)
    with pytest.raises(ValueError, match="2\\*\\*31 - 1"):
        native.forward_coupled(plane, start, goal, plane, 0.3, W * W)
    with pytest.raises(ValueError, match="2\\*\\*31 - 1"):
        native.batch_steps(ts, ts, W * W)
    with pytest.raises(ValueError, match="2\\*\\*31 - 1"):
        native.backward(plane, start, goal, plane, plane, W * W, ts, 0.5)
    assert native.launch_count() == before
