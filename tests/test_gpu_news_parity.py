"""The 4-connected (NEWS) search checked like the 8-connected one: the Moore checks of test_gpu_forward_parity.py,
test_gpu_backward_parity.py and test_gpu_engine_schedules.py with mechanism="news", against the C oracle's NEWS
mode (oracle/astar_oracle.c; its LITERAL form equals the reference on tests/golden/news/, test_news_oracle_cpu.py).

Every shape asserts the engine it is meant to reach (nastar_b200_engine_for): 1 (32-wide), 4 (64-wide), 2 (generic,
state in shared memory) and 3 (generic, HBM workspace).  Engine 5 is Moore-only.
"""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from golden_util import Golden
from oracle import oracle
from search_steps import MOVES, SpecMachine
from grad_bound import assert_within_bound, relerr_to_max
from test_news_oracle_cpu import problems

pytestmark = pytest.mark.gpu
TOL = 1e-5
GENERIC_CTAS_PER_SM = 8   # nastar_api.cu kGlobalCtasPerSm: generic_slots(B) = min(B, 8 x SMs)
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def native():
    from neural_astar import _native

    _native.lib()
    return _native


def _cu(x):
    return torch.from_numpy(np.ascontiguousarray(x)).cuda()


def _np(x):
    return x.detach().cpu().numpy()


def _engine(native, H, W):
    return native.lib().nastar_b200_engine_for(H, W)


def _fwd_vs_spec(native, planes, T, g_ratio=0.5, dev=None, trace=True, no_early_exit=False, alias=False, **kw):
    """NEWS forward on the device planes against SPEC on the host planes: histories, paths, t_solve, n_steps, trace
    and both per-map counts bit for bit.  Returns (t_solve, n_steps) on the device and the oracle's output."""
    cost, start, goal, obst = planes
    if dev is None:
        dev = [_cu(x) for x in planes]
        if alias:
            dev[3] = dev[0]
    hist, paths, ts, ns, tr, (ncl, plen) = native.forward(*dev, g_ratio, T, trace, no_early_exit, want_counts=True,
                                                          mechanism="news", **kw)
    ref = oracle.forward(cost, start, goal, obst, g_ratio=g_ratio, mode="spec", want_trace=trace, T=T,
                         no_early_exit=no_early_exit, mechanism="news")
    what = (cost.shape, g_ratio, T, no_early_exit)
    np.testing.assert_array_equal(_np(ts), ref.t_solve, err_msg=str(what))
    np.testing.assert_array_equal(_np(ns), ref.n_steps, err_msg=str(what))
    if trace:
        np.testing.assert_array_equal(_np(tr), ref.trace, err_msg=str(what))
    np.testing.assert_array_equal(_np(hist), ref.histories, err_msg=str(what))
    np.testing.assert_array_equal(_np(paths), ref.paths, err_msg=str(what))
    np.testing.assert_array_equal(_np(ncl), ref.histories.sum((1, 2, 3)).astype(np.int64), err_msg=str(what))
    np.testing.assert_array_equal(_np(plen), ref.paths.sum((1, 2, 3)), err_msg=str(what))
    return ts, ns, ref


def _bwd_vs_oracle(native, planes, dev, ts, ns, T, G, g_ratio=0.5, T_batch=None):
    """NEWS backward for the forward's T_batch (or a given shorter one) against the oracle's closed form."""
    cost, start, goal, obst = planes
    Tb = native.batch_steps(ts, ns, T) if T_batch is None else torch.full((1,), T_batch, dtype=torch.int32,
                                                                          device="cuda")
    gc = _np(native.backward(*dev, _cu(G), Tb, ts, g_ratio, mechanism="news"))
    want, M = oracle.backward_with_bound(cost, start, goal, obst, G, int(Tb.item()), g_ratio=g_ratio, mechanism="news")
    assert_within_bound(gc, want, M, (cost.shape, g_ratio, T, int(Tb.item())), mechanism="news")
    return int(Tb.item())


def _max_f_over_sqrt_w(planes, g_ratio, T):
    """An upper bound of f / sqrt(W) over every cell that is ever open in the first T steps (early exit at the goal):
    g of an opened cell is g + cost of a closed one.  Kept below 80 so that exp(-f / sqrt(W)) stays a normal fp32
    number, in the oracle's softmax as in the reference's."""
    cost, start, goal, obst = planes
    gr, omg, sqw = oracle.scalars(g_ratio, cost.shape[-1])
    worst = 0.0
    for b in range(cost.shape[0]):
        gi = int(goal[b].argmax())
        m = SpecMachine(cost[b, 0], obst[b, 0], int(start[b].argmax()), gi, "news")
        gmax = 0.0
        for _ in range(T):
            ind = m.select(gr, omg)
            if ind < 0:
                break
            gmax = max(gmax, float(m.g[ind] + m.cost[ind]))
            m.close_and_expand(ind)
            if ind == gi:
                break
        worst = max(worst, (float(gr) * gmax + float(omg) * float(m.h.max())) / float(sqw))
    return worst


def _edge_problems(rs, kinds, H, W, p_obst=0.15):
    """One map per entry of `kinds`:
      short       goal within a few cells of the start (over 4-connected moves, may still be unreachable);
      long        start in the top-left corner, goal a quarter of the map away (at the far corner for `far`);
      same        start == goal;
      walled      the start's 4 neighbours are obstacles: the open set empties after one step (t_solve -2);
      enclosed    no obstacles but around the goal: every other cell is reachable (capped for T < N - 5);
      on_obstacle the start cell itself is an obstacle (the reference opens it all the same)."""
    B = len(kinds)
    obst = (rs.rand(B, 1, H, W) > p_obst).astype(np.float32)
    start = np.zeros_like(obst)
    goal = np.zeros_like(obst)
    for b, kind in enumerate(kinds):
        sy, sx = rs.randint(H), rs.randint(W)
        if kind == "short":
            gy, gx = min(max(sy + rs.randint(-3, 4), 0), H - 1), min(max(sx + rs.randint(-3, 4), 0), W - 1)
        elif kind in ("long", "far"):
            (sy, sx) = (0, 0)
            (gy, gx) = (H - 1, W - 1) if kind == "far" else (H // 4, W // 4)
        elif kind == "same":
            gy, gx = sy, sx
        elif kind == "walled":
            gy, gx = (sy + H // 2) % H, (sx + W // 2) % W
        elif kind == "enclosed":
            (sy, sx), (gy, gx) = (0, 0), (H // 2, W // 2)
            obst[b] = 1
        elif kind == "on_obstacle":
            gy, gx = min(sy + 2, H - 1), min(sx + 2, W - 1)
        else:
            raise ValueError(kind)
        obst[b, 0, sy, sx] = obst[b, 0, gy, gx] = 1
        for dy, dx in MOVES["news"]:
            if kind == "walled" and 0 <= sy + dy < H and 0 <= sx + dx < W:
                obst[b, 0, sy + dy, sx + dx] = 0
            if kind == "enclosed" and 0 <= gy + dy < H and 0 <= gx + dx < W:
                obst[b, 0, gy + dy, gx + dx] = 0
        if kind == "on_obstacle":
            obst[b, 0, sy, sx] = 0
        start[b, 0, sy, sx] = 1
        goal[b, 0, gy, gx] = 1
    return obst, start, goal


def _learned(rs, shape, scale=1.0):
    return (1.0 / (1.0 + np.exp(-rs.randn(*shape)))).astype(np.float32) * np.float32(scale)


# ------------------------------------------------------------------------------------------------ 1. forward vs SPEC
FWD_SHAPES = [(12, 12, 1), (5, 40, 4), (32, 32, 1), (33, 31, 4), (64, 64, 4), (65, 64, 2), (128, 128, 2),
              (131, 131, 2), (131, 132, 3), (1, 32, 1), (32, 1, 1), (2, 64, 4), (64, 2, 4), (1, 200, 2)]


@pytest.mark.parametrize("learned", [True, False], ids=["learned", "binary"])
@pytest.mark.parametrize("H,W,engine", FWD_SHAPES)
def test_forward_vs_spec_every_g_ratio(native, H, W, engine, learned):
    """g_ratio 0.0 / 0.3 / 0.8 / 1.0 at obstacle densities 0 / 0.25 / 0.45, every output bit for bit.  `binary`
    passes the obstacle plane itself as the cost; above 64 that must not go to the Moore-only engine 5, also without
    a trace (where Moore would offer it there): one launch, equal to SPEC."""
    assert _engine(native, H, W) == engine
    N = H * W
    B = 2 if N > 8192 else (4 if N > 2048 else 8)
    rs = np.random.RandomState(977 * H + W + learned)
    for p_obst in (0.0, 0.25, 0.45):
        planes = problems(rs, B, H, W, p_obst, learned)
        for g_ratio in (0.0, 0.3, 0.8, 1.0):
            _fwd_vs_spec(native, planes, W * W, g_ratio, alias=not learned)
        if not learned and engine in (2, 3):
            before = native.launch_count()
            _fwd_vs_spec(native, planes, W * W, 0.5, trace=False, alias=True)
            assert native.launch_count() - before == 1


# ------------------------------------------------------------------------------------------------ 2. no early exit
@pytest.mark.parametrize("H,W,engine,B", [(32, 32, 1, 6), (64, 64, 4, 4), (100, 72, 2, 3), (144, 136, 3, 2)])
def test_no_early_exit_vs_spec(native, H, W, engine, B):
    """NASTAR_FWD_NO_EARLY_EXIT (the batch-coupled path's search) at g_ratio 0.0 / 0.3 / 0.5, for T below every map's
    solve step and for T past all of them (post-solve steps re-select the goal or leave it)."""
    assert _engine(native, H, W) == engine
    rs = np.random.RandomState(H * 3 + W)
    planes = problems(rs, B, H, W, 0.15, True)
    for g_ratio in (0.0, 0.3, 0.5):
        ts = oracle.forward(*planes, g_ratio=g_ratio, mode="spec", T=W * W, mechanism="news").t_solve
        assert (ts > 0).all()
        for T in (int(ts.min()), int(ts.max()) + 40):
            _fwd_vs_spec(native, planes, T, g_ratio, no_early_exit=True)


# ------------------------------------------------------------------------------------------------ 3. edge maps
EDGE_KINDS = ["short", "same", "walled", "enclosed", "on_obstacle", "long", "short", "same"]


@pytest.mark.parametrize("H,W,engine", [(32, 32, 1), (48, 64, 4), (100, 72, 2), (144, 136, 3)])
def test_edge_maps_in_one_batch(native, H, W, engine):
    """start == goal (t_solve 0), walled-in start (-2), step cap (-1 and a backtrack of T - 1 hops) and a start on an
    obstacle, next to ordinary maps, at g_ratio 0.5 and 0.3, with T = N / 2."""
    assert _engine(native, H, W) == engine
    rs = np.random.RandomState(H + 5 * W)
    obst, start, goal = _edge_problems(rs, EDGE_KINDS, H, W)
    planes = (_learned(rs, obst.shape, 3.0), start, goal, obst)
    T = H * W // 2
    for g_ratio in (0.5, 0.3):
        ts, _, ref = _fwd_vs_spec(native, planes, T, g_ratio)
        ts = _np(ts)
        for kind, want in (("same", 0), ("walled", -2), ("enclosed", -1)):
            assert (ts[[b for b, k in enumerate(EDGE_KINDS) if k == kind]] == want).all(), kind
        b = EDGE_KINDS.index("enclosed")
        assert ref.paths[b].sum() >= 1 and ref.n_steps[b] == T


# ------------------------------------------------------------------------------------------------ 4. batch coupling
@pytest.mark.parametrize("H,W,engine,B", [(32, 32, 1, 6), (48, 40, 4, 5), (100, 72, 2, 3), (144, 136, 3, 2)])
@pytest.mark.parametrize("g_ratio", [0.0, 0.3])
@pytest.mark.parametrize("train", [False, True])
def test_coupled_module_vs_literal(native, H, W, engine, B, g_ratio, train):
    """DifferentiableAstar(g_ratio < 0.5, mechanism="news") with B > 1 against the LITERAL oracle (the reference's loop
    as written): frame count = T_batch + 1, masks, every frame's selection, and cost.grad against the closed form for
    T_batch steps."""
    from neural_astar.planner.differentiable_astar import DifferentiableAstar

    assert _engine(native, H, W) == engine
    rs = np.random.RandomState(H * W + int(10 * g_ratio) + 7 * train)
    cost, start, goal, obst = problems(rs, B, H, W, 0.15, True)
    cost = cost * np.float32(10.0)
    G = rs.randn(B, 1, H, W).astype(np.float32)
    T = int((0.25 if train else 1.0) * W * W)
    lit = oracle.forward(cost, start, goal, obst, g_ratio=g_ratio, mode="literal", want_trace=True, T=T,
                         mechanism="news")
    astar = DifferentiableAstar(g_ratio=g_ratio, Tmax=0.25, mechanism="news").cuda().train(train)
    c = _cu(cost).requires_grad_(True)
    out = astar(c, _cu(start), _cu(goal), _cu(obst), store_intermediate_results=True)
    assert len(out.intermediate_results) == lit.T_batch + 1
    np.testing.assert_array_equal(_np(out.histories), lit.histories)
    np.testing.assert_array_equal(_np(out.paths), lit.paths)
    sel = torch.stack([f["paths"].reshape(B, -1).argmax(1) for f in out.intermediate_results[:-1]], 1)
    np.testing.assert_array_equal(_np(sel), lit.trace[:, :lit.T_batch])
    (out.histories * _cu(G)).sum().backward()
    want, M = oracle.backward_with_bound(cost, start, goal, obst, G, lit.T_batch, g_ratio=g_ratio, mechanism="news")
    assert_within_bound(_np(c.grad), want, M, (H, W, g_ratio, train, lit.T_batch), mechanism="news")


def test_all064_lowg_golden_through_the_module(native):
    """The reference's g_ratio 0.3 batch at 64x64: masks, T_batch, every frame's selection and the gradient."""
    from neural_astar.planner.differentiable_astar import DifferentiableAstar

    g = Golden("news/news_all064_lowg")
    assert _engine(native, g.H, g.W) == 4
    astar = DifferentiableAstar(g_ratio=g.g_ratio, mechanism="news").cuda().eval()
    c = _cu(g.cost).requires_grad_(True)
    out = astar(c, _cu(g.start), _cu(g.goal), _cu(g.obst), store_intermediate_results=True)
    np.testing.assert_array_equal(_np(out.histories) != 0, g.bits("hist_bits") != 0)
    np.testing.assert_array_equal(_np(out.paths) != 0, g.bits("path_bits") != 0)
    assert len(out.intermediate_results) == int(g.z["T_batch"]) + 1
    sel = torch.stack([f["paths"].reshape(g.B, -1).argmax(1) for f in out.intermediate_results[:-1]], 1)
    np.testing.assert_array_equal(_np(sel), g.z["trace"])
    (out.histories * _cu(g.plane("rand_G"))).sum().backward()
    assert relerr_to_max(_np(c.grad), g.plane("rand_grad_cost")) < TOL


def test_all064_learned_golden_eval_and_training(native):
    from neural_astar.planner.differentiable_astar import DifferentiableAstar

    g = Golden("news/news_all064_learned")
    assert _engine(native, g.H, g.W) == 4
    astar = DifferentiableAstar(Tmax=0.25, mechanism="news").cuda().eval()
    with torch.no_grad():
        out = astar(_cu(g.cost), _cu(g.start), _cu(g.goal), _cu(g.obst), store_intermediate_results=True)
    np.testing.assert_array_equal(_np(out.histories) != 0, g.bits("hist_bits") != 0)
    np.testing.assert_array_equal(_np(out.paths) != 0, g.bits("path_bits") != 0)
    assert len(out.intermediate_results) == int(g.z["T_batch"]) + 1
    sel = torch.stack([f["paths"].reshape(g.B, -1).argmax(1) for f in out.intermediate_results[:-1]], 1)
    np.testing.assert_array_equal(_np(sel), g.z["trace"])
    astar.train()
    c = _cu(g.cost).requires_grad_(True)
    out = astar(c, _cu(g.start), _cu(g.goal), _cu(g.obst))
    np.testing.assert_array_equal(_np(out.histories) != 0, g.bits("train_hist_bits") != 0)
    np.testing.assert_array_equal(_np(out.paths) != 0, g.bits("train_path_bits") != 0)
    (out.histories * _cu(g.plane("rand_G"))).sum().backward()
    assert relerr_to_max(_np(c.grad), g.plane("train_grad_cost")) < TOL


def test_mazes032_gr08_golden_with_gradient(native):
    from neural_astar.planner.differentiable_astar import DifferentiableAstar

    g = Golden("news/news_mazes032_gr08")
    assert _engine(native, g.H, g.W) == 1
    astar = DifferentiableAstar(g_ratio=g.g_ratio, mechanism="news").cuda().eval()
    c = _cu(g.cost).requires_grad_(True)
    out = astar(c, _cu(g.start), _cu(g.goal), _cu(g.obst))
    np.testing.assert_array_equal(_np(out.histories) != 0, g.bits("hist_bits") != 0)
    np.testing.assert_array_equal(_np(out.paths) != 0, g.bits("path_bits") != 0)
    (out.histories * _cu(g.plane("rand_G"))).sum().backward()
    assert relerr_to_max(_np(c.grad), g.plane("rand_grad_cost")) < TOL


def test_large144_golden(native):
    g = Golden("news/news_large144_learned")
    assert _engine(native, g.H, g.W) == 3
    with torch.no_grad():
        hist, paths, _, ns, trace = native.forward(_cu(g.cost), _cu(g.start), _cu(g.goal), _cu(g.obst), 0.5,
                                                   g.W * g.W, want_trace=True, mechanism="news")
    np.testing.assert_array_equal(_np(hist) != 0, g.bits("hist_bits") != 0)
    np.testing.assert_array_equal(_np(paths) != 0, g.bits("path_bits") != 0)
    tr, ns = _np(trace), _np(ns)
    for b in range(g.B):
        np.testing.assert_array_equal(tr[b, :ns[b]], g.z["trace"][b, :ns[b]])


# ------------------------------------------------------------------------------------------------ 5. backward
BWD_KINDS = ["short", "long", "walled", "enclosed", "short", "long"]


@pytest.mark.parametrize("g_ratio", [0.3, 0.5, 0.8])
@pytest.mark.parametrize("H,W,engine,B", [(32, 32, 1, 6), (12, 20, 1, 6), (48, 40, 4, 6), (64, 64, 4, 4),
                                          (100, 72, 2, 4), (144, 136, 3, 3)])
def test_backward_every_engine(native, H, W, engine, B, g_ratio):
    """Eval-length and Tmax 0.25 loops, costs x1 and x10.  g_ratio >= 0.5: one batch mixing early-solved, capped and
    exhausted maps (the post-solve fold, and T_batch = T).  g_ratio < 0.5: the raw entry points map by map, where
    T_batch is the map's own stop step (the batch-coupled module path is test_coupled_module_vs_literal)."""
    assert _engine(native, H, W) == engine
    rs = np.random.RandomState(H * 100 + W + int(10 * g_ratio))
    obst, start, goal = _edge_problems(rs, BWD_KINDS[:B], H, W)
    for scale in (1.0, 10.0):
        cost = _learned(rs, obst.shape, scale)
        planes = (cost, start, goal, obst)
        G = rs.randn(*obst.shape).astype(np.float32)
        for T in (W * W, int(0.25 * W * W)):
            assert _max_f_over_sqrt_w(planes, g_ratio, T) < 80
            if g_ratio >= 0.5:
                dev = [_cu(x) for x in planes]
                ts, ns, ref = _fwd_vs_spec(native, planes, T, g_ratio, dev=dev, trace=False)
                _bwd_vs_oracle(native, planes, dev, ts, ns, T, G, g_ratio)
                continue
            for i in range(B):
                one = tuple(x[i:i + 1] for x in planes)
                dev = [_cu(x) for x in one]
                ts, ns, ref = _fwd_vs_spec(native, one, T, g_ratio, dev=dev, trace=False)
                lit = (oracle.forward(*one, g_ratio=g_ratio, mode="literal", T=T, mechanism="news")
                       if ref.t_solve[0] != -2 else None)
                Tb = _bwd_vs_oracle(native, one, dev, ts, ns, T, G[i:i + 1], g_ratio)
                if lit is not None:
                    assert lit.T_batch == Tb


@pytest.mark.parametrize("mechanism", ["news", "moore"])
@pytest.mark.parametrize("H,W,engine", [(32, 32, 1), (64, 64, 4), (100, 100, 2), (132, 132, 3)])
def test_backward_map_exhausted_after_a_long_search(native, oracle, H, W, engine, mechanism):
    """One map, no obstacles but the ring around the goal: the search closes every other cell and then runs out of
    open cells (t_solve -2).  At g_ratio 0.8 with learned costs x10 the last open cells have v = exp(-f/sqrt(W)) near
    e^-40, far below the early terms of the running sums S and D; the rounding left in D by those early terms used to
    swamp it (NEWS: relative error 0.7 at 64x64 and 7e-5 at 32x32 on engines 4 and 1).  The kernels now recompute S and
    D from the per-cell numerators once S has shrunk 2^16-fold (bwd_resum).  Checked for both mechanisms, Moore
    against the C oracle, with T = H*W so that every engine reaches exhaustion."""
    assert _engine(native, H, W) == engine
    rs = np.random.RandomState(H + W)
    obst = np.ones((1, 1, H, W), np.float32)
    start = np.zeros_like(obst)
    goal = np.zeros_like(obst)
    gy, gx = H // 2, W // 2
    obst[0, 0, gy - 1:gy + 2, gx - 1:gx + 2] = 0
    obst[0, 0, gy, gx] = 1
    start[0, 0, 0, 0] = 1
    goal[0, 0, gy, gx] = 1
    cost = _learned(rs, obst.shape, 10.0)
    planes = (cost, start, goal, obst)
    G = rs.randn(*obst.shape).astype(np.float32)
    T = H * W
    dev = [_cu(x) for x in planes]
    if mechanism == "news":
        assert _max_f_over_sqrt_w(planes, 0.8, T) < 80
        ts, ns, ref = _fwd_vs_spec(native, planes, T, 0.8, dev=dev, trace=False)
        assert ref.t_solve[0] == -2 and ref.n_steps[0] == H * W - 9
        _bwd_vs_oracle(native, planes, dev, ts, ns, T, G, 0.8)
        return
    hist, paths, ts, ns, _ = native.forward(*dev, 0.8, T)
    ref = oracle.forward(*planes, g_ratio=0.8, mode="spec", T=T)
    np.testing.assert_array_equal(_np(hist), ref.histories)
    assert _np(ts)[0] == -2 and _np(ns)[0] == H * W - 9
    Tb = native.batch_steps(ts, ns, T)
    gc = _np(native.backward(*dev, _cu(G), Tb, ts, 0.8))
    want, M = oracle.backward_with_bound(*planes, G, int(Tb.item()), g_ratio=0.8)
    assert_within_bound(gc, want, M, (H, W, "moore"))


@pytest.mark.parametrize("H,W,engine", [(48, 40, 4), (64, 64, 4), (100, 72, 2)])
@pytest.mark.parametrize("g_ratio", [0.3, 0.8])
def test_event_based_backward_single_map(native, H, W, engine, g_ratio):
    """B = 1, no batch coupling: below 0.5 the post-solve steps are replayed one by one, above they are folded.  The
    reference's own step count (LITERAL) is the kernel's T_batch."""
    assert _engine(native, H, W) == engine
    rs = np.random.RandomState(H + 3 * W + int(10 * g_ratio))
    for trial in range(2):
        cost, start, goal, obst = problems(rs, 1, H, W, 0.15, True)
        cost = cost * np.float32(10.0)
        planes = (cost, start, goal, obst)
        G = rs.randn(1, 1, H, W).astype(np.float32)
        for T in (W * W, W * W // 8):
            assert _max_f_over_sqrt_w(planes, g_ratio, T) < 80
            lit = oracle.forward(*planes, g_ratio=g_ratio, mode="literal", T=T, mechanism="news")
            dev = [_cu(x) for x in planes]
            hist, paths, ts, ns, _ = native.forward(*dev, g_ratio, T, mechanism="news")
            Tb = native.batch_steps(ts, ns, T)
            assert int(Tb.item()) == lit.T_batch
            gc = _np(native.backward(*dev, _cu(G), Tb, ts, g_ratio, mechanism="news"))
            want, M = oracle.backward_with_bound(*planes, G, lit.T_batch, g_ratio=g_ratio, mechanism="news")
            assert_within_bound(gc, want, M, (H, W, g_ratio, T, trial), mechanism="news")


# ------------------------------------------------------------------------------------------------ 6. schedules
@pytest.mark.parametrize("H,W,engine", [(48, 64, 4), (50, 47, 4), (96, 64, 2), (96, 50, 2), (65, 41, 2),
                                        (160, 128, 3)])
@pytest.mark.parametrize("misaligned", [False, True])
def test_prologue_variants(native, H, W, engine, misaligned):
    """16-byte aligned planes take the TMA / 128-bit prologues, the same planes one float past a 16-byte boundary the
    scalar ones.  Forward bit for bit with its trace, and the backward (256 steps) within the oracle's bound."""
    assert _engine(native, H, W) == engine
    rs = np.random.RandomState(H * 131 + W)
    kinds = [("long", "short", "long", "same")[b % 4] for b in range(8)]
    obst, start, goal = _edge_problems(rs, kinds, H, W, p_obst=0.2)
    planes = (_learned(rs, obst.shape, 3.0), start, goal, obst)
    dev = []
    for x in planes:
        if misaligned:
            buf = torch.zeros(x.size + 1, device="cuda")
            v = buf[1:1 + x.size].view(x.shape)
            v.copy_(torch.from_numpy(x))
            assert v.data_ptr() % 16 != 0
            dev.append(v)
        else:
            dev.append(_cu(x))
    ts, ns, _ = _fwd_vs_spec(native, planes, W * W, dev=dev)
    G = rs.randn(*obst.shape).astype(np.float32)
    _bwd_vs_oracle(native, planes, dev, ts, ns, W * W, G, T_batch=256)


FOLLOWERS = ("short", "same", "walled", "enclosed")


@pytest.mark.parametrize("H,W,engine", [(65, 40, 2), (144, 136, 3)])
def test_generic_slots_take_a_second_map(native, H, W, engine):
    """B = 8 x SMs + 64 maps: slot k runs map k (a long search) and then map k + slots (short, start == goal, walled-in
    start or step-capped).  Forward with trace and counts bit for bit; backward (the per-map reset) for 48 steps."""
    assert _engine(native, H, W) == engine
    slots = GENERIC_CTAS_PER_SM * torch.cuda.get_device_properties(0).multi_processor_count
    B = slots + 64
    kinds = ["short"] * B
    for k in range(B - slots):
        kinds[k] = "long"
        kinds[k + slots] = FOLLOWERS[k % len(FOLLOWERS)]
    rs = np.random.RandomState(H + W)
    obst, start, goal = _edge_problems(rs, kinds, H, W)
    planes = (_learned(rs, obst.shape), start, goal, obst)
    dev = [_cu(x) for x in planes]
    T = 2048
    ts, ns, _ = _fwd_vs_spec(native, planes, T, dev=dev)
    ts_h = _np(ts)
    for kind, want in (("same", 0), ("walled", -2), ("enclosed", -1)):
        assert (ts_h[[b for b in range(slots, B) if kinds[b] == kind]] == want).all(), kind
    _bwd_vs_oracle(native, planes, dev, ts, ns, T, rs.randn(*obst.shape).astype(np.float32), T_batch=48)


def test_engine3_workspace_left_by_moore_then_news(native, oracle):
    """Engine 3 with the same (B, H, W) three times: a Moore call, then two NEWS calls.  The caching allocator hands
    each call the workspace block the previous one left its g / f / parent planes and backward sums in."""
    H, W, B = 144, 136, 6
    assert _engine(native, H, W) == 3
    rs = np.random.RandomState(31)
    obst, start, goal = _edge_problems(rs, ["long"] * B, H, W)
    planes = (_learned(rs, obst.shape), start, goal, obst)
    dev = [_cu(x) for x in planes]
    hist, paths, ts, ns, _ = native.forward(*dev, 0.5, W * W)
    ref = oracle.forward(*planes, mode="spec", T=W * W)
    np.testing.assert_array_equal(_np(hist), ref.histories)
    G = rs.randn(*obst.shape).astype(np.float32)
    Tb = torch.full((1,), 256, dtype=torch.int32, device="cuda")
    gc = _np(native.backward(*dev, _cu(G), Tb, ts, 0.5))
    want, M = oracle.backward_with_bound(*planes, G, 256)
    assert_within_bound(gc, want, M, "moore before news")
    for kinds in (["long", "short", "long", "same", "long", "walled"], [FOLLOWERS[b % 4] for b in range(B)]):
        obst, start, goal = _edge_problems(rs, kinds, H, W)
        planes = (_learned(rs, obst.shape), start, goal, obst)
        dev = [_cu(x) for x in planes]
        ts, ns, _ = _fwd_vs_spec(native, planes, W * W, dev=dev)
        _bwd_vs_oracle(native, planes, dev, ts, ns, W * W, rs.randn(*obst.shape).astype(np.float32), T_batch=256)


@pytest.mark.parametrize("H,W,engine", [(32, 32, 1), (40, 50, 4), (100, 72, 2)])
def test_strided_and_multichannel_inputs(native, H, W, engine):
    """Only channel 0 of the cost is searched; start and goal are channel views of 3-channel tensors, the obstacle
    plane a window of a larger one.  Forward and backward against the oracle on the contiguous planes."""
    assert _engine(native, H, W) == engine
    rs = np.random.RandomState(9 * H + W)
    planes = problems(rs, 6, H, W, 0.2, True)
    cost, start, goal, obst = planes
    z = np.zeros_like(start)
    c3 = _cu(np.concatenate([cost, cost * 0 + 7, cost * 0 + 9], 1))
    s_view = _cu(np.concatenate([z, start, z], 1))[:, 1:2]
    g_view = _cu(np.concatenate([goal, z, z], 1))[:, 0:1]
    big = torch.zeros((6, 1, H + 8, W + 8), device="cuda")
    big[:, :, 3:3 + H, 5:5 + W] = _cu(obst)
    o_view = big[:, :, 3:3 + H, 5:5 + W]
    assert not (s_view.is_contiguous() or g_view.is_contiguous() or o_view.is_contiguous())
    dev = [c3, s_view, g_view, o_view]
    ts, ns, _ = _fwd_vs_spec(native, planes, W * W, dev=dev)
    G = rs.randn(*obst.shape).astype(np.float32)
    _bwd_vs_oracle(native, planes, dev, ts, ns, W * W, G)


# ------------------------------------------------------------------------------------------------ 7. launch forms
@pytest.mark.parametrize("H,W,engine", [(32, 32, 1), (20, 31, 1), (64, 64, 4), (40, 57, 4)])
def test_cost_logit_equals_the_plane_search(native, H, W, engine):
    """NASTAR_COST_LOGIT: the prologue's sigmoid(x) * scale equals torch.sigmoid(x) * scale bit for bit, so every
    output equals the plane search on that plane (and SPEC on it)."""
    assert _engine(native, H, W) == engine
    rs = np.random.RandomState(H * W)
    _, start, goal, obst = problems(rs, 6, H, W, 0.15, False)
    s, g, o = _cu(start), _cu(goal), _cu(obst)
    logits = _cu(rs.randn(6, 1, H, W).astype(np.float32) * 2)
    for scale in (10.0, 0.37):
        plane = torch.sigmoid(logits) * scale
        _fwd_vs_spec(native, (_np(plane), start, goal, obst), W * W, dev=[plane, s, g, o])
        a = native.forward(plane, s, g, o, 0.5, W * W, True, want_counts=True, mechanism="news")
        b = native.forward(logits, s, g, o, 0.5, W * W, True, want_counts=True, mechanism="news",
                           cost_kind=native.COST_LOGIT, cost_scale=scale)
        for x, y in zip(a[:5] + tuple(a[5]), b[:5] + tuple(b[5])):
            assert torch.equal(x, y)


@pytest.mark.parametrize("H,W,engine", [(20, 27, 1), (33, 31, 4)])
def test_cost_taps_ragged(native, H, W, engine):
    """NASTAR_COST_TAPS at ragged shapes (W not a multiple of 32): equals the plane search on cost_from_taps."""
    assert _engine(native, H, W) == engine
    rs = np.random.RandomState(H + W)
    _, start, goal, obst = problems(rs, 6, H, W, 0.15, False)
    s, g, o = _cu(start), _cu(goal), _cu(obst)
    taps = _cu(rs.randn(6, H, W, 9).astype(np.float32) * 0.5)
    bias, scale = 0.1, 2.0
    plane = native.cost_from_taps(taps, bias, scale)
    _fwd_vs_spec(native, (_np(plane), start, goal, obst), W * W, dev=[plane, s, g, o])
    a = native.forward(plane, s, g, o, 0.5, W * W, True, want_counts=True, mechanism="news")
    b = native.forward(taps, s, g, o, 0.5, W * W, True, want_counts=True, mechanism="news",
                       cost_kind=native.COST_TAPS, cost_scale=scale, cost_bias=bias)
    for x, y in zip(a[:5] + tuple(a[5]), b[:5] + tuple(b[5])):
        assert torch.equal(x, y)


@pytest.mark.parametrize("H,W,engine", [(32, 32, 1), (64, 64, 4), (100, 100, 2)])
def test_pair_launch_with_counts(native, H, W, engine):
    """NASTAR_FWD_PAIR with counts and no trace: the first half is SPEC on the learned costs, the second SPEC with
    cost = obstacles (both NEWS)."""
    assert _engine(native, H, W) == engine
    rs = np.random.RandomState(5 * H)
    cost, start, goal, obst = problems(rs, 6, H, W, 0.2, True)
    c, s, g, o = _cu(cost), _cu(start), _cu(goal), _cu(obst)
    hist, paths, ts, ns, tr, (ncl, plen) = native.forward(c, s, g, o, 0.5, W * W, pair=True, want_counts=True,
                                                          mechanism="news")
    assert tr is None
    for half, cst in ((slice(0, 6), cost), (slice(6, 12), obst)):
        ref = oracle.forward(cst, start, goal, obst, mode="spec", T=W * W, mechanism="news")
        np.testing.assert_array_equal(_np(hist[half]), ref.histories)
        np.testing.assert_array_equal(_np(paths[half]), ref.paths)
        np.testing.assert_array_equal(_np(ts[half]), ref.t_solve)
        np.testing.assert_array_equal(_np(ns[half]), ref.n_steps)
        np.testing.assert_array_equal(_np(ncl[half]), ref.histories.sum((1, 2, 3)).astype(np.int64))
        np.testing.assert_array_equal(_np(plen[half]), ref.paths.sum((1, 2, 3)))


@pytest.mark.parametrize("H,W", [(32, 32), (64, 64)])
def test_neural_astar_fused_forward_equals_encode_then_search(native, H, W):
    """NeuralAstar(mechanism="news") at inference takes the fused COST_TAPS path; it must equal encode() followed by
    a plane search, and SPEC on the encoder's cost."""
    from neural_astar.planner import NeuralAstar

    torch.manual_seed(H)
    na = NeuralAstar(encoder_arch="CNN", mechanism="news").cuda().eval()
    rs = np.random.RandomState(H + 1)
    _, start, goal, maps = problems(rs, 6, H, W, 0.2, False)
    m, s, g = _cu(maps), _cu(start), _cu(goal)
    with torch.no_grad():
        fused = na(m, s, g)
        cost = na.encode(m, s, g)
        plain = na.astar(cost, s, g, m)
    assert torch.equal(fused.histories, plain.histories) and torch.equal(fused.paths, plain.paths)
    ref = oracle.forward(_np(cost), start, goal, maps, mode="spec", mechanism="news")
    np.testing.assert_array_equal(_np(fused.histories), ref.histories)
    np.testing.assert_array_equal(_np(fused.paths), ref.paths)


# ------------------------------------------------------------------------------------------------ 8. heuristic tables
_FIRST_USE = r"""
import sys
sys.path[:0] = [{root!r}, {pkg!r}, {tests!r}]
import numpy as np, torch
from test_news_oracle_cpu import problems
from neural_astar import _native
from oracle import oracle

oracle.build()
for H, W, engine in ((32, 32, 1), (64, 64, 4)):
    assert _native.lib().nastar_b200_engine_for(H, W) == engine
    planes = problems(np.random.RandomState(H), 6, H, W, 0.2, True)
    dev = [torch.from_numpy(x).cuda() for x in planes]
    for mech, stream in (("news", torch.cuda.Stream()), ("moore", None), ("news", None)):
        with torch.cuda.stream(stream or torch.cuda.default_stream()):
            hist, paths, ts, ns, tr = _native.forward(*dev, 0.5, W * W, True, mechanism=mech)
        torch.cuda.synchronize()
        ref = oracle.forward(*planes, mode="spec", want_trace=True, T=W * W, mechanism=mech)
        for got, want in ((hist, ref.histories), (paths, ref.paths), (ts, ref.t_solve), (tr, ref.trace)):
            assert np.array_equal(got.cpu().numpy(), want), (H, W, mech)
print("first use ok")
"""


def test_news_heuristic_table_on_first_use():
    """A fresh process whose first search is NEWS on a non-default stream (engines 1 and 4), then Moore, then NEWS on
    the default stream: ensure_heur<kSide, true> fills the NEWS half of the table and publishes it before any use."""
    code = _FIRST_USE.format(root=ROOT, pkg=os.path.join(ROOT, "neural-astar_b200"),
                             tests=os.path.join(ROOT, "tests"))
    r = subprocess.run([sys.executable, "-c", code], cwd=ROOT, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0 and "first use ok" in r.stdout, r.stdout + r.stderr
