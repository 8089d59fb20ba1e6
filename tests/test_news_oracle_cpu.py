"""The C oracle's NEWS mode (oracle/astar_oracle.c, mechanism="news") checked where the GPU tests trust it, without a
GPU:

  * against the reference's own outputs on the goldens above 32x32, at g_ratio 0.3 and 0.8, and with gradients
    (tests/golden/news/, made by tests/golden/make_golden_news.py);
  * SPEC against LITERAL on random square and rectangular problems, binary and learned costs, capped maps included;
  * the fp64 closed-form backward against autograd through an independent torch restatement of the reference's loop.
"""
import math

import numpy as np
import pytest
import torch

from golden_util import Golden
from oracle import labels as label_oracle
from oracle import oracle
from search_steps import MOVES, SpecMachine, heuristic

F32 = np.float32


def _relerr(a, b):
    return float(np.abs(a - b).max() / (np.abs(b).max() + 1e-30))


def _forward(g, mode, **kw):
    return oracle.forward(g.cost, g.start, g.goal, g.obst, g_ratio=g.g_ratio, mode=mode, mechanism="news", **kw)


def _assert_masks(o, g, hist_key="hist_bits", path_key="path_bits"):
    np.testing.assert_array_equal(o.histories != 0, g.bits(hist_key) != 0)
    np.testing.assert_array_equal(o.paths != 0, g.bits(path_key) != 0)


# ------------------------------------------------------------------------------------------------ new goldens
def test_all064_learned_eval_and_training_gradient():
    """64x64 (engine 4) with learned costs: eval masks and every selection in both forms, then the Tmax 0.25 training
    batch and the closed-form gradient against the reference's autograd."""
    g = Golden("news/news_all064_learned")
    lit = _forward(g, "literal", want_trace=True)
    _assert_masks(lit, g)
    assert lit.T_batch == int(g.z["T_batch"])
    np.testing.assert_array_equal(lit.trace[:, :lit.T_batch], g.z["trace"])
    spec = _forward(g, "spec", want_trace=True)
    _assert_masks(spec, g)
    assert spec.T_batch == int(g.z["T_batch"])
    for b in range(g.B):
        n = int(spec.n_steps[b])
        np.testing.assert_array_equal(spec.trace[b, :n], g.z["trace"][b, :n])
        assert (g.z["trace"][b, n:] == g.z["goal_idx"][b]).all()
    T_train = int(0.25 * g.W * g.W)
    for mode in ("literal", "spec"):
        o = _forward(g, mode, T=T_train, want_trace=True)
        _assert_masks(o, g, "train_hist_bits", "train_path_bits")
        assert o.T_batch == int(g.z["train_T_batch"])
    lit = _forward(g, "literal", T=T_train, want_trace=True)
    np.testing.assert_array_equal(lit.trace[:, :lit.T_batch], g.z["train_trace"])
    gc = oracle.backward(g.cost, g.start, g.goal, g.obst, g.plane("rand_G"), int(g.z["train_T_batch"]),
                         g_ratio=g.g_ratio, mechanism="news")
    assert _relerr(gc, g.plane("train_grad_cost")) < 1e-5


def spec_batch_coupled(g):
    """SPEC form of the batch-synchronous loop for g_ratio < 0.5 (no early exit, stopped after the first step at which
    every map selects its goal), and that step count."""
    T = g.W * g.W
    full = _forward(g, "spec", want_trace=True, T=T, no_early_exit=True)
    at_goal = (full.trace == g.z["goal_idx"][:, None]).all(0)
    T_batch = int(np.argmax(at_goal)) + 1 if at_goal.any() else T
    return _forward(g, "spec", want_trace=True, T=T_batch, no_early_exit=True), T_batch


def test_all064_low_g_ratio_batch_coupled():
    """g_ratio 0.3 at 64x64: LITERAL and the coupled SPEC form give the reference's masks, T_batch and every selection,
    and the backward over T_batch steps its gradient.  The batch has maps whose goal is selected once and maps whose
    goal is selected again (gradient blocked there)."""
    g = Golden("news/news_all064_lowg")
    o = _forward(g, "literal", want_trace=True)
    _assert_masks(o, g)
    assert o.T_batch == int(g.z["T_batch"])
    np.testing.assert_array_equal(o.trace[:, :o.T_batch], g.z["trace"])
    s, T_batch = spec_batch_coupled(g)
    assert T_batch == int(g.z["T_batch"])
    _assert_masks(s, g)
    np.testing.assert_array_equal(s.trace, g.z["trace"])
    reselected = (g.z["trace"] == g.z["goal_idx"][:, None]).sum(1) >= 2
    assert reselected.any() and not reselected.all()
    gc = oracle.backward(g.cost, g.start, g.goal, g.obst, g.plane("rand_G"), T_batch, g_ratio=g.g_ratio,
                         mechanism="news")
    assert _relerr(gc, g.plane("rand_grad_cost")) < 1e-5


def test_large144_learned():
    """144x144 (engine 3's HBM workspace): masks, T_batch and every selection in both forms."""
    g = Golden("news/news_large144_learned")
    lit = _forward(g, "literal", want_trace=True)
    _assert_masks(lit, g)
    assert lit.T_batch == int(g.z["T_batch"])
    np.testing.assert_array_equal(lit.trace[:, :lit.T_batch], g.z["trace"])
    spec = _forward(g, "spec", want_trace=True)
    _assert_masks(spec, g)
    for b in range(g.B):
        n = int(spec.n_steps[b])
        np.testing.assert_array_equal(spec.trace[b, :n], g.z["trace"][b, :n])
        assert (g.z["trace"][b, n:] == g.z["goal_idx"][b]).all()


def test_mazes032_g_ratio_08_with_gradient():
    g = Golden("news/news_mazes032_gr08")
    lit = _forward(g, "literal", want_trace=True)
    _assert_masks(lit, g)
    assert lit.T_batch == int(g.z["T_batch"])
    np.testing.assert_array_equal(lit.trace[:, :lit.T_batch], g.z["trace"])
    spec = _forward(g, "spec", want_trace=True)
    _assert_masks(spec, g)
    assert spec.T_batch == int(g.z["T_batch"])
    for b in range(g.B):
        n = int(spec.n_steps[b])
        np.testing.assert_array_equal(spec.trace[b, :n], g.z["trace"][b, :n])
        assert (g.z["trace"][b, n:] == g.z["goal_idx"][b]).all()
    gc = oracle.backward(g.cost, g.start, g.goal, g.obst, g.plane("rand_G"), int(g.z["T_batch"]), g_ratio=g.g_ratio,
                         mechanism="news")
    assert _relerr(gc, g.plane("rand_grad_cost")) < 1e-5


# ------------------------------------------------------------------------------------------------ random problems
def problems(rs, B, H, W, p_obst, learned):
    """B maps with obstacle density p_obst whose start reaches the goal over 4-connected moves; learned costs in
    [0, 1) or the map itself as cost."""
    maps = (rs.rand(B, 1, H, W) >= p_obst).astype(F32)
    start = np.zeros_like(maps)
    goal = np.zeros_like(maps)
    for b in range(B):
        plane = maps[b, 0].reshape(-1)
        gi = int(rs.randint(H * W))
        plane[gi] = 1
        while True:
            d = label_oracle.opt_labels(maps[b:b + 1], np.array([gi]), mechanism="news")[0].reshape(-1)
            cand = np.flatnonzero((d > -(H * W)) & (d < 0))
            if len(cand) or H * W == 1:
                break
            # walled-in goal: open one of its 4-neighbours
            r, c = divmod(gi, W)
            nb = [(r + dr) * W + c + dc for dr, dc in MOVES["news"] if 0 <= r + dr < H and 0 <= c + dc < W]
            plane[nb[rs.randint(len(nb))]] = 1
        goal[b, 0].reshape(-1)[gi] = 1
        start[b, 0].reshape(-1)[int(cand[rs.randint(len(cand))])] = 1
    cost = rs.rand(B, 1, H, W).astype(F32) if learned else maps
    return cost, start, goal, maps


RANDOM_SHAPES = [(16, 16), (12, 20), (5, 40), (33, 31), (1, 32), (32, 1)]


def near_tie(cost, start, goal, obst, b, g_ratio, k, a_spec, a_lit):
    """True when step k of map b is a near tie that the two forms resolve differently (DESIGN.md "Selection
    semantics"): SPEC takes the strictly smaller f, while the two cells' fp32 softmax values are equal, so the
    reference's first argmax takes the lower flat index."""
    m = SpecMachine(cost[b, 0], obst[b, 0], int(start[b].argmax()), int(goal[b].argmax()), "news")
    gr, omg, sqw = oracle.scalars(g_ratio, cost.shape[-1])
    for _ in range(k):
        m.close_and_expand(m.select(gr, omg))
    f = m.f(gr, omg)
    e = torch.exp(torch.from_numpy((F32(-1) * f) / sqw)).numpy() * m.open
    y = e / e.sum()
    return bool(a_lit < a_spec and f[a_spec] < f[a_lit] and y[a_spec] == y[a_lit])


@pytest.mark.parametrize("learned", [True, False], ids=["learned", "binary"])
@pytest.mark.parametrize("H,W", RANDOM_SHAPES)
def test_spec_equals_literal_on_random_problems(H, W, learned):
    """g_ratio >= 0.5: equal masks, and traces equal up to each map's solve step (the reference then re-selects the
    goal).  g_ratio < 0.5: SPEC without early exit for LITERAL's T_batch steps equals LITERAL, trace included.  T =
    W*W is below the number of cells when H > W, so (33, 31) and (32, 1) have step-capped maps; a short training loop
    (T = N // 8) caps the others.  The one permitted difference is a near tie (test_news_near_tie_spec_vs_literal): a
    map whose traces part there is not compared further; every other map of the batch still is."""
    rs = np.random.RandomState(100 * H + W + 7 * learned)
    N = H * W
    capped = ties = 0
    for p_obst in (0.0, 0.25, 0.45):
        cost, start, goal, obst = problems(rs, 8, H, W, p_obst, learned)
        gidx = goal.reshape(8, -1).argmax(1)
        for T in (W * W, max(N // 8, 1)):
            for g_ratio in (0.5, 0.8, 1.0, 0.0, 0.3):
                what = (p_obst, T, g_ratio)
                kw = dict(g_ratio=g_ratio, want_trace=True, mechanism="news")
                lit = oracle.forward(cost, start, goal, obst, mode="literal", T=T, **kw)
                if g_ratio >= 0.5:
                    spec = oracle.forward(cost, start, goal, obst, mode="spec", T=T, **kw)
                    assert spec.T_batch == lit.T_batch, what
                else:
                    spec = oracle.forward(cost, start, goal, obst, mode="spec", T=lit.T_batch, no_early_exit=True, **kw)
                for b in range(8):
                    n = int(spec.n_steps[b])
                    diff = np.flatnonzero(spec.trace[b, :n] != lit.trace[b, :n])
                    if len(diff):
                        k = int(diff[0])
                        assert near_tie(cost, start, goal, obst, b, g_ratio, k, spec.trace[b, k], lit.trace[b, k]), \
                            (what, b, k)
                        ties += 1
                        continue
                    if g_ratio >= 0.5:
                        assert (lit.trace[b, n:lit.T_batch] == gidx[b]).all(), (what, b)
                    else:
                        assert n == lit.T_batch, (what, b)
                    assert spec.t_solve[b] == lit.t_solve[b], (what, b)
                    np.testing.assert_array_equal(spec.histories[b], lit.histories[b], err_msg=str((what, b)))
                    np.testing.assert_array_equal(spec.paths[b], lit.paths[b], err_msg=str((what, b)))
                capped += int((spec.t_solve == -1).sum())
    assert capped > 0
    assert ties <= 2, ties


@pytest.fixture(scope="module")
def news_near_tie():
    """The near tie the random comparison met: 33x31, no obstacles, cost = map (VanillaAstar), g_ratio 0.8, map 4 of
    the first draw of test_spec_equals_literal_on_random_problems[33-31-binary]."""
    cost, start, goal, obst = problems(np.random.RandomState(100 * 33 + 31), 8, 33, 31, 0.0, False)
    return tuple(x[4:5] for x in (cost, start, goal, obst))


def test_news_near_tie_spec_vs_literal(news_near_tie):
    """At step 358 two open cells have f = 15.404604 and 15.404605 (one ulp apart) and equal fp32 softmax values:
    the reference's first argmax takes the lower index 35, SPEC (and the engines) the smaller f, cell 173.  The next
    step takes the other one, so the two traces differ by one swap and every output agrees; the Moore near-tie vector
    (adversarial_neartie) is the same rule with a different outcome."""
    cost, start, goal, obst = news_near_tie
    lit = oracle.forward(cost, start, goal, obst, g_ratio=0.8, mode="literal", want_trace=True, mechanism="news")
    spec = oracle.forward(cost, start, goal, obst, g_ratio=0.8, mode="spec", want_trace=True, mechanism="news")
    diff = np.flatnonzero(spec.trace[0, :spec.T_batch] != lit.trace[0, :spec.T_batch])
    assert diff.tolist() == [358, 359]
    assert spec.trace[0, 358:360].tolist() == [173, 35] and lit.trace[0, 358:360].tolist() == [35, 173]
    assert near_tie(cost, start, goal, obst, 0, 0.8, 358, 173, 35)
    assert spec.T_batch == lit.T_batch and spec.t_solve.tolist() == lit.t_solve.tolist() == [425]
    np.testing.assert_array_equal(spec.histories, lit.histories)
    np.testing.assert_array_equal(spec.paths, lit.paths)


# ------------------------------------------------------------------------------------------------ backward vs autograd
def autograd_grad(cost, start, goal, obst, G, g_ratio, T):
    """d sum(histories * G) / d cost by autograd through a float64 torch restatement of the reference's batch loop
    with the NEWS neighbourhood and heuristic.  Selection, g, the open set and the stop rule follow the fp32 values
    (g and the open set carry no gradient in the reference); f enters the softmax as f32 + (f_live - f_live.detach()),
    so the softmax sees exactly the fp32 f that the closed form sees, and the gradient flows through
    h + cost -> f -> softmax -> straight-through selection -> clamp(histories + selection, 0, 1).
    Returns (grad [B,1,H,W] float64, T_batch, number of times each map selected its goal)."""
    B, _, H, W = cost.shape
    N = H * W
    c32 = cost.reshape(B, N).astype(F32)
    gi = goal.reshape(B, N).argmax(1)
    si = start.reshape(B, N).argmax(1)
    o = obst.reshape(B, N).astype(F32)
    gr, omg = F32(g_ratio), F32(1 - g_ratio)
    sqw = F32(math.sqrt(W))
    heur = np.stack([heuristic(H, W, gi[b], "news") for b in range(B)])
    h32 = heur + c32
    g32 = np.zeros((B, N), F32)
    open32 = np.zeros((B, N), F32)
    open32[np.arange(B), si] = 1
    closed = np.zeros((B, N), bool)

    leaf = torch.tensor(c32, dtype=torch.float64, requires_grad=True)
    h_live = torch.tensor(heur, dtype=torch.float64) + leaf
    hist = torch.zeros(B, N, dtype=torch.float64)
    goal_hits = np.zeros(B, int)
    T_batch = 0
    for t in range(T):
        f32 = gr * g32 + omg * h32
        f_live = float(gr) * torch.tensor(g32, dtype=torch.float64) + float(omg) * h_live
        f = torch.tensor(f32, dtype=torch.float64) + (f_live - f_live.detach())
        e = torch.exp(-f / float(sqw)) * torch.tensor(open32, dtype=torch.float64)
        y = e / e.sum(1, keepdim=True)
        # the selection itself: first maximum of the fp32 softmax, as the reference evaluates it
        e32 = torch.exp(torch.from_numpy((F32(-1) * f32) / sqw)).numpy() * open32
        ind = (e32 / e32.sum(1, keepdims=True)).argmax(1)
        hard = torch.zeros(B, N, dtype=torch.float64)
        hard[torch.arange(B), torch.from_numpy(ind)] = 1
        sel = (hard - y).detach() + y
        hist = torch.clamp(hist + sel, 0, 1)
        at_goal = ind == gi
        goal_hits += at_goal
        for b in range(B):
            k = int(ind[b])
            closed[b, k] = True
            if not at_goal[b]:
                open32[b, k] = 0
            g2 = g32[b, k] + c32[b, k]
            r, cc = divmod(k, W)
            for dr, dc in MOVES["news"]:
                y_, x_ = r + dr, cc + dc
                if not (0 <= y_ < H and 0 <= x_ < W):
                    continue
                n = y_ * W + x_
                if o[b, n] == 0:
                    continue
                if (open32[b, n] == 0 and not closed[b, n]) or (open32[b, n] != 0 and g32[b, n] > g2):
                    g32[b, n] = g2
                    open32[b, n] = 1
        T_batch = t + 1
        if at_goal.all():
            break
    (hist * torch.tensor(G.reshape(B, N), dtype=torch.float64)).sum().backward()
    return leaf.grad.numpy().reshape(B, 1, H, W), T_batch, goal_hits


@pytest.mark.parametrize("g_ratio", [0.0, 0.3, 0.5, 0.8])
@pytest.mark.parametrize("H,W,T", [(12, 12, None), (16, 16, None), (10, 14, None), (16, 16, 12), (9, 13, 8)])
def test_closed_form_backward_equals_fp64_autograd(H, W, T, g_ratio):
    """oracle.backward for the loop's T_batch against autograd, 1e-9 relative.  T = None is the eval loop (W*W steps);
    the short loops leave maps step-capped.  Each case asserts that it contains what it is meant to: a capped map in
    the short loops, and in the eval loops a map whose goal is selected more than once (its goal gradient blocked)."""
    rs = np.random.RandomState(H * 31 + W + int(10 * g_ratio) + (T or 0))
    B = 6
    cost, start, goal, obst = problems(rs, B, H, W, 0.2, True)
    cost = cost * F32(3.0)
    G = rs.randn(B, 1, H, W).astype(F32)
    T = T if T is not None else W * W
    got, T_batch, hits = autograd_grad(cost, start, goal, obst, G, g_ratio, T)
    lit = oracle.forward(cost, start, goal, obst, g_ratio=g_ratio, mode="literal", T=T, mechanism="news")
    assert lit.T_batch == T_batch
    if T < W * W:
        assert (lit.t_solve == -1).any() and T_batch == T
    else:
        assert (hits >= 2).any()
    want = oracle.backward(cost, start, goal, obst, G, T_batch, g_ratio=g_ratio, dtype=np.float64, mechanism="news")
    assert np.abs(want).max() > 0
    assert _relerr(want, got) < 1e-9
