"""The 4-connected (NEWS) search without a GPU: the C oracle's NEWS mode (oracle/astar_oracle.c) against the reference's own outputs
(tests/golden/news/, made by tests/golden/make_golden_news.py), the NEWS heuristic, the planners' `mechanism` keyword
and the C ABI's rejection of an unknown mechanism."""
import ctypes
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from golden_util import Golden
from oracle import oracle

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

NEWS_GOLDENS = ["news/news_mazes032_vanilla", "news/news_mazes032_neural", "news/news_all064_vanilla",
                "news/news_large128_learned"]
EINVAL = 1


def _relerr(a, b):
    return float(np.abs(a - b).max() / (np.abs(b).max() + 1e-30))


def _forward(g, mode, **kw):
    return oracle.forward(g.cost, g.start, g.goal, g.obst, g_ratio=g.g_ratio, mode=mode, mechanism="news", **kw)


def spec_batch_coupled(g):
    """SPEC form of the batch-synchronous loop for g_ratio < 0.5: every map steps without early exit, and the state is
    taken after the first step at which all maps select their goal."""
    T = g.W * g.W
    full = _forward(g, "spec", want_trace=True, T=T, no_early_exit=True)
    at_goal = (full.trace == g.z["goal_idx"][:, None]).all(0)
    T_batch = int(np.argmax(at_goal)) + 1 if at_goal.any() else T
    return _forward(g, "spec", want_trace=True, T=T_batch, no_early_exit=True), T_batch


@pytest.mark.parametrize("name", NEWS_GOLDENS)
def test_literal_news_matches_reference(name):
    """LITERAL NEWS = the reference's loop with the generator's NEWS filter and heuristic: masks, T_batch and every
    selection index."""
    g = Golden(name)
    o = _forward(g, "literal", want_trace=True)
    np.testing.assert_array_equal(o.histories != 0, g.bits("hist_bits") != 0)
    np.testing.assert_array_equal(o.paths != 0, g.bits("path_bits") != 0)
    assert o.T_batch == int(g.z["T_batch"])
    np.testing.assert_array_equal(o.trace[:, :o.T_batch], g.z["trace"])


@pytest.mark.parametrize("name", NEWS_GOLDENS)
def test_spec_news_equals_literal(name):
    """SPEC (arg-min of (f, index), per-map early exit) gives the reference's masks; its selections are the
    reference's up to each map's solve step (later reference steps re-select the goal)."""
    g = Golden(name)
    o = _forward(g, "spec", want_trace=True)
    np.testing.assert_array_equal(o.histories != 0, g.bits("hist_bits") != 0)
    np.testing.assert_array_equal(o.paths != 0, g.bits("path_bits") != 0)
    assert o.T_batch == int(g.z["T_batch"])
    for b in range(g.B):
        n = int(o.n_steps[b])
        np.testing.assert_array_equal(o.trace[b, :n], g.z["trace"][b, :n])
        assert (g.z["trace"][b, n:] == g.z["goal_idx"][b]).all()


def test_news_training_mode_and_gradient():
    """Training mode (Tmax 0.25): masks, T_batch and the fp64 closed-form backward against the reference's autograd."""
    g = Golden("news/news_mazes032_neural")
    for mode in ("literal", "spec"):
        o = _forward(g, mode, Tmax=0.25, training=True)
        np.testing.assert_array_equal(o.histories != 0, g.bits("train_hist_bits") != 0)
        np.testing.assert_array_equal(o.paths != 0, g.bits("train_path_bits") != 0)
        assert o.T_batch == int(g.z["train_T_batch"])
    gc = oracle.backward(g.cost, g.start, g.goal, g.obst, g.plane("rand_G"), int(g.z["train_T_batch"]),
                         g_ratio=g.g_ratio, mechanism="news")
    assert _relerr(gc, g.plane("train_grad_cost")) < 1e-5


def test_news_batch_coupled_low_g_ratio():
    """g_ratio = 0.2: the batch-coupled loop in LITERAL and SPEC form, and the backward over its T_batch steps."""
    g = Golden("news/news_mazes032_lowg")
    o = _forward(g, "literal", want_trace=True)
    np.testing.assert_array_equal(o.histories != 0, g.bits("hist_bits") != 0)
    np.testing.assert_array_equal(o.paths != 0, g.bits("path_bits") != 0)
    assert o.T_batch == int(g.z["T_batch"])
    s, T_batch = spec_batch_coupled(g)
    assert T_batch == int(g.z["T_batch"])
    np.testing.assert_array_equal(s.histories != 0, g.bits("hist_bits") != 0)
    np.testing.assert_array_equal(s.trace, g.z["trace"])
    gc = oracle.backward(g.cost, g.start, g.goal, g.obst, g.plane("rand_G"), T_batch, g_ratio=g.g_ratio,
                         mechanism="news")
    assert _relerr(gc, g.plane("rand_grad_cost")) < 1e-5


def test_news_paths_never_move_diagonally():
    g = Golden("news/news_mazes032_vanilla")
    o = _forward(g, "spec")
    for b in np.flatnonzero(o.t_solve >= 0):
        ys, xs = np.nonzero(o.paths[b, 0])
        cells = set(zip(ys.tolist(), xs.tolist()))
        for y, x in cells:   # consecutive path cells are 4-neighbours, so every cell has one on the path
            deg = sum((y + dy, x + dx) in cells for dy, dx in ((-1, 0), (1, 0), (0, -1), (0, 1)))
            assert deg >= 1


def test_get_news_heuristic_equals_the_generator():
    from neural_astar.planner.differentiable_astar import get_news_heuristic

    g = Golden("news/news_mazes032_neural")
    idx = g.z["heur_goal_idx"]
    goal = torch.zeros(len(idx), 1, 32, 32)
    goal.view(len(idx), -1)[torch.arange(len(idx)), torch.from_numpy(idx).long()] = 1
    h = get_news_heuristic(goal[:, 0])
    assert torch.equal(h, torch.from_numpy(g.z["heur_values"]))
    # the expression over any H x W: a non-square plane equals the square one's top-left block
    hs = get_news_heuristic(torch.nn.functional.pad(goal[:, 0], (0, 8)))
    assert torch.equal(hs[..., :32], h)


def test_mechanism_keyword():
    from neural_astar.planner import NeuralAstar, VanillaAstar
    from neural_astar.planner.differentiable_astar import DifferentiableAstar, get_heuristic, get_news_heuristic

    news = torch.zeros(1, 1, 3, 3)
    news[0, 0, 0, 1] = news[0, 0, 1, 0] = news[0, 0, 1, 2] = news[0, 0, 2, 1] = 1
    moore = torch.ones(1, 1, 3, 3)
    moore[0, 0, 1, 1] = 0
    for planner in (VanillaAstar(mechanism="news"), NeuralAstar(mechanism="news")):
        assert planner.astar.mechanism == "news"
        assert torch.equal(planner.state_dict()["astar.neighbor_filter"], news)
        assert planner.astar.get_heuristic is get_news_heuristic
    for planner in (VanillaAstar(), NeuralAstar(), DifferentiableAstar()):
        astar = getattr(planner, "astar", planner)
        assert astar.mechanism == "moore"
        assert torch.equal(astar.state_dict()["neighbor_filter"], moore)
        assert astar.get_heuristic is get_heuristic
    for make in (lambda: DifferentiableAstar(mechanism="bogus"), lambda: VanillaAstar(mechanism="Moore"),
                 lambda: NeuralAstar(mechanism="news8")):
        with pytest.raises(ValueError):
            make()
    with pytest.raises(NotImplementedError):
        VanillaAstar(use_differentiable_astar=False, mechanism="news")
    VanillaAstar(use_differentiable_astar=False)   # the Moore heap search stays available
    with pytest.raises(TypeError):                  # keyword-only: __init__ keeps the reference's parameters
        VanillaAstar(0.5, True, "news")


def test_planner_module_baseline_follows_the_planner():
    from neural_astar.planner import NeuralAstar
    from neural_astar.utils.training import PlannerModule

    assert PlannerModule(NeuralAstar(mechanism="news"), None).vanilla_astar.astar.mechanism == "news"
    assert PlannerModule(NeuralAstar(), None).vanilla_astar.astar.mechanism == "moore"


@pytest.fixture(scope="module")
def native():
    subprocess.check_call(["make", "-C", os.path.join(ROOT, "neural-astar_b200"), "-s", "all"])
    from neural_astar import _native

    return _native


def test_backward_mech_rejects_an_unknown_mechanism_without_a_launch(native):
    L = native.lib()
    p = native.BwdParams()
    dummy = ctypes.c_void_p(16)
    for name in ("cost", "start", "goal", "obst", "grad_histories", "grad_cost", "T_batch", "t_solve"):
        setattr(p, name, dummy.value)
    p.B, p.H, p.W = 1, 8, 8
    before = L.nastar_b200_launch_count()
    for mech in (-1, 2, 7):
        assert L.nastar_b200_backward_mech(ctypes.byref(p), mech, None) == EINVAL
    p.cost = None   # the plain entry point keeps validating as before
    assert L.nastar_b200_backward(ctypes.byref(p), None) == EINVAL
    assert L.nastar_b200_launch_count() == before
    with pytest.raises(ValueError):
        native.mechanism_code("diagonal")
