"""The 4-connected (NEWS) search on the GPU: every engine it runs on (1, 4, 2, 3; engine 5 is Moore-only) against the
reference's own outputs (tests/golden/news/) and against the C oracle's NEWS SPEC form, the backward, the fused
cost hand-offs, the pair launch, the batch-coupled path, the graphed and pipelined planners, and optimal paths on
maps labelled with the NEWS mechanism."""
import numpy as np
import pytest
import torch

from golden_util import Golden
from grad_bound import assert_within_bound, relerr_to_max
from oracle import labels as label_oracle
from oracle import oracle

pytestmark = pytest.mark.gpu


def _cu(x):
    return torch.from_numpy(np.ascontiguousarray(x)).cuda()


def _bits(x):
    return x.detach().cpu().numpy() != 0


def _problems(B, H, W, seed, learned=True, p_obst=0.25):
    """Random maps with start and goal in one 4-connected region (so every map is solvable), optional learned costs."""
    rs = np.random.RandomState(seed)
    maps = (rs.rand(B, 1, H, W) >= p_obst).astype(np.float32)
    start = np.zeros_like(maps)
    goal = np.zeros_like(maps)
    for b in range(B):
        while True:
            free = np.flatnonzero(maps[b, 0].reshape(-1))
            gi = int(free[rs.randint(len(free))])
            d = label_oracle.opt_labels(maps[b:b + 1], np.array([gi]), mechanism="news")[0].reshape(-1)
            cand = np.flatnonzero((d > -(H * W)) & (d < 0))
            if len(cand):
                break
            maps[b, 0].reshape(-1)[gi] = 0.0 if len(free) > 1 else 1.0
        goal[b, 0].reshape(-1)[gi] = 1.0
        start[b, 0].reshape(-1)[int(cand[rs.randint(len(cand))])] = 1.0
    cost = rs.rand(B, 1, H, W).astype(np.float32) if learned else maps
    return cost, start, goal, maps


# ------------------------------------------------------------------------------------------------ reference goldens
@pytest.mark.parametrize("name", ["news/news_mazes032_vanilla", "news/news_all064_vanilla"])
def test_vanilla_goldens(name):
    from neural_astar.planner import VanillaAstar

    g = Golden(name)
    with torch.no_grad():
        out = VanillaAstar(mechanism="news").cuda()(_cu(g.obst), _cu(g.start), _cu(g.goal))
    np.testing.assert_array_equal(_bits(out.histories), g.bits("hist_bits") != 0)
    np.testing.assert_array_equal(_bits(out.paths), g.bits("path_bits") != 0)


@pytest.mark.parametrize("name", ["news/news_mazes032_neural", "news/news_large128_learned"])
def test_learned_cost_goldens(name):
    from neural_astar import _native

    g = Golden(name)
    with torch.no_grad():
        hist, paths, _, _, trace = _native.forward(_cu(g.cost), _cu(g.start), _cu(g.goal), _cu(g.obst), 0.5,
                                                  g.W * g.W, want_trace=True, mechanism="news")
    np.testing.assert_array_equal(_bits(hist), g.bits("hist_bits") != 0)
    np.testing.assert_array_equal(_bits(paths), g.bits("path_bits") != 0)
    tr = trace.cpu().numpy()
    for b in range(g.B):
        n = int((tr[b] >= 0).sum())
        np.testing.assert_array_equal(tr[b, :n], g.z["trace"][b, :n])


def test_training_batch_and_gradient_golden():
    from neural_astar.planner.differentiable_astar import DifferentiableAstar

    g = Golden("news/news_mazes032_neural")
    astar = DifferentiableAstar(Tmax=0.25, mechanism="news").cuda().train()
    cost = _cu(g.cost).requires_grad_(True)
    out = astar(cost, _cu(g.start), _cu(g.goal), _cu(g.obst))
    (out.histories * _cu(g.plane("rand_G"))).sum().backward()
    np.testing.assert_array_equal(_bits(out.histories), g.bits("train_hist_bits") != 0)
    np.testing.assert_array_equal(_bits(out.paths), g.bits("train_path_bits") != 0)
    assert relerr_to_max(cost.grad.cpu().numpy(), g.plane("train_grad_cost")) < 1e-5


def test_batch_coupled_low_g_ratio_golden():
    """g_ratio = 0.2: the module's batch-coupled path (trace search, then exactly T_batch steps) and its backward."""
    from neural_astar.planner.differentiable_astar import DifferentiableAstar

    g = Golden("news/news_mazes032_lowg")
    astar = DifferentiableAstar(g_ratio=0.2, mechanism="news").cuda().eval()
    cost = _cu(g.cost).requires_grad_(True)
    out = astar(cost, _cu(g.start), _cu(g.goal), _cu(g.obst))
    (out.histories * _cu(g.plane("rand_G"))).sum().backward()
    np.testing.assert_array_equal(_bits(out.histories), g.bits("hist_bits") != 0)
    np.testing.assert_array_equal(_bits(out.paths), g.bits("path_bits") != 0)
    assert relerr_to_max(cost.grad.cpu().numpy(), g.plane("rand_grad_cost")) < 1e-5


# ------------------------------------------------------------------------------------------------ oracle, every engine
SHAPES = [(12, 12), (5, 40), (32, 32), (33, 31), (64, 64), (65, 64), (128, 128), (131, 131), (131, 132)]


@pytest.mark.parametrize("learned", [True, False], ids=["learned", "binary"])
@pytest.mark.parametrize("H,W", SHAPES)
def test_random_vs_spec_oracle(H, W, learned):
    """histories, paths, t_solve, n_steps and the selection trace, bit for bit, on both sides of every engine
    boundary.  `binary` passes the obstacle plane as the cost (VanillaAstar): above 64x64 that is engine 5's input for
    Moore, and NEWS must run it on engine 2/3."""
    from neural_astar import _native

    B = 6 if H * W > 4096 else 12
    cost, start, goal, maps = _problems(B, H, W, 1000 * H + W + learned, learned)
    T = W * W
    c = _cu(cost)
    obst = c if not learned else _cu(maps)
    hist, paths, ts, ns, trace = _native.forward(c, _cu(start), _cu(goal), obst, 0.5, T, want_trace=True,
                                                 mechanism="news")
    ref = oracle.forward(cost, start, goal, maps, mode="spec", want_trace=True, T=T, mechanism="news")
    np.testing.assert_array_equal(hist.cpu().numpy(), ref.histories)
    np.testing.assert_array_equal(paths.cpu().numpy(), ref.paths)
    np.testing.assert_array_equal(ts.cpu().numpy(), ref.t_solve)
    np.testing.assert_array_equal(ns.cpu().numpy(), ref.n_steps)
    np.testing.assert_array_equal(trace.cpu().numpy(), ref.trace)
    assert (ref.t_solve >= 0).all()


@pytest.mark.parametrize("H,W,engine", [(32, 32, 1), (64, 64, 4), (100, 100, 2), (131, 132, 3)])
def test_backward_vs_oracle(H, W, engine):
    from neural_astar import _native
    from neural_astar.planner.differentiable_astar import DifferentiableAstar

    assert _native.lib().nastar_b200_engine_for(H, W) == engine
    cost, start, goal, maps = _problems(4, H, W, 7 * H + W)
    G = np.random.RandomState(H).randn(4, 1, H, W).astype(np.float32)
    astar = DifferentiableAstar(Tmax=0.25, mechanism="news").cuda().train()
    c = _cu(cost).requires_grad_(True)
    out = astar(c, _cu(start), _cu(goal), _cu(maps))
    (out.histories * _cu(G)).sum().backward()
    T = int(0.25 * W * W)
    ref = oracle.forward(cost, start, goal, maps, mode="spec", T=T, mechanism="news")
    np.testing.assert_array_equal(out.histories.detach().cpu().numpy(), ref.histories)
    T_batch = T if (ref.t_solve < 0).any() else int(ref.t_solve.max()) + 1
    want, M = oracle.backward_with_bound(cost, start, goal, maps, G, T_batch, mechanism="news")
    assert_within_bound(c.grad.cpu().numpy(), want, M, "news module training", mechanism="news")


# ------------------------------------------------------------------------------------------------ launch forms
@pytest.mark.parametrize("H,W", [(32, 32), (64, 64)])
def test_cost_taps_equal_the_plane_search(H, W):
    from neural_astar import _native
    from neural_astar.planner.differentiable_astar import DifferentiableAstar

    _, start, goal, maps = _problems(8, H, W, H + 3)
    taps = torch.randn(8, H, W, 9, device="cuda") * 0.5
    bias, scale = 0.1, 2.0
    astar = DifferentiableAstar(mechanism="news").cuda().eval()
    s, g, o = _cu(start), _cu(goal), _cu(maps)
    with torch.no_grad():
        want = astar(_native.cost_from_taps(taps, bias, scale), s, g, o)
        got = astar.search_from_taps(taps, bias, scale, s, g, o)
    assert torch.equal(got.histories, want.histories) and torch.equal(got.paths, want.paths)


@pytest.mark.parametrize("H,W", [(32, 32), (64, 64), (100, 100)])
def test_pair_launch_equals_two_calls(H, W):
    from neural_astar import _native

    cost, start, goal, maps = _problems(8, H, W, 5 * H)
    c, s, g, o = _cu(cost), _cu(start), _cu(goal), _cu(maps)
    pair = _native.forward(c, s, g, o, 0.5, W * W, want_trace=True, pair=True, mechanism="news")
    one = _native.forward(c, s, g, o, 0.5, W * W, want_trace=True, mechanism="news")
    two = _native.forward(o, s, g, o, 0.5, W * W, want_trace=True, mechanism="news")
    for k in range(5):
        assert torch.equal(pair[k], torch.cat([one[k], two[k]])), k


@pytest.mark.parametrize("H,W", [(32, 32), (64, 64), (100, 100), (200, 200)])
def test_news_makes_as_many_launches_as_moore(H, W):
    from neural_astar import _native

    cost, start, goal, maps = _problems(4, H, W, H)
    args = (_cu(cost), _cu(start), _cu(goal), _cu(maps), 0.5, W * W)
    counts = {}
    for mech in ("moore", "news", "moore", "news"):   # the second round: the heuristic tables are filled
        before = _native.launch_count()
        _native.forward(*args, mechanism=mech)
        counts[mech] = _native.launch_count() - before
    assert counts["news"] == counts["moore"] == 1


def test_binary_256_skips_engine_5():
    """A NEWS VanillaAstar at 256x256 (Moore would offer it to engine 5 first) equals the oracle in one launch."""
    from neural_astar import _native
    from neural_astar.planner import VanillaAstar

    _, start, goal, maps = _problems(2, 256, 256, 256, learned=False)
    planner = VanillaAstar(mechanism="news").cuda()
    m, s, g = _cu(maps), _cu(start), _cu(goal)
    with torch.no_grad():
        planner(m, s, g)
        before = _native.launch_count()
        out = planner(m, s, g)
        assert _native.launch_count() - before == 1
    ref = oracle.forward(maps, start, goal, maps, mode="spec", mechanism="news")
    np.testing.assert_array_equal(out.histories.cpu().numpy(), ref.histories)
    np.testing.assert_array_equal(out.paths.cpu().numpy(), ref.paths)


# ------------------------------------------------------------------------------------------------ end to end
@pytest.mark.parametrize("H,W", [(32, 32), (64, 64), (100, 100)])
def test_paths_are_news_optimal_on_news_labels(H, W):
    """On maps labelled by compute_opt_labels(..., mechanism="news"), a NEWS VanillaAstar path has exactly
    -opt_dists[start] + 1 cells (h's tie-break term stays below 1 on these sizes, so the search is optimal on unit
    costs), and consecutive cells are 4-neighbours."""
    from neural_astar.planner import VanillaAstar
    from neural_astar.utils.data import compute_opt_labels

    _, start, goal, maps = _problems(16, H, W, 3 * H, learned=False)
    _, dists, _ = compute_opt_labels(_cu(maps), _cu(goal), mechanism="news")
    with torch.no_grad():
        out = VanillaAstar(mechanism="news").cuda()(_cu(maps), _cu(start), _cu(goal))
    d = dists.cpu().numpy().reshape(16, -1)
    si = start.reshape(16, -1).argmax(1)
    paths = out.paths.cpu().numpy()[:, 0]
    for b in range(16):
        assert paths[b].sum() == -d[b, si[b]] + 1
        ys, xs = np.nonzero(paths[b])
        cells = set(zip(ys.tolist(), xs.tolist()))
        for y, x in cells:
            assert any((y + dy, x + dx) in cells for dy, dx in ((-1, 0), (1, 0), (0, -1), (0, 1)))


def _ckpt_news_planner():
    import os

    from neural_astar.planner import NeuralAstar

    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    state = np.load(os.path.join(root, "tests", "golden", "mazes032_ckpt_planner_state.npz"))
    na = NeuralAstar(encoder_arch="CNN", mechanism="news")
    sd = {k: torch.from_numpy(state[k]) for k in state.files}
    sd["astar.neighbor_filter"] = na.astar.neighbor_filter.detach().clone()
    na.load_state_dict(sd)
    return na.cuda().eval()


def test_graphed_and_pipelined_planners_match_eager():
    from neural_astar.planner import VanillaAstar
    from neural_astar.utils.inference import GraphedPlanner, PipelinedPlanner

    g = Golden("news/news_mazes032_vanilla")
    na = _ckpt_news_planner()
    maps, start, goal = (_cu(x) for x in (g.obst, g.start, g.goal))
    torch.manual_seed(0)
    batches = []
    for _ in range(3):
        perm = torch.randperm(100, device="cuda")
        batches.append((maps[perm], start[perm], goal[perm]))
    with torch.no_grad():
        want = [na(*b) for b in batches]
        neural = Golden("news/news_mazes032_neural")
        eager0 = na(maps, start, goal)
    np.testing.assert_array_equal(_bits(eager0.histories), neural.bits("hist_bits") != 0)
    graphed = GraphedPlanner(na, maps, start, goal)
    for b, w in zip(batches, want):
        got = graphed(*b)
        assert torch.equal(got.histories, w.histories) and torch.equal(got.paths, w.paths)
    pipe = PipelinedPlanner(na, maps, start, goal)
    got = []
    for b in batches:
        prev = pipe.submit(*b)
        if prev is not None:
            got.append((prev.histories.clone(), prev.paths.clone()))
    last = pipe.drain()
    got.append((last.histories.clone(), last.paths.clone()))
    for (h, p), w in zip(got, want):
        assert torch.equal(h, w.histories) and torch.equal(p, w.paths)
    va = GraphedPlanner(VanillaAstar(mechanism="news").cuda().eval(), maps, start, goal)
    out = va.replay()
    np.testing.assert_array_equal(_bits(out.histories), g.bits("hist_bits") != 0)
    np.testing.assert_array_equal(_bits(out.paths), g.bits("path_bits") != 0)


def test_pair_validation_uses_the_planners_mechanism():
    from neural_astar.planner import VanillaAstar

    g = Golden("news/news_mazes032_vanilla")
    na = _ckpt_news_planner()
    maps, start, goal = (_cu(x) for x in (g.obst, g.start, g.goal))
    with torch.no_grad():
        learned, vanilla, _ = na.forward_pair(maps, start, goal)
        want = na(maps, start, goal)
        want_v = VanillaAstar(mechanism="news").cuda()(maps, start, goal)
    assert torch.equal(learned.histories, want.histories) and torch.equal(learned.paths, want.paths)
    assert torch.equal(vanilla.histories, want_v.histories) and torch.equal(vanilla.paths, want_v.paths)


def test_graphed_train_step_on_a_news_dataset():
    """GraphedTrainStep on a DeviceMazeDataset batch of NEWS labels: the same losses as the eager steps."""
    from types import SimpleNamespace

    from neural_astar.planner import NeuralAstar
    from neural_astar.utils.data import DeviceMazeDataset, compute_opt_labels
    from neural_astar.utils.training import GraphedTrainStep, PlannerModule

    g = Golden("news/news_mazes032_vanilla")
    maps, goal = _cu(g.obst), _cu(g.goal)
    policies, dists, _ = compute_opt_labels(maps, goal, mechanism="news")
    ds = DeviceMazeDataset.from_labels(maps, goal, policies, dists)
    gen = torch.Generator(device="cuda").manual_seed(3)
    batch = list(ds.sample(torch.arange(64, device="cuda"), generator=gen))

    def make():
        torch.manual_seed(1234)
        planner = NeuralAstar(encoder_input="m+", encoder_arch="CNN", encoder_depth=4, Tmax=0.25, mechanism="news")
        return PlannerModule(planner, SimpleNamespace(params=SimpleNamespace(lr=1e-3))).cuda().train()

    eager = make()
    opt = eager.configure_optimizers()
    eager_losses = []
    for step in range(3):
        opt.zero_grad()
        loss = eager.training_step(batch, step)
        loss.backward()
        opt.step()
        eager_losses.append(float(loss))
    graphed = make()
    step_fn = GraphedTrainStep(graphed, batch)
    graph_losses = [float(step_fn(batch)) for _ in range(3)]
    np.testing.assert_allclose(graph_losses, eager_losses, rtol=2e-3)
