"""The batch-coupled search for g_ratio < 0.5 with T_batch decided on the device (_native.forward_coupled,
nastar_b200_forward_coupled) against the host procedure it replaces (_coupled_steps, then a NO_EARLY_EXIT search of
exactly T_batch steps), the reference's goldens, and the graphed wrappers that can now capture such batches."""
import numpy as np
import pytest
import torch

from golden_util import Golden
from grad_bound import relerr_to_max

pytestmark = pytest.mark.gpu
TOL = 1e-5


def _cu(x):
    return torch.from_numpy(np.ascontiguousarray(x)).cuda()


def _problems(B, H, W, seed, kinds=None, p_obst=0.2, cost_scale=10.0):
    """Random maps with costs x `cost_scale` (the cost a NeuralAstar hands the search, scaled up so that low g_ratio
    searches wander after their solve step).  `kinds[b]`: "normal" (random start and goal), "same" (start == goal),
    "walled" (the start is walled in: the open set empties), "capped" (obstacle-free map with a walled-in goal: more
    reachable cells than steps)."""
    rs = np.random.RandomState(seed)
    kinds = kinds or ["normal"] * B
    maps = (rs.rand(B, 1, H, W) >= p_obst).astype(np.float32)
    start = np.zeros_like(maps)
    goal = np.zeros_like(maps)
    for b, kind in enumerate(kinds):
        sy, sx = rs.randint(1, H - 1), rs.randint(1, W - 1)
        gy, gx = rs.randint(1, H - 1), rs.randint(1, W - 1)
        if kind == "same":
            gy, gx = sy, sx
        if kind == "capped":
            maps[b, 0] = 1
            maps[b, 0, gy - 1:gy + 2, gx - 1:gx + 2] = 0
            if abs(sy - gy) <= 1 and abs(sx - gx) <= 1:
                sy, sx = (gy + H // 2) % H, (gx + W // 2) % W
        if kind == "walled":
            maps[b, 0, max(sy - 1, 0):sy + 2, max(sx - 1, 0):sx + 2] = 0
            if abs(sy - gy) <= 1 and abs(sx - gx) <= 1:
                gy, gx = (sy + H // 2) % H, (sx + W // 2) % W
        maps[b, 0, sy, sx] = maps[b, 0, gy, gx] = 1
        start[b, 0, sy, sx] = 1
        goal[b, 0, gy, gx] = 1
    cost = (rs.rand(B, 1, H, W) * cost_scale).astype(np.float32)
    return cost, start, goal, maps


def _host(cost, start, goal, obst, g_ratio, T, mechanism):
    """The host procedure of DifferentiableAstar.forward: trace search, host decision, then T_batch steps."""
    from neural_astar import _native
    from neural_astar.planner.differentiable_astar import _coupled_steps

    T_batch, clamped = _coupled_steps(cost, start, goal, obst, g_ratio, T, mechanism)
    hist, paths, ts, ns, _, counts = _native.forward(cost, start, goal, obst, g_ratio, T_batch, no_early_exit=True,
                                                     want_counts=True, mechanism=mechanism)
    clamp = torch.where(clamped, torch.zeros_like(ts), torch.full_like(ts, T_batch))
    return hist, paths, ts, ns, T_batch, clamp, counts


def _compare(cost, start, goal, obst, g_ratio, T, mechanism, **kw):
    from neural_astar import _native

    got = _native.forward_coupled(cost, start, goal, obst, g_ratio, T, mechanism=mechanism, want_counts=True, **kw)
    want = _host(cost, start, goal, obst, g_ratio, T, mechanism)
    hist, paths, ts, ns, Tb, clamp, counts = got
    assert int(Tb.item()) == want[4]
    for a, b in ((hist, want[0]), (paths, want[1]), (ts, want[2]), (ns, want[3]), (clamp, want[5]),
                 (counts[0], want[6][0]), (counts[1], want[6][1])):
        assert torch.equal(a, b)
    return want


def _engine(H, W):
    from neural_astar import _native

    return _native.lib().nastar_b200_engine_for(H, W)


SHAPES = [(12, 12, 1), (32, 32, 1), (33, 31, 4), (64, 64, 4), (48, 40, 4), (100, 72, 2), (144, 136, 3)]


@pytest.mark.parametrize("mechanism", ["moore", "news"])
@pytest.mark.parametrize("g_ratio", [0.0, 0.2, 0.3, 0.45])
@pytest.mark.parametrize("H,W,engine", SHAPES)
@pytest.mark.parametrize("Tmax", [1.0, 0.25])
def test_forward_coupled_equals_host_procedure(H, W, engine, g_ratio, mechanism, Tmax):
    assert _engine(H, W) == engine
    B = 8 if H * W > 4096 else 16
    cost, start, goal, maps = _problems(B, H, W, 31 * H + W + int(100 * g_ratio))
    T = int(Tmax * W * W)
    _compare(_cu(cost), _cu(start), _cu(goal), _cu(maps), g_ratio, T, mechanism)


@pytest.mark.parametrize("mechanism", ["moore", "news"])
@pytest.mark.parametrize("H,W", [(32, 32), (64, 64), (100, 72)])
def test_odd_cap_and_solved_maps_that_wander(H, W, mechanism):
    """T not a multiple of 32, and a batch in which some solved map selects non-goal cells after its solve step (the
    case the coupling exists for)."""
    from neural_astar import _native

    cost, start, goal, maps = _problems(12, H, W, 7 * H + W)
    c, s, g, m = _cu(cost), _cu(start), _cu(goal), _cu(maps)
    T = W * W // 3 + 7
    assert T % 32
    _, _, ts, _, T_batch, _, _ = _compare(c, s, g, m, 0.2, T, mechanism)
    _, _, _, _, trace = _native.forward(c, s, g, m, 0.2, T, want_trace=True, no_early_exit=True, mechanism=mechanism)
    gi = g.reshape(12, -1).argmax(1).to(torch.int32)
    wander = False
    for b in range(12):
        t0 = int(ts[b])
        if 0 <= t0 < T_batch - 1:
            wander |= bool((trace[b, t0 + 1:T_batch] != gi[b]).any())
    assert wander


@pytest.mark.parametrize("mechanism", ["moore", "news"])
@pytest.mark.parametrize("H,W", [(32, 32), (64, 64), (100, 72), (144, 136)])
def test_mixed_batch_and_no_common_goal_step(H, W, mechanism):
    kinds = ["normal", "same", "walled", "capped", "normal", "normal", "same", "normal"]
    cost, start, goal, maps = _problems(len(kinds), H, W, 3 * H + W, kinds=kinds)
    T = W * W // 4
    want = _compare(_cu(cost), _cu(start), _cu(goal), _cu(maps), 0.3, T, mechanism)
    assert want[4] == T                      # the capped and the walled-in map never select their goal
    ts = want[2].cpu().numpy()
    assert ts[2] == -2 and ts[3] == -1 and ts[1] == 0
    # the same batch without its two unsolvable maps
    keep = [0, 1, 4, 5, 6, 7]
    _compare(*(_cu(x[keep]) for x in (cost, start, goal, maps)), 0.3, T, mechanism)


@pytest.mark.parametrize("name", ["mazes032_lowg_gr00_cost10", "mazes032_lowg_gr02", "mazes032_lowg_gr04_cost10",
                                  "news/news_mazes032_lowg", "news/news_all064_lowg"])
def test_goldens_masks_T_batch_and_captured_gradient(name):
    from neural_astar import _native
    from neural_astar.planner.differentiable_astar import DifferentiableAstar

    g = Golden(name)
    mech = g.meta.get("mechanism", "moore")
    cost, start, goal, obst = _cu(g.cost), _cu(g.start), _cu(g.goal), _cu(g.obst)
    T = g.W * g.W
    hist, paths, _, _, T_batch, _ = _native.forward_coupled(cost, start, goal, obst, g.g_ratio, T, mechanism=mech)
    assert int(T_batch.item()) == int(g.z["T_batch"])
    np.testing.assert_array_equal(hist.cpu().numpy() != 0, g.bits("hist_bits") != 0)
    np.testing.assert_array_equal(paths.cpu().numpy() != 0, g.bits("path_bits") != 0)
    # forward + backward captured in one graph: the module takes the device procedure while capturing
    astar = DifferentiableAstar(g_ratio=g.g_ratio, mechanism=mech).cuda().eval()
    c = cost.clone().requires_grad_(True)
    G = _cu(g.plane("rand_G").astype(np.float32))
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):   # warm-up (host procedure, eager)
        torch.autograd.grad((astar(c, start, goal, obst).histories * G).sum(), c)
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        out = astar(c, start, goal, obst)
        grad, = torch.autograd.grad((out.histories * G).sum(), c)
    graph.replay()
    torch.cuda.synchronize()
    np.testing.assert_array_equal(out.histories.detach().cpu().numpy() != 0, g.bits("hist_bits") != 0)
    assert relerr_to_max(grad.cpu().numpy(), g.plane("rand_grad_cost")) < TOL


@pytest.mark.parametrize("mechanism", ["moore", "news"])
@pytest.mark.parametrize("H,W", [(32, 32), (48, 40), (64, 64)])
def test_taps_and_logit_equal_the_plane(H, W, mechanism):
    from neural_astar import _native

    B = 10
    _, start, goal, maps = _problems(B, H, W, 5 * H + W)
    rs = np.random.RandomState(H)
    taps = _cu(rs.randn(B, H, W, 9).astype(np.float32))
    logit = _cu(rs.randn(B, 1, H, W).astype(np.float32) * 3)
    s, g, m = _cu(start), _cu(goal), _cu(maps)
    T = W * W
    for kind, src, bias, scale in ((_native.COST_TAPS, taps, 0.3, 10.0), (_native.COST_LOGIT, logit, 0.0, 10.0)):
        plane = (_native.cost_from_taps(src, bias, scale) if kind == _native.COST_TAPS
                 else torch.sigmoid(src) * scale)
        a = _native.forward_coupled(src, s, g, m, 0.2, T, cost_kind=kind, cost_scale=scale, cost_bias=bias,
                                    mechanism=mechanism)
        b = _native.forward_coupled(plane, s, g, m, 0.2, T, mechanism=mechanism)
        for x, y in zip(a, b):
            assert torch.equal(x, y)


@pytest.mark.parametrize("B", [2, 300])
def test_three_launches_and_graph_replay_on_new_inputs(B):
    from neural_astar import _native

    H = W = 32
    T = W * W
    cost, start, goal, maps = _problems(B, H, W, B)
    ins = [_cu(x) for x in (cost, start, goal, maps)]
    _native.forward_coupled(*ins, 0.2, T)
    before = _native.launch_count()
    _native.forward_coupled(*ins, 0.2, T)
    assert _native.launch_count() - before == 3
    torch.cuda.synchronize()
    static = [x.clone() for x in ins]
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):   # a host synchronisation would make the capture fail
        out = _native.forward_coupled(*static, 0.2, T)
    for seed in (B + 1, B + 2):
        new = [_cu(x) for x in _problems(B, H, W, seed)]
        for d, s_ in zip(static, new):
            d.copy_(s_)
        graph.replay()
        want = _native.forward_coupled(*new, 0.2, T)
        for x, y in zip(out, want):
            assert torch.equal(x, y)


def _ckpt_planner(g_ratio, mechanism="moore"):
    import os

    from neural_astar.planner import NeuralAstar

    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    state = np.load(os.path.join(root, "tests", "golden", "mazes032_ckpt_planner_state.npz"))
    na = NeuralAstar(g_ratio=g_ratio, encoder_arch="CNN", mechanism=mechanism)
    sd = {k: torch.from_numpy(state[k]) for k in state.files}
    sd["astar.neighbor_filter"] = na.astar.neighbor_filter.detach().clone()
    na.load_state_dict(sd)
    return na.cuda().eval()


def _batches(maps, start, goal, n=3):
    torch.manual_seed(0)
    out = []
    for _ in range(n):
        perm = torch.randperm(maps.shape[0], device="cuda")
        out.append((maps[perm], start[perm], goal[perm]))
    return out


@pytest.mark.parametrize("mechanism", ["moore", "news"])
def test_graphed_planners_low_g_ratio(mechanism):
    from neural_astar.planner import VanillaAstar
    from neural_astar.utils.inference import GraphedPlanner

    g = Golden("mazes032_vanilla_test")
    maps, start, goal = _cu(g.obst), _cu(g.start), _cu(g.goal)
    batches = _batches(maps, start, goal)
    for planner in (VanillaAstar(g_ratio=0.2, mechanism=mechanism).cuda().eval(), _ckpt_planner(0.3, mechanism)):
        with torch.no_grad():
            want = [planner(*b) for b in batches]
        graphed = GraphedPlanner(planner, maps, start, goal)
        for b, w in zip(batches, want):
            got = graphed(*b)
            assert torch.equal(got.histories, w.histories) and torch.equal(got.paths, w.paths)
        with pytest.raises(ValueError):
            graphed(maps, start, goal, store_intermediate_results=True)


@pytest.mark.parametrize("host", [False, True])
def test_pipelined_planner_low_g_ratio(host):
    from neural_astar.utils.inference import PipelinedPlanner

    g = Golden("mazes032_vanilla_test")
    maps, start, goal = _cu(g.obst), _cu(g.start), _cu(g.goal)
    na = _ckpt_planner(0.3)
    batches = _batches(maps, start, goal, n=4)
    with torch.no_grad():
        want = [na(*b) for b in batches]
    pipe = PipelinedPlanner(na, maps, start, goal, host=host)
    got = {}   # batch index -> (histories, paths), cloned before the graph-owned buffers are reused
    for k, b in enumerate(batches):
        if host:
            for d, s_ in zip(pipe.host_inputs[k % 3], b):
                d.copy_(s_.cpu())
            prev, done = pipe.submit(), k - 2
        else:
            prev, done = pipe.submit(*b), k - 1
        if prev is not None:
            got[done] = (prev.histories.clone(), prev.paths.clone())
    last = pipe.drain()
    got[len(batches) - 1] = (last.histories.clone(), last.paths.clone())
    assert len(got) >= 3
    for k, (h, p) in got.items():
        assert torch.equal(h, want[k].histories) and torch.equal(p, want[k].paths), k


@pytest.mark.parametrize("mechanism", ["moore", "news"])
def test_graphed_train_step_low_g_ratio(mechanism):
    from types import SimpleNamespace

    from neural_astar.planner import NeuralAstar
    from neural_astar.utils.data import DeviceMazeDataset, compute_opt_labels
    from neural_astar.utils.training import GraphedTrainStep, PlannerModule

    g = Golden("mazes032_vanilla_test")
    maps, goal = _cu(g.obst), _cu(g.goal)
    policies, dists, _ = compute_opt_labels(maps, goal, mechanism=mechanism)
    ds = DeviceMazeDataset.from_labels(maps, goal, policies, dists)
    gen = torch.Generator(device="cuda").manual_seed(3)
    batch = list(ds.sample(torch.arange(64, device="cuda"), generator=gen))

    def make():
        torch.manual_seed(1234)
        planner = NeuralAstar(g_ratio=0.3, encoder_input="m+", encoder_arch="CNN", encoder_depth=4, Tmax=0.25,
                              mechanism=mechanism)
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
    step_fn = GraphedTrainStep(make(), batch)
    graph_losses = [float(step_fn(batch)) for _ in range(3)]
    np.testing.assert_allclose(graph_losses, eager_losses, rtol=2e-3)


def test_single_map_under_capture_is_not_coupled():
    from neural_astar.planner import VanillaAstar
    from neural_astar.utils.inference import GraphedPlanner

    g = Golden("mazes032_vanilla_test")
    maps, start, goal = _cu(g.obst[:1]), _cu(g.start[:1]), _cu(g.goal[:1])
    planner = VanillaAstar(g_ratio=0.2).cuda().eval()
    with torch.no_grad():
        want = planner(maps, start, goal)
    graphed = GraphedPlanner(planner, maps, start, goal)
    assert graphed.native_launches_per_replay == 1      # one per-map early-exit search, no coupling
    got = graphed(maps, start, goal)
    assert torch.equal(got.histories, want.histories) and torch.equal(got.paths, want.paths)
