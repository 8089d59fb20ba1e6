"""BB-A* on the H100: BBAstar's forward against NeuralAstar's, the black-box backward against the CPU oracle
(tests/bbastar_oracle.py) bit for bit on every search engine, its launch count, graph capture and its errors."""
from types import SimpleNamespace

import numpy as np
import pytest
import torch

import bbastar_oracle

pytestmark = pytest.mark.gpu
F32 = np.float32
DEV = "cuda"


def _native():
    from neural_astar import _native

    return _native


def _problem(seed, B, H, W, far=None):
    """Random maps, 90 % passable (goals stay reachable, which the coupled oracle's literal loop needs), one start and
    one goal per map, learned-looking costs in [0.1, 1.1).  `far` bounds |start - goal| per axis (keeps the CPU oracle
    quick on large maps)."""
    rng = np.random.RandomState(seed)
    maps = (rng.rand(B, 1, H, W) > 0.1).astype(F32)
    start = np.zeros_like(maps)
    goal = np.zeros_like(maps)
    for b in range(B):
        sy, sx = rng.randint(H), rng.randint(W)
        if far is None:
            gy, gx = rng.randint(H), rng.randint(W)
        else:
            gy, gx = min(H - 1, sy + rng.randint(1, far)), min(W - 1, sx + rng.randint(1, far))
        if (gy, gx) == (sy, sx):
            gy = (sy + 1) % H
        maps[b, 0, sy, sx] = maps[b, 0, gy, gx] = 1
        start[b, 0, sy, sx] = 1
        goal[b, 0, gy, gx] = 1
    cost = (0.1 + rng.rand(B, 1, H, W)).astype(F32)
    return cost, start, goal, maps


def _upstream(seed, shape, lam, negative):
    """An L1-like incoming gradient scaled so that lambda * g moves the search; with `negative`, w' < 0 in row 0."""
    rng = np.random.RandomState(seed + 1)
    g = (np.sign(rng.rand(*shape) - 0.5) * rng.choice([0.0, 0.3, 1.0], shape) / lam).astype(F32)
    if negative:
        g[:, :, 0, :] = F32(-3.0 / lam)
    return g


def _t(x):
    return torch.from_numpy(np.ascontiguousarray(x)).to(DEV)


def _engine(H, W):
    return int(_native().lib().nastar_b200_engine_for(H, W))


# (H, W, engine): every engine the black-box backward runs on
SHAPES = [(32, 32, 1), (20, 12, 1), (64, 64, 4), (40, 64, 4), (100, 100, 2), (256, 256, 3)]
# (g_ratio, B, coupled): per-map exit, a single map below 0.5 (never coupled), a coupled batch
G_CASES = [(0.5, 4, False), (0.7, 3, False), (0.2, 1, False), (0.2, 4, True)]


def _grad_cases():
    for H, W, engine in SHAPES:
        for mech in ("moore", "news"):
            for g_ratio, B, coupled in G_CASES:
                for lam in (20.0, 3.7):
                    if engine == 3 and (lam != 20.0 or g_ratio == 0.7):
                        continue      # the largest maps: fewer combinations
                    yield pytest.param(H, W, engine, mech, g_ratio, B, coupled, lam,
                                       id=f"{H}x{W}-e{engine}-{mech}-g{g_ratio}-B{B}-lam{lam}")


@pytest.mark.parametrize("H,W,engine,mech,g_ratio,B,coupled,lam", list(_grad_cases()))
def test_gradient_equals_oracle(H, W, engine, mech, g_ratio, B, coupled, lam):
    """dL/dw through BlackboxAstar (training mode, Tmax 0.5) equals the oracle's bit for bit, and so do the forward's
    histories; some perturbed costs are negative."""
    from neural_astar.planner.differentiable_astar import BlackboxAstar, batch_coupled

    assert _engine(H, W) == engine
    assert batch_coupled(g_ratio, B) == coupled
    far = 24 if (engine == 3 or (mech == "news" and H * W > 4096)) else None
    cost, start, goal, obst = _problem(H * 7 + W + B, B, H, W, far)
    g = _upstream(H + W + B, cost.shape, lam, negative=True)
    astar = BlackboxAstar(g_ratio=g_ratio, Tmax=0.5, bbastar_lambda=lam, mechanism=mech).to(DEV).train()
    T = astar.num_steps(W)
    w = _t(cost).requires_grad_()
    out = astar(w, _t(start), _t(goal), _t(obst))
    out.histories.backward(_t(g))
    ref = bbastar_oracle.blackbox_backward(cost, start, goal, obst, g, lam, g_ratio, T, mech, coupled)
    assert (ref.costs < 0).any()
    assert np.array_equal(out.histories.detach().cpu().numpy(), ref.histories)
    got = w.grad.cpu().numpy()
    bad = np.argwhere(got != ref.grad)
    assert bad.size == 0, f"{len(bad)} cells differ, first {tuple(bad[0])}: {got[tuple(bad[0])]} vs {ref.grad[tuple(bad[0])]}"
    assert np.abs(ref.grad).sum() > 0, "the perturbation is meant to change some search"


def test_multichannel_cost_gets_channel0_gradient_only():
    from neural_astar.planner.differentiable_astar import BlackboxAstar

    cost, start, goal, obst = _problem(3, 3, 32, 32)
    extra = np.concatenate([cost, 0.5 * cost], 1)
    g = _upstream(3, cost.shape, 20.0, negative=False)
    astar = BlackboxAstar().to(DEV).eval()
    w = _t(extra).requires_grad_()
    astar(w, _t(start), _t(goal), _t(obst)).histories.backward(_t(g))
    ref = bbastar_oracle.blackbox_backward(cost, start, goal, obst, g, 20.0, 0.5, 32 * 32)
    assert np.array_equal(w.grad[:, :1].cpu().numpy(), ref.grad)
    assert not w.grad[:, 1:].any()


@pytest.mark.parametrize("H,W", [(32, 32), (64, 64), (100, 100)])
def test_binding_launches_and_strided_gradient(H, W):
    """The non-coupled backward is one launch, the coupled one three; a strided upstream gradient is read right."""
    nat = _native()
    cost, start, goal, obst = _problem(11, 4, H, W)
    g = _upstream(11, cost.shape, 20.0, negative=False)
    c, s, gl, o = (_t(x) for x in (cost, start, goal, obst))
    T = H * W // 2
    hist = nat.forward(c, s, gl, o, 0.5, T)[0]
    wide = torch.zeros((4, 3, H, W), device=DEV)
    wide[:, 1:2] = _t(g)
    nat.backward_blackbox(c, s, gl, o, hist, _t(g), 20.0, 0.5, T)   # warm-up (heuristic tables)
    torch.cuda.synchronize()
    n0 = nat.launch_count()
    got = nat.backward_blackbox(c, s, gl, o, hist, wide[:, 1:2], 20.0, 0.5, T)
    assert nat.launch_count() - n0 == 1
    ref = bbastar_oracle.blackbox_backward(cost, start, goal, obst, g, 20.0, 0.5, T)
    assert np.array_equal(got.cpu().numpy(), ref.grad)
    n0 = nat.launch_count()
    nat.backward_blackbox(c, s, gl, o, hist, _t(g), 20.0, 0.3, T, coupled=True)
    assert nat.launch_count() - n0 == 3


def _planner_pair(kind, **kw):
    from neural_astar.planner import BBAstar, NeuralAstar

    torch.manual_seed(99)
    na = NeuralAstar(**kw).to(DEV)
    bb = BBAstar(**kw).to(DEV)
    bb.load_state_dict(na.state_dict())
    return na, bb


FWD_CASES = [
    pytest.param(dict(Tmax=0.25), 32, 32, 1, id="32x32"),
    pytest.param(dict(Tmax=0.25), 64, 64, 1, id="64x64"),
    pytest.param(dict(Tmax=0.25), 20, 12, 1, id="20x12"),
    pytest.param(dict(Tmax=0.25, encoder_depth=3), 128, 128, 1, id="128x128"),
    pytest.param(dict(Tmax=0.25, encoder_input="rgb+", encoder_arch="CNNDownSize", encoder_depth=3,
                      learn_obstacles=True), 12, 12, 3,
                 id="rgb+96-CNNDownSize-12x12"),
    pytest.param(dict(Tmax=0.25, g_ratio=0.3), 32, 32, 1, id="32x32-g0.3"),
    pytest.param(dict(Tmax=0.25, learn_obstacles=True, mechanism="news"), 32, 32, 1, id="32x32-news-learn_obstacles"),
]


@pytest.mark.parametrize("kw,H,W,C", FWD_CASES)
@pytest.mark.parametrize("mode", ["train", "eval", "eval-no-grad"])
def test_forward_bit_identical_to_neural_astar(kw, H, W, C, mode):
    """Same weights, same outputs: histories and paths in train and eval mode, and through the fused TAPS search of
    the eval fast path (no grad)."""
    na, bb = _planner_pair("pair", **kw)
    B = 6
    cost, start, goal, maps = _problem(5, B, H, W)
    if C == 3:
        rng = np.random.RandomState(8)
        img = rng.rand(B, 3, 8 * H, 8 * W).astype(F32)    # 96x96 images planned on a 12x12 grid
    else:
        img = maps
    x, s, g = _t(img), _t(start), _t(goal)
    for m in (na, bb):
        m.train(mode == "train")
    ctx = torch.no_grad() if mode == "eval-no-grad" else torch.enable_grad()
    with ctx:
        o1 = na(x, s, g)
        o2 = bb(x, s, g)
    assert torch.equal(o1.histories, o2.histories)
    assert torch.equal(o1.paths, o2.paths)
    if mode == "train":
        assert o2.histories.requires_grad


def test_graphed_train_step_matches_eager():
    """GraphedTrainStep captures BBAstar's step (the black-box backward included) unchanged: the same losses and
    parameters as eager steps, at g_ratio 0.5 and at 0.3 (both searches batch-coupled on the device).  lambda is large
    here: with the L1 loss's mean over 16 maps, lambda * dL/dhistories is about 1e-3 at the default 20, which may change
    no search of this batch and leave every gradient zero."""
    from neural_astar.planner import BBAstar
    from neural_astar.utils.training import GraphedTrainStep, PlannerModule

    B, H, W = 16, 32, 32
    _, start, goal, maps = _problem(21, B, H, W)
    rng = np.random.RandomState(22)
    opt = (rng.rand(B, 1, H, W) > 0.9).astype(F32)
    batch = [_t(x) for x in (maps, start, goal, opt)]
    for g_ratio in (0.5, 0.3):
        def make():
            torch.manual_seed(1234)
            planner = BBAstar(g_ratio=g_ratio, Tmax=0.25, encoder_depth=4, bbastar_lambda=5000.0)
            return PlannerModule(planner, SimpleNamespace(params=SimpleNamespace(lr=1e-3))).cuda().train()

        eager = make()
        optim = eager.configure_optimizers()
        eager_losses = []
        for step in range(4):
            optim.zero_grad()
            loss = eager.training_step(batch, step)
            loss.backward()
            optim.step()
            eager_losses.append(float(loss))
        graphed = make()
        step_fn = GraphedTrainStep(graphed, batch)
        graph_losses = [float(step_fn(batch)) for _ in range(4)]
        np.testing.assert_allclose(graph_losses, eager_losses, rtol=2e-3)
        pe = float(sum(p.detach().abs().sum() for p in eager.planner.parameters()))
        pg = float(sum(p.detach().abs().sum() for p in graphed.planner.parameters()))
        assert pg == pytest.approx(pe, rel=1e-3)
        assert any(p.grad is not None and p.grad.abs().sum() > 0 for p in eager.planner.parameters())


def test_fit_and_validation_take_bbastar():
    """PlannerModule.fit trains a BBAstar unchanged, and validation uses the single-launch pair."""
    from neural_astar.planner import BBAstar
    from neural_astar.utils.training import PlannerModule

    B, H, W = 8, 32, 32
    _, start, goal, maps = _problem(31, B, H, W)
    opt = (np.random.RandomState(32).rand(B, 1, H, W) > 0.9).astype(F32)
    torch.manual_seed(0)
    module = PlannerModule(BBAstar(Tmax=0.25, bbastar_lambda=5000.0), SimpleNamespace(params=SimpleNamespace(lr=1e-3)))
    batch = [maps, start, goal, opt]
    before = [p.detach().clone().cuda() for p in module.planner.parameters()]
    curve = module.fit([batch, batch], [batch], num_epochs=1)
    assert len(curve) == 2 and all(np.isfinite(curve))
    assert any(not torch.equal(p, q) for p, q in zip(module.planner.parameters(), before))
    if hasattr(module, "logged"):      # without Lightning, _record keeps the last value of every metric
        assert {"metrics/p_opt", "metrics/p_exp", "metrics/h_mean"} <= set(module.logged)


def test_errors_before_any_launch():
    nat = _native()
    from neural_astar.planner import BBAstar

    cost, start, goal, obst = _problem(41, 2, 32, 32)
    c, s, gl, o = (_t(x) for x in (cost, start, goal, obst))
    hist = nat.forward(c, s, gl, o, 0.5, 512)[0]
    g = torch.ones_like(c)
    torch.cuda.synchronize()
    n0 = nat.launch_count()
    for lam in (0.0, -1.0, float("nan"), float("inf"), 1e-46):
        with pytest.raises(ValueError, match="lambda"):
            nat.backward_blackbox(c, s, gl, o, hist, g, lam, 0.5, 512)
    with pytest.raises(RuntimeError, match="CUDA"):
        nat.backward_blackbox(c.cpu(), s.cpu(), gl.cpu(), o.cpu(), hist.cpu(), g.cpu(), 20.0, 0.5, 512)
    with pytest.raises(ValueError):
        nat.backward_blackbox(c, s, gl, o, hist[:1], g, 20.0, 0.5, 512)
    with pytest.raises(ValueError, match="use_differentiable_astar"):
        BBAstar(use_differentiable_astar=False)
    with pytest.raises(ValueError, match="lambda"):
        BBAstar(bbastar_lambda=0.0)
    assert nat.launch_count() == n0
