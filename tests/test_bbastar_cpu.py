"""CPU checks of the black-box backward (BB-A*): the C ABI's and the binding's argument checks (nothing launches), the
oracle's gradient against a direct restatement, and BBAstar's state dict against NeuralAstar's."""
import ctypes
import math
import os
import subprocess

import numpy as np
import pytest
import torch

import bbastar_oracle

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EINVAL, EUNSUPPORTED, EWORKSPACE = 1, 2, 4
F32 = np.float32


@pytest.fixture(scope="module")
def native():
    subprocess.check_call(["make", "-C", os.path.join(ROOT, "neural-astar_b200"), "-s", "all"])
    from neural_astar import _native

    return _native


@pytest.fixture
def no_launch(native):
    L = native.lib()
    before = L.nastar_b200_launch_count()
    yield L
    assert L.nastar_b200_launch_count() == before, "a rejected call launched something"


# fake device addresses, never dereferenced: every case below returns before any launch
HIST, GRAD, OUT, TB, CLAMP, WS = 0x50000, 0x60000, 0x70000, 0x80000, 0x90000, 0xA0000


def _fwd(native, **kw):
    p = native.FwdParams()
    p.cost, p.start, p.goal, p.obst = 0x10000, 0x20000, 0x30000, 0x40000
    p.cost_stride = p.start_stride = p.goal_stride = p.obst_stride = 32 * 32
    p.B, p.H, p.W, p.T = 4, 32, 32, 100
    p.g_ratio, p.one_minus_g_ratio = 0.5, 0.5
    for k, v in kw.items():
        setattr(p, k, v)
    return ctypes.byref(p)


def _call(L, p, hist=HIST, grad=GRAD, lam=20.0, out=OUT, T_batch=None, clamp=None):
    return L.nastar_b200_backward_blackbox(p, hist, grad, 32 * 32, lam, out, T_batch, clamp, None)


def test_export(native):
    # an added entry point: the structs and the existing entry points are unchanged, so the ABI version stays
    assert "nastar_b200_backward_blackbox" in native.EXPORTS
    with open(os.path.join(ROOT, "include", "nastar_b200.h")) as f:
        header = f.read()
    assert "int nastar_b200_backward_blackbox(" in header
    assert hasattr(native.lib(), "nastar_b200_backward_blackbox")


@pytest.mark.parametrize("lam", [0.0, -1.0, -0.0, math.inf, -math.inf, math.nan])
def test_abi_rejects_lambda(native, no_launch, lam):
    assert _call(no_launch, _fwd(native), lam=lam) == EINVAL


@pytest.mark.parametrize("field", ["cost", "start", "goal", "obst"])
def test_abi_rejects_null_plane(native, no_launch, field):
    assert _call(no_launch, _fwd(native, **{field: None})) == EINVAL


@pytest.mark.parametrize("kw", [dict(hist=None), dict(grad=None), dict(out=None), dict(T_batch=TB),
                                dict(clamp=CLAMP)])
def test_abi_rejects_null_outputs_and_half_coupled(native, no_launch, kw):
    assert _call(no_launch, _fwd(native), **kw) == EINVAL


@pytest.mark.parametrize("kw,status", [
    (dict(B=0), EINVAL),
    (dict(T=0), EINVAL),
    (dict(cost_kind=1), EINVAL),                 # NASTAR_COST_LOGIT: the perturbation needs a cost plane
    (dict(cost_kind=2), EINVAL),                 # NASTAR_COST_TAPS
    (dict(flags=1), EINVAL),                     # NASTAR_FWD_NO_EARLY_EXIT
    (dict(flags=2), EINVAL),                     # NASTAR_FWD_PAIR
    (dict(flags=4 | 1), EINVAL),
    (dict(trace=0xB0000), EINVAL),
    (dict(H=600, W=2048), EUNSUPPORTED),
    (dict(B=4, H=300, W=300), EWORKSPACE),       # engine 3 without its slots
])
def test_abi_rejects_params(native, no_launch, kw, status):
    assert _call(no_launch, _fwd(native, **kw)) == status


def test_abi_coupled_needs_the_coupled_workspace(native, no_launch):
    need = no_launch.nastar_b200_forward_coupled_workspace_bytes(4, 32, 32, 100)
    assert need > 0
    assert _call(no_launch, _fwd(native), T_batch=TB, clamp=CLAMP) == EWORKSPACE
    assert _call(no_launch, _fwd(native, workspace=WS, workspace_bytes=need - 1), T_batch=TB, clamp=CLAMP) == EWORKSPACE


@pytest.mark.parametrize("lam", [0.0, -2.0, math.inf, math.nan, 1e-50, 1e39])
def test_binding_rejects_lambda_before_anything(native, no_launch, lam):
    x = torch.zeros(2, 1, 8, 8)
    with pytest.raises(ValueError, match="lambda"):
        native.backward_blackbox(x, x, x, x, x, x, lam, 0.5, 64)


def test_binding_rejects_cpu_tensors(native, no_launch):
    x = torch.zeros(2, 1, 8, 8)
    with pytest.raises(RuntimeError, match="CUDA"):
        native.backward_blackbox(x, x, x, x, x, x, 20.0, 0.5, 64)


def test_binding_rejects_bad_mechanism_and_steps(native, no_launch):
    x = torch.zeros(2, 1, 8, 8)
    with pytest.raises(ValueError, match="mechanism"):
        native.backward_blackbox(x, x, x, x, x, x, 20.0, 0.5, 64, mechanism="hex")
    with pytest.raises(ValueError, match="2\\*\\*31"):
        native.backward_blackbox(x, x, x, x, x, x, 20.0, 0.5, 2**31)


# ---- the oracle -------------------------------------------------------------------------------------------------

def _problem(rng, B, H, W, lo=0.1):
    maps = (rng.rand(B, 1, H, W) > 0.25).astype(F32)
    start = np.zeros_like(maps)
    goal = np.zeros_like(maps)
    for b in range(B):
        cells = np.flatnonzero(maps[b, 0])
        s, g = rng.choice(cells, 2, replace=False)
        start[b, 0].flat[s] = 1
        goal[b, 0].flat[g] = 1
    cost = (lo + rng.rand(B, 1, H, W)).astype(F32)
    return cost, start, goal, maps


def _restated(cost, start, goal, obst, grad, lam, g_ratio, T, mechanism, coupled):
    """The same gradient restated: w' rounded once per operation from exact float64 arithmetic, y from the search."""
    w = cost[:, :1].astype(np.float64)
    prod = (np.float64(np.float32(lam)) * grad.astype(np.float64)).astype(F32)           # fl(lambda * g)
    w2 = (w + prod.astype(np.float64)).astype(F32)                                       # fl(w + .)
    y = bbastar_oracle.search(cost, start, goal, obst, g_ratio, T, mechanism, coupled)
    y2 = bbastar_oracle.search(w2, start, goal, obst, g_ratio, T, mechanism, coupled)
    inv = F32(1.0 / np.float64(np.float32(lam)))                                         # fl(1/lambda)
    return np.where(y2 > y, inv, np.where(y2 < y, -inv, F32(0))).astype(F32), w2


@pytest.mark.parametrize("mechanism", ["moore", "news"])
@pytest.mark.parametrize("g_ratio,B,coupled", [(0.5, 3, False), (0.7, 2, False), (0.2, 1, False), (0.2, 3, True)])
@pytest.mark.parametrize("lam", [20.0, 3.7])
def test_oracle_matches_restatement(mechanism, g_ratio, B, coupled, lam):
    rng = np.random.RandomState(7)
    H, W = 9, 11
    cost, start, goal, obst = _problem(rng, B, H, W)
    T = int(0.5 * W * W)
    y = bbastar_oracle.search(cost, start, goal, obst, g_ratio, T, mechanism, coupled)
    # an L1-like upstream gradient, large enough to move the search, and negative in places so that some w' < 0
    grad = (np.sign(rng.rand(B, 1, H, W) - 0.5) * rng.choice([0.0, 0.5, 1.5], (B, 1, H, W)) / lam).astype(F32)
    grad[:, :, 0, :] = F32(-4.0 / lam)
    out = bbastar_oracle.blackbox_backward(cost, start, goal, obst, grad, lam, g_ratio, T, mechanism, coupled)
    want, w2 = _restated(cost, start, goal, obst, grad, lam, g_ratio, T, mechanism, coupled)
    assert np.array_equal(out.costs, w2)
    assert (out.costs < 0).any(), "the case is meant to search some negative costs"
    assert np.array_equal(out.histories, y)
    assert np.array_equal(out.grad, want)
    assert out.grad.dtype == np.float32
    assert set(np.unique(np.abs(out.grad))) <= {F32(0), F32(1) / F32(lam)}
    assert np.abs(out.grad).sum() > 0, "the perturbation is meant to change the search"


def test_oracle_w_prime_rounds_each_operation():
    # fl(w + fl(lambda * g)), each operation rounded to float32: on random data some cells differ from the singly
    # rounded fl(w + lambda * g) that an FMA would give, so the check below tells the two apart
    rng = np.random.RandomState(5)
    w = rng.randn(4, 1, 32, 32).astype(F32)
    g = rng.randn(4, 1, 32, 32).astype(F32)
    lam = 3.7
    l32 = np.float64(F32(lam))
    two = bbastar_oracle.perturbed_costs(w, g, lam)
    prod = (l32 * g.astype(np.float64)).astype(F32)
    assert np.array_equal(two, (w.astype(np.float64) + prod.astype(np.float64)).astype(F32))
    fused = (w.astype(np.float64) + l32 * g.astype(np.float64)).astype(F32)   # exact product: fits in float64
    assert (fused != two).any()


def test_oracle_zero_gradient_gives_zero():
    rng = np.random.RandomState(3)
    cost, start, goal, obst = _problem(rng, 2, 8, 8)
    out = bbastar_oracle.blackbox_backward(cost, start, goal, obst, np.zeros_like(cost), 20.0, 0.5, 64)
    assert np.array_equal(out.grad, np.zeros_like(cost)) and not np.signbit(out.grad).any()


# ---- BBAstar's module surface ------------------------------------------------------------------------------------

@pytest.mark.parametrize("kw", [dict(), dict(encoder_arch="CNNDownSize", encoder_input="rgb+", encoder_depth=3),
                                dict(encoder_arch="Unet", encoder_depth=2, const=5.0, learn_obstacles=True)])
def test_state_dict_interchange(native, kw):
    from neural_astar.planner import BBAstar, NeuralAstar

    torch.manual_seed(0)
    bb = BBAstar(Tmax=0.25, bbastar_lambda=7.5, **kw)
    torch.manual_seed(1)
    na = NeuralAstar(Tmax=0.25, **kw)
    sd_bb, sd_na = bb.state_dict(), na.state_dict()
    assert list(sd_bb) == list(sd_na)
    assert all(sd_bb[k].shape == sd_na[k].shape and sd_bb[k].dtype == sd_na[k].dtype for k in sd_bb)
    na.load_state_dict(sd_bb)                 # a checkpoint trained as BB-A* loads into NeuralAstar ...
    assert all(torch.equal(v, sd_bb[k]) for k, v in na.state_dict().items())
    torch.manual_seed(2)
    bb2 = BBAstar(Tmax=0.25, **kw)
    bb2.load_state_dict(sd_na)                # ... and the reverse
    assert all(torch.equal(v, sd_na[k]) for k, v in bb2.state_dict().items())
    assert bb.bbastar_lambda == 7.5 and bb2.bbastar_lambda == 20.0   # lambda is not part of the state


def test_constructor_checks(native):
    from neural_astar.planner import BBAstar, NeuralAstar
    from neural_astar.planner.differentiable_astar import BlackboxAstar, DifferentiableAstar

    with pytest.raises(ValueError, match="use_differentiable_astar"):
        BBAstar(use_differentiable_astar=False)
    for lam in (0.0, -1.0, math.nan, math.inf):
        with pytest.raises(ValueError, match="lambda"):
            BBAstar(bbastar_lambda=lam)
    p = BBAstar(g_ratio=0.3, Tmax=0.5, mechanism="news")
    assert isinstance(p, NeuralAstar) and isinstance(p.astar, BlackboxAstar)
    assert p.astar.mechanism == "news" and p.astar.g_ratio == 0.3 and p.astar.Tmax == 0.5
    assert torch.equal(p.astar.neighbor_filter, NeuralAstar(mechanism="news").astar.neighbor_filter)
    assert type(NeuralAstar().astar) is DifferentiableAstar
    # positional arguments are NeuralAstar's, lambda comes last
    q = BBAstar(0.5, 0.25, "m", "CNN", 2, False, None, True, 4.0)
    assert q.encoder_input == "m" and q.bbastar_lambda == 4.0
