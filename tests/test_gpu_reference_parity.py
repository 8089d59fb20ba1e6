"""The product's search modules on the GPU against the reference's own DifferentiableAstar, on the matrix of
tests/test_reference_parity_cpu.py (every engine, non-square maps, g_ratio 0 to 1, eval and training loop bounds, single
maps and batch-coupled batches, edge cases).

Per case, `DifferentiableAstar(g_ratio, Tmax, mechanism=...)` runs on CUDA in the case's mode, then
`(out.histories * G).sum().backward()`.  Histories and paths must equal the staged reference run in fp32 bit for bit,
except on a map where the oracles' LITERAL and SPEC forms differ too (the documented exp-collision: two distinct f with
equal fl(exp(-f / sqrt(W)))), where they must equal SPEC.  `cost.grad` must meet the element-wise bound of the CPU file against
the reference's autograd run in float64, on every map whose fp64 run selects what the fp32 one does.  Every case
asserts the engine its shape reaches.  Engine 5 (binary cost maps above 64x64, Moore) is checked forward-only, through
VanillaAstar.
"""
import numpy as np
import pytest
import torch

import test_reference_parity_cpu as rp
from test_reference_parity_cpu import C, CASES, E, R2

pytestmark = pytest.mark.gpu

# engine 5: VanillaAstar on binary maps larger than 64x64 (the cost plane is the obstacle plane)
BIN16_CASES = [
    C("moore", 100, 72, 0.5, E, R2, "binary", 2),
    C("moore", 65, 96, 0.8, E, ("rand", "far"), "binary", 2),
    C("moore", 72, 100, 0.3, E, ("rand",), "binary", 2),
    C("moore", 131, 132, 0.5, E, ("far",), "binary", 3),
    C("moore", 144, 136, 0.8, E, ("rand",), "binary", 3),
]
STATS = {"excluded": [], "worst": {}}


@pytest.fixture(scope="module")
def native():
    from neural_astar import _native

    _native.lib()
    return _native


@pytest.fixture(scope="module")
def reference():
    ref = rp.staged_reference()
    if ref is None:
        pytest.skip("the reference is not staged in oracle/_ref/")
    return ref


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    for key in sorted(STATS["worst"]):
        print(f"\nworst element-wise gradient ratio {key[0]} engine {key[1]}: {STATS['worst'][key]:.3f}")
    print(f"\nmaps excluded from the gradient check: {len(STATS['excluded'])} {STATS['excluded']}")


def _cu(x):
    return torch.from_numpy(np.ascontiguousarray(x)).cuda()


def _forward_matches(hist, paths, r32, p, what):
    """[B] bool: the maps whose device outputs equal the fp32 reference.  Any other map must be one where the oracles'
    SPEC and LITERAL forms differ (an exp-collision), and must equal SPEC, the engines' selection rule."""
    equal = (hist == r32.histories).all((1, 2, 3)) & (paths == r32.paths).all((1, 2, 3))
    if equal.all():
        return equal
    lit = rp.oracle_literal(p)
    spec, _ = rp.oracle_spec(p)
    collided = rp.assert_exp_collisions(p, spec, lit)
    for b in np.flatnonzero(~equal):
        assert b in collided, (what, b, "differs from the reference without an exp-collision")
        np.testing.assert_array_equal(hist[b], spec.histories[b], err_msg=str((what, b)))
        np.testing.assert_array_equal(paths[b], spec.paths[b], err_msg=str((what, b)))
    return equal


@pytest.mark.parametrize("case", CASES, ids=[c.id for c in CASES])
def test_module_matches_reference(native, reference, case):
    from neural_astar.planner.differentiable_astar import DifferentiableAstar

    assert native.lib().nastar_b200_engine_for(case.H, case.W) == case.engine
    p = rp.problem(case)
    astar = DifferentiableAstar(g_ratio=case.g_ratio, Tmax=case.Tmax, mechanism=case.mechanism).cuda()
    astar.train(case.train)
    cost = _cu(p.cost).requires_grad_(True)
    before = native.launch_count()
    out = astar(cost, _cu(p.start), _cu(p.goal), _cu(p.obst))
    (out.histories * _cu(p.G)).sum().backward()
    torch.cuda.synchronize()
    assert native.launch_count() > before
    hist, paths = out.histories.detach().cpu().numpy(), out.paths.cpu().numpy()
    grad = cost.grad.cpu().numpy()

    r32 = rp.run_reference(reference, p, torch.float32)
    equal = _forward_matches(hist, paths, r32, p, case.id)
    if p.cost.shape[1] > 1:
        assert not grad[:, 1:].any(), "the channels the search ignores get no gradient"
    r64 = rp.run_reference(reference, p, torch.float64, p.G)
    same = rp.same_selection(r32, r64) & equal
    for b in range(p.B):
        if not same[b]:
            STATS["excluded"].append(f"{case.id}[{b}]")
            continue
        ratio = rp.assert_grad(grad[b, :1], r64.grad[b, :1], p.G[b], (case.id, b))
        key = (case.mechanism, case.engine)
        STATS["worst"][key] = max(STATS["worst"].get(key, 0.0), ratio)


@pytest.mark.parametrize("case", BIN16_CASES, ids=[c.id for c in BIN16_CASES])
def test_vanilla_bin16_matches_reference(native, reference, case):
    """Forward only: binary maps above 64x64 searched by engine 5 (one launch, then the generic engine's redo pass for
    the maps it flags, so two launches) equal the fp32 reference bit for bit."""
    from neural_astar.planner import VanillaAstar

    L = native.lib()
    assert L.nastar_b200_engine_for(case.H, case.W) == case.engine and L.nastar_b200_bin16_supported(case.H, case.W)
    p = rp.problem(case)
    planner = VanillaAstar(g_ratio=case.g_ratio).cuda().eval()
    before = native.launch_count()
    with torch.no_grad():
        out = planner(_cu(p.obst), _cu(p.start), _cu(p.goal))
    torch.cuda.synchronize()
    assert native.launch_count() - before == 2
    r32 = rp.run_reference(reference, p, torch.float32)
    hist, paths = out.histories.cpu().numpy(), out.paths.cpu().numpy()
    _forward_matches(hist, paths, r32, p, case.id)
