"""Pin both search oracles to the reference's own DifferentiableAstar on generated problems no golden covers.

The staged reference (oracle/_ref/neural_astar/planner/differentiable_astar.py, byte for byte, put there by build())
is run on seeded problems: non-square maps, every engine's shape range, g_ratio 0 to 1, eval and training loop bounds,
single maps and batches (batch-coupled below g_ratio 0.5) and the edge cases listed with `CASES`.  For NEWS it is given
the generator's NorthEastWestSouth filter and heuristic (oracle/_ref/planning_datasets/mechanism.py), as a user of the
reference configures it.  Checked per case:
  forward   the LITERAL oracle (oracle/astar_oracle.c, either mechanism) equals the reference in fp32 bit
            for bit: histories, paths, T_batch and the selected cell of every step;
  spec      SPEC (arg-min of (f, index), what the engines do) differs from LITERAL only by the documented
            exp-collision: two distinct f with equal fl(exp(-f / sqrt(W)));
  backward  the closed-form backward against the autograd gradient of sum(histories * G) of the reference run in
            float64, element by element, and to 1e-5 of the largest magnitude.  The reference's fp32 autograd is not
            used as the yardstick: on 100x72 maps at g_ratio 0.8 it is 4.5e-4 (relative to the largest gradient) away
            from its own fp64 run.

tests/test_gpu_reference_parity.py runs the same matrix through the product's modules on the GPU.
"""
from __future__ import annotations

import importlib
import importlib.util
import os
import sys
import types
import zlib
from typing import NamedTuple, Optional, Tuple

import numpy as np
import pytest
import scipy.ndimage
import torch

from oracle import oracle
from search_steps import machines

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF_PLANNER = os.path.join(ROOT, "oracle", "_ref", "neural_astar", "planner")
REF_MECHANISM = os.path.join(ROOT, "oracle", "_ref", "planning_datasets", "mechanism.py")

# Element-wise bound of a gradient against the fp64 reference: |got - want| <= ATOL * max|G| + RTOL * |want|.
# The worst |got - want| / bound over the whole matrix is 0.52 for oracle.backward
# (test_backward_tolerance_is_tight); the largest |got - want| measured is 5.8e-8 * max|G|.
RTOL = 1e-6
ATOL = 2e-8
REL_TO_MAX = 1e-5      # the existing check: max |got - want| over max |want|
EXP_LIMIT = 80.0       # max f / sqrt(W) of an open cell: beyond it exp(-f / sqrt(W)) nears fp32's underflow


# ------------------------------------------------------------------------------------------------- the reference
def staged_reference():
    """(DifferentiableAstar, NorthEastWestSouth) of the staged reference, its planner imported under a private package
    name so that it does not meet this project's `neural_astar`; None where oracle/_ref/ is not staged."""
    if not (os.path.isfile(os.path.join(REF_PLANNER, "differentiable_astar.py")) and os.path.isfile(REF_MECHANISM)):
        return None
    if "_ref_planner" not in sys.modules:
        pkg = types.ModuleType("_ref_planner")
        pkg.__path__ = [REF_PLANNER]
        sys.modules["_ref_planner"] = pkg
    da = importlib.import_module("_ref_planner.differentiable_astar")
    mech = sys.modules.get("_ref_planner_mechanism")
    if mech is None:
        spec = importlib.util.spec_from_file_location("_ref_planner_mechanism", REF_MECHANISM)
        mech = importlib.util.module_from_spec(spec)
        spec.loader.exec_module(mech)
        sys.modules["_ref_planner_mechanism"] = mech
    return da.DifferentiableAstar, mech.NorthEastWestSouth


@pytest.fixture(scope="module")
def reference():
    ref = staged_reference()
    if ref is None:
        pytest.skip("the reference is not staged in oracle/_ref/")
    return ref


class RefRun(NamedTuple):
    histories: np.ndarray        # [B,1,H,W] in the run's dtype
    paths: np.ndarray            # [B,1,H,W] int64
    T_batch: int                 # iterations of the reference's loop
    trace: np.ndarray            # [B,T_batch] selected cell of every step
    grad: Optional[np.ndarray]   # d sum(histories * G) / d cost, the cost's shape, or None


def run_reference(reference, p, dtype, G=None) -> RefRun:
    """The reference's DifferentiableAstar on CPU planes in `dtype` (module and inputs alike), with the autograd gradient
    of sum(histories * G) when G is given."""
    DifferentiableAstar, NEWS = reference
    astar = DifferentiableAstar(g_ratio=p.g_ratio, Tmax=p.Tmax)
    if p.mechanism == "news":
        astar.neighbor_filter.data = NEWS.get_neighbor_filter()
        astar.get_heuristic = NEWS.get_heuristic
    astar = astar.to(dtype).train(p.train)
    cost = torch.from_numpy(p.cost).to(dtype).requires_grad_(G is not None)
    start, goal, obst = (torch.from_numpy(x).to(dtype) for x in (p.start, p.goal, p.obst))
    with torch.set_grad_enabled(G is not None):
        out = astar(cost, start, goal, obst, store_intermediate_results=True)
        frames = out.intermediate_results[:-1]
        trace = torch.stack([fr["paths"].reshape(p.B, -1).argmax(1) for fr in frames], 1).numpy()
        grad = None
        if G is not None:
            (out.histories * torch.from_numpy(G).to(dtype)).sum().backward()
            grad = cost.grad.numpy()
    return RefRun(out.histories.detach().numpy(), out.paths.numpy(), len(frames), trace, grad)


# ------------------------------------------------------------------------------------------------- the problems
class Case(NamedTuple):
    mechanism: str     # "moore" or "news"
    H: int
    W: int
    g_ratio: float
    train: bool        # training mode: loop bound int(Tmax * W * W); eval: W * W
    Tmax: float
    kinds: Tuple[str, ...]   # one start/goal layout per map (see `problem`)
    costs: str         # cost kind (see `problem`)
    engine: int        # nastar_b200_engine_for(H, W)

    @property
    def B(self):
        return len(self.kinds)

    @property
    def id(self):
        mode = f"train{self.Tmax}" if self.train else "eval"
        return (f"{self.mechanism}-{self.H}x{self.W}-e{self.engine}-g{self.g_ratio}-{mode}-B{self.B}-"
                f"{'+'.join(sorted(set(self.kinds)))}-{self.costs}")


def C(mechanism, H, W, g_ratio, mode, kinds, costs, engine):
    train = mode != "eval"
    return Case(mechanism, H, W, g_ratio, train, float(mode) if train else 1.0, tuple(kinds), costs, engine)


E, T25, T05 = "eval", "0.25", "0.05"
R2, R3 = ("rand",) * 2, ("rand",) * 3
# Every Moore shape of engines 1 (up to 32x32), 4 (up to 64x64), 2 (generic, state in shared memory) and 3 (generic,
# HBM workspace) meets several g_ratios, both loop bounds and B = 1 and B > 1; below 0.5 a batch is coupled.  Engines
# 2 and 3 run training-mode bounds of Tmax 0.05: the reference keeps about ten [B,H,W] planes per step for autograd.
# NEWS maps are square: the generator's heuristic reads size = shape[-1].
CASES = [
    # engine 1
    C("moore", 32, 32, 0.5, E, R3, "learned", 1),
    C("moore", 32, 32, 0.3, E, R3, "quarter", 1),
    C("moore", 32, 32, 1.0, T25, R2, "learned", 1),
    C("moore", 12, 20, 0.8, E, ("rand", "adjacent"), "x10", 1),
    C("moore", 12, 20, 0.0, E, R3, "learned", 1),
    C("moore", 20, 12, 0.5, T05, ("far", "far"), "learned", 1),          # capped by T = 7 before the goal, H > W
    C("moore", 20, 12, 0.3, E, ("rand",), "x10", 1),
    C("moore", 7, 5, 0.5, E, ("same", "adjacent", "rand", "far"), "quarter", 1),
    C("moore", 7, 5, 0.8, T25, ("rand", "far"), "learned", 1),
    C("moore", 7, 5, 0.3, E, ("corridor", "same", "rand"), "learned", 1),
    C("moore", 31, 29, 0.8, T25, R2, "two_channel", 1),
    C("moore", 31, 29, 0.0, E, ("rand",), "zero", 1),
    C("moore", 31, 29, 1.0, E, ("corridor",), "learned", 1),
    # engine 4
    C("moore", 33, 33, 0.5, E, R2, "learned", 4),
    C("moore", 33, 33, 0.3, T25, R3, "learned", 4),
    C("moore", 48, 40, 0.8, E, ("rand",), "learned", 4),
    C("moore", 48, 40, 0.5, "0.02", ("far", "rand"), "quarter", 4),       # capped by T = 32, H > W
    C("moore", 40, 48, 0.0, E, R3, "learned", 4),
    C("moore", 40, 48, 1.0, T25, ("rand",), "zero", 4),
    C("moore", 64, 64, 0.5, T25, R2, "two_channel", 4),
    C("moore", 64, 64, 0.3, E, R2, "learned", 4),
    C("moore", 64, 64, 0.8, E, ("corridor",), "learned", 4),
    C("moore", 64, 2, 0.5, E, ("far", "rand", "adjacent"), "learned", 4),  # capped by T = 4, H > W
    C("moore", 64, 2, 0.8, T25, R2, "learned", 4),                         # a one-step loop: the gradient is 0
    # engine 2
    C("moore", 100, 72, 0.8, T05, R2, "learned", 2),
    C("moore", 100, 72, 0.3, T05, R2, "learned", 2),
    C("moore", 72, 100, 0.5, T05, R2, "quarter", 2),
    C("moore", 72, 100, 1.0, T05, ("rand",), "learned", 2),
    C("moore", 65, 96, 0.0, E, R2, "learned", 2),
    C("moore", 65, 96, 0.5, T05, ("far",), "learned", 2),
    # engine 3
    C("moore", 131, 132, 0.5, T05, ("rand",), "learned", 3),
    C("moore", 131, 132, 0.0, E, R2, "learned", 3),
    C("moore", 144, 136, 0.3, T05, R2, "learned", 3),
    C("moore", 144, 136, 0.8, "0.02", ("far",), "learned", 3),            # capped by T = 369, H > W
    C("moore", 131, 132, 0.5, E, ("far",), "binary", 3),                  # an exp-collision: SPEC closes one cell more
    # NEWS
    C("news", 32, 32, 0.5, E, R2, "learned", 1),
    C("news", 32, 32, 0.3, E, R3, "quarter", 1),
    C("news", 32, 32, 0.8, T25, ("same", "adjacent", "corridor"), "learned", 1),
    C("news", 48, 48, 0.8, T25, R2, "learned", 4),
    C("news", 48, 48, 0.0, E, R2, "x10", 4),
    C("news", 64, 64, 1.0, T25, ("rand",), "learned", 4),
    C("news", 64, 64, 0.3, E, R2, "learned", 4),
    C("news", 100, 100, 0.5, T05, R2, "learned", 2),
    C("news", 144, 144, 0.3, T05, R2, "learned", 3),
]


class Problem(NamedTuple):
    mechanism: str
    g_ratio: float
    Tmax: float
    train: bool
    cost: np.ndarray    # [B,C,H,W] float32 (C = 2 for "two_channel")
    start: np.ndarray   # [B,1,H,W] float32
    goal: np.ndarray
    obst: np.ndarray
    G: np.ndarray       # [B,1,H,W] float32 upstream gradient of histories

    @property
    def B(self):
        return self.start.shape[0]

    @property
    def T(self):
        return int((self.Tmax if self.train else 1.0) * self.start.shape[-1] ** 2)


def _connectivity(mechanism):
    return np.ones((3, 3), int) if mechanism == "moore" else scipy.ndimage.generate_binary_structure(2, 1)


def _distance(mechanism, a, b):
    dy, dx = abs(a[0] - b[0]), abs(a[1] - b[1])
    return max(dy, dx) if mechanism == "moore" else dy + dx


def _layout(rng, kind, mechanism, H, W):
    """(obstacles [H,W], start (y, x), goal (y, x)) of one map, the goal reachable from the start:
      rand      20 % obstacles, start and goal drawn from one connected region, a third of the map apart if it can;
      far       the same, the goal the region's cell farthest from the start;
      adjacent  the goal a passable neighbour of the start;
      same      start == goal;
      corridor  a one-cell L-shaped corridor from the top-left to the bottom-right corner, walls everywhere else."""
    if kind == "corridor":
        obst = np.zeros((H, W), np.float32)
        obst[:, 0] = 1
        obst[H - 1, :] = 1
        return obst, (0, 0), (H - 1, W - 1)
    structure = _connectivity(mechanism)
    while True:
        obst = (rng.rand(H, W) > 0.2).astype(np.float32)
        labels, _ = scipy.ndimage.label(obst, structure=structure)
        sy, sx = rng.randint(H), rng.randint(W)
        if not obst[sy, sx]:
            continue
        region = np.argwhere(labels == labels[sy, sx])
        if kind == "same":
            return obst, (sy, sx), (sy, sx)
        if kind == "adjacent":
            region = [c for c in region if 0 < _distance(mechanism, c, (sy, sx)) <= 1 and (
                mechanism == "moore" or c[0] == sy or c[1] == sx)]
        else:
            region = [c for c in region if tuple(c) != (sy, sx)]
        if not region:
            continue
        if kind == "far":
            gy, gx = max(region, key=lambda c: (_distance(mechanism, c, (sy, sx)), c[0], c[1]))
        else:
            # a third of the map away where the region allows it: long enough searches to sum many softmax steps
            away = [c for c in region if _distance(mechanism, c, (sy, sx)) >= max(H, W) // 3]
            region = away or region
            gy, gx = region[rng.randint(len(region))]
        return obst, (sy, sx), (int(gy), int(gx))


def _costs(rng, kind, B, H, W):
    """learned: sigmoid(N(0, 1)), like the encoder's output; quarter: multiples of 0.25 in [0, 1], so that equal f values
    are broken by index; zero; x10: ten times learned; two_channel: learned plus a second channel the search ignores;
    binary: None, the cost is the obstacle plane."""
    learned = (1.0 / (1.0 + np.exp(-rng.randn(B, 1, H, W)))).astype(np.float32)
    if kind == "learned":
        return learned
    if kind == "quarter":
        return (rng.randint(0, 5, (B, 1, H, W)) * 0.25).astype(np.float32)
    if kind == "zero":
        return np.zeros((B, 1, H, W), np.float32)
    if kind == "x10":
        return learned * np.float32(10)
    if kind == "two_channel":
        return np.concatenate([learned, rng.rand(B, 1, H, W).astype(np.float32)], 1)
    if kind == "binary":
        return None    # the obstacle planes themselves, as VanillaAstar searches
    raise ValueError(kind)


def problem(case: Case) -> Problem:
    """The seeded problem of a case; asserts that exp(-f / sqrt(W)) stays far from underflow on every open cell."""
    rng = np.random.RandomState(zlib.crc32(case.id.encode()))
    B, H, W = case.B, case.H, case.W
    obst = np.zeros((B, 1, H, W), np.float32)
    start, goal = np.zeros_like(obst), np.zeros_like(obst)
    for b, kind in enumerate(case.kinds):
        o, s, g = _layout(rng, kind, case.mechanism, H, W)
        obst[b, 0], start[b, 0][s], goal[b, 0][g] = o, 1, 1
    cost = _costs(rng, case.costs, B, H, W)
    p = Problem(case.mechanism, case.g_ratio, case.Tmax, case.train, obst.copy() if cost is None else cost, start, goal,
                obst, rng.randn(B, 1, H, W).astype(np.float32))
    worst = max_f_over_sqrt_w(p)
    assert worst < EXP_LIMIT, f"{case.id}: max f / sqrt(W) = {worst:.1f}: exp(-f / sqrt(W)) would underflow"
    return p


def max_f_over_sqrt_w(p: Problem) -> float:
    """max over steps and open cells of f / sqrt(W), replaying SPEC for the loop bound with no early exit (so that the
    post-solve steps of a batch-coupled loop are covered too)."""
    gr, omg, sqw = oracle.scalars(p.g_ratio, p.start.shape[-1])
    worst = 0.0
    for m in machines(p.cost, p.start, p.goal, p.obst, p.mechanism):
        for _ in range(p.T):
            ind = m.select(gr, omg)
            if ind < 0:
                break
            worst = max(worst, float(m.f(gr, omg)[m.open].max()))
            m.close_and_expand(ind)
    return worst / float(sqw)


# ------------------------------------------------------------------------------------------------- the oracles
def oracle_literal(p: Problem, want_trace=True):
    return oracle.forward(p.cost[:, :1], p.start, p.goal, p.obst, g_ratio=p.g_ratio, Tmax=p.Tmax, training=p.train,
                          mode="literal", want_trace=want_trace, mechanism=p.mechanism)


def oracle_spec(p: Problem):
    """SPEC: each map's own search, or below g_ratio 0.5 with B > 1 the batch-coupled one (every map stepped with no
    early exit, stopped after the first step at which all maps select their goal).  Returns (output, T_batch)."""
    args = (p.cost[:, :1], p.start, p.goal, p.obst)
    kw = dict(g_ratio=p.g_ratio, mode="spec", want_trace=True, mechanism=p.mechanism)
    if p.g_ratio < 0.5 and p.B > 1:
        full = oracle.forward(*args, **kw, T=p.T, no_early_exit=True)
        goal_idx = p.goal.reshape(p.B, -1).argmax(1)
        at_goal = (full.trace == goal_idx[:, None]).all(0)
        T_batch = int(np.argmax(at_goal)) + 1 if at_goal.any() else p.T
        out = oracle.forward(*args, **kw, T=T_batch, no_early_exit=True)
        return out, T_batch
    out = oracle.forward(*args, **kw, Tmax=p.Tmax, training=p.train)
    return out, int(out.T_batch)


def oracle_backward(p: Problem, T_batch: int) -> np.ndarray:
    return oracle.backward(p.cost[:, :1], p.start, p.goal, p.obst, p.G, T_batch, g_ratio=p.g_ratio,
                           mechanism=p.mechanism)


def assert_exp_collisions(p: Problem, spec, lit):
    """Where the SPEC and LITERAL traces of a map differ, they differ by the documented exp-collision: at the first
    differing step both open cells have distinct f, equal fl(exp(-f / sqrt(W))), and LITERAL's first maximum takes the
    lower index where SPEC takes the smaller f.  The searches then go on from different states: adjacent selections
    swapped, or one cell more or less in histories (test_oracle_golden.py has both on the reference's own vectors).
    Returns the maps that differ."""
    gr, omg, sqw = oracle.scalars(p.g_ratio, p.start.shape[-1])
    maps = machines(p.cost, p.start, p.goal, p.obst, p.mechanism)
    differ = []
    for b in range(p.B):
        n = min(int(spec.n_steps[b]), int(lit.T_batch))
        diff = np.nonzero(spec.trace[b, :n] != lit.trace[b, :n])[0]
        if not len(diff) and np.array_equal(spec.histories[b], lit.histories[b]):
            continue
        differ.append(b)
        k = int(diff[0]) if len(diff) else n
        m = maps[b]
        for t in range(k):
            m.close_and_expand(int(lit.trace[b, t]))
        a, z = int(spec.trace[b, k]), int(lit.trace[b, k])
        f = m.f(gr, omg)
        e = torch.exp(torch.from_numpy((np.float32(-1) * f[[a, z]]) / sqw)).numpy()
        assert m.open[a] and m.open[z] and f[a] < f[z] and e[0] == e[1] and z < a, (b, k, f[a], f[z])
    return differ


def same_selection(r32: RefRun, r64: RefRun):
    """[B] bool: the fp64 reference selected what the fp32 one did, step for step.  Equal histories and paths are not
    enough: a capped search can close the same cells in another order, and the gradient sums every step's softmax."""
    if r32.T_batch != r64.T_batch:
        return np.zeros(r32.trace.shape[0], bool)
    same = (r32.histories == r64.histories).all((1, 2, 3)) & (r32.paths == r64.paths).all((1, 2, 3))
    return same & (r32.trace == r64.trace).all(1)


def grad_ratio(got, want, G):
    """Worst |got - want| / (ATOL * max|G| + RTOL * |want|) of one map: the element-wise bound holds iff <= 1."""
    bound = ATOL * float(np.abs(G).max()) + RTOL * np.abs(want)
    return float((np.abs(got.astype(np.float64) - want) / bound).max())


def assert_grad(got, want, G, what):
    """`got` against the fp64 reference gradient `want` of one map: element by element, and to 1e-5 of the largest
    magnitude.  Where the exact gradient is 0 (g_ratio 1, a one-step loop) or no larger than fp64 rounding of it (a map
    solved at its first step that keeps re-selecting its goal), below 1e-12 * max|G|."""
    assert np.isfinite(got).all(), what
    if float(np.abs(want).max()) <= 1e-12 * float(np.abs(G).max()):
        assert float(np.abs(got).max()) <= 1e-12 * float(np.abs(G).max()), what
        return 0.0
    ratio = grad_ratio(got, want, G)
    assert ratio <= 1.0, (what, ratio)
    assert float(np.abs(got - want).max()) <= REL_TO_MAX * float(np.abs(want).max()), what
    return ratio


# ------------------------------------------------------------------------------------------------- the tests
WORST = {}           # (mechanism, engine) -> worst element-wise ratio of the oracles' gradients
EXCLUDED = []        # ids of maps whose fp64 reference selected differently from the fp32 one
RAN = set()          # ids of the cases whose gradients were compared


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    for key in sorted(WORST):
        print(f"\nworst element-wise gradient ratio {key[0]} engine {key[1]}: {WORST[key]:.3f}")
    print(f"\nmaps excluded from the gradient check (fp32 and fp64 reference selections differ, or an exp-collision): "
          f"{len(EXCLUDED)} "
          f"{EXCLUDED}")


def test_matrix_reaches_every_engine():
    """Each case's shape selects the engine it names (tests/test_abi_cpu.py pins the full table)."""
    from neural_astar import _native

    lib = _native.lib()
    for case in CASES:
        assert lib.nastar_b200_engine_for(case.H, case.W) == case.engine, case.id
        assert min(case.H, case.W) > 1, "the reference's expand().squeeze() collapses 1-wide maps"
    for mech in ("moore", "news"):
        assert {c.engine for c in CASES if c.mechanism == mech} == {1, 2, 3, 4}
    assert all(c.H == c.W for c in CASES if c.mechanism == "news")


@pytest.mark.parametrize("case", CASES, ids=[c.id for c in CASES])
def test_oracles_match_reference(reference, case):
    p = problem(case)
    r32 = run_reference(reference, p, torch.float32)
    # forward: LITERAL is the reference's loop, bit for bit
    lit = oracle_literal(p)
    assert lit.T_batch == r32.T_batch
    np.testing.assert_array_equal(lit.histories, r32.histories)
    np.testing.assert_array_equal(lit.paths, r32.paths)
    np.testing.assert_array_equal(lit.trace[:, :r32.T_batch], r32.trace)
    # SPEC: the same maps up to the exp-collision
    spec, T_batch = oracle_spec(p)
    collided = assert_exp_collisions(p, spec, lit)
    if not collided:
        assert T_batch == r32.T_batch
        np.testing.assert_array_equal(spec.histories, lit.histories)
        np.testing.assert_array_equal(spec.paths, lit.paths)
    # backward: the closed form against the fp64 reference's autograd
    r64 = run_reference(reference, p, torch.float64, p.G)
    if p.cost.shape[1] > 1:
        assert not r64.grad[:, 1:].any()
    got = oracle_backward(p, r32.T_batch)
    same = same_selection(r32, r64)
    for b in range(p.B):
        if not same[b] or b in collided:    # the closed form replays SPEC
            EXCLUDED.append(f"{case.id}[{b}]")
            continue
        ratio = assert_grad(got[b], r64.grad[b, :1], p.G[b], (case.id, b))
        key = (case.mechanism, case.engine)
        WORST[key] = max(WORST.get(key, 0.0), ratio)
    RAN.add(case.id)


def test_backward_tolerance_is_tight():
    """The element-wise bound is at most 4x looser than the worst case of the whole matrix: 0.52 of it (NEWS, 64x64,
    g_ratio 0.3), with no engine's worst below 0.1."""
    if len(RAN) < len(CASES):
        pytest.skip("needs the whole matrix")
    assert max(WORST.values()) >= 0.25, WORST
