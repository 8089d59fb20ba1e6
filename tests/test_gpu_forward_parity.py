"""GPU parity: the CUDA engine (called through the C ABI of libnastar_b200.so) vs

  (1) the golden vectors produced by the reference itself (tests/golden/*.npz), bit-exact masks;
  (2) the CPU oracle (oracle/astar_oracle.c, SPEC form) on seeded random inputs, bit-exact
      histories / paths / solve step / step count / selection trace.
"""
import numpy as np
import pytest
import torch

from golden_util import Golden, all_names

pytestmark = pytest.mark.gpu

NAMES = all_names()


@pytest.fixture(scope="module")
def native():
    from neural_astar import _native

    _native.lib()  # fail loudly if the extension is not built
    return _native


def _dev(x):
    return torch.from_numpy(np.ascontiguousarray(x)).cuda()


def _run_native(native, cost, start, goal, obst, g_ratio=0.5, T=None, trace=False, alias=False):
    c = _dev(cost)
    o = c if alias else _dev(obst)
    W = cost.shape[-1]
    T = T if T is not None else W * W
    hist, paths, ts, ns, tr = native.forward(c, _dev(start), _dev(goal), o, g_ratio, T, trace)
    torch.cuda.synchronize()
    return (hist.cpu().numpy(), paths.cpu().numpy(), ts.cpu().numpy(), ns.cpu().numpy(),
            tr.cpu().numpy() if tr is not None else None)


@pytest.mark.parametrize("name", [n for n in NAMES if not Golden(n).meta.get("lowg")])
def test_golden_masks_bit_exact(native, name):
    g = Golden(name)
    vanilla = bool(g.meta.get("vanilla"))
    hist, paths, ts, ns, _ = _run_native(native, g.cost, g.start, g.goal, g.obst, g.g_ratio, alias=vanilla)
    assert hist.dtype == np.float32 and paths.dtype == np.int64
    assert hist.shape == (g.B, 1, g.H, g.W) and paths.shape == (g.B, 1, g.H, g.W)
    np.testing.assert_array_equal(hist != 0, g.bits("hist_bits") != 0)
    np.testing.assert_array_equal(paths != 0, g.bits("path_bits") != 0)
    assert set(np.unique(hist)) <= {0.0, 1.0} and set(np.unique(paths)) <= {0, 1}
    # per-map solve step + 1 == number of closed nodes (each step closes exactly one new node)
    np.testing.assert_array_equal(ts + 1, g.z["hist_sum"])
    np.testing.assert_array_equal(ns, g.z["hist_sum"])


def test_adversarial_near_tie_engine_equals_spec(native, oracle):
    """The one documented deviation from the reference (DESIGN.md "Selection semantics"): on the adversarial near-tie
    vectors the engine — like the SPEC oracle — closes one cell fewer than the reference; everything else agrees."""
    g = Golden("adversarial_neartie")
    hist, paths, ts, ns, _ = _run_native(native, g.cost, g.start, g.goal, g.obst, g.g_ratio)
    spec = oracle.forward(g.cost, g.start, g.goal, g.obst, mode="spec")
    np.testing.assert_array_equal(hist, spec.histories)
    np.testing.assert_array_equal(paths, spec.paths)
    np.testing.assert_array_equal(ns, spec.n_steps)
    np.testing.assert_array_equal(paths != 0, g.bits("path_bits") != 0)
    diff = (hist != 0) != (g.bits("hist_bits") != 0)
    assert diff.reshape(g.B, -1).sum(1).tolist() == [1] * g.B


@pytest.mark.parametrize("name", ["mazes032_neural_test", "warcraft12_synth"])
def test_golden_training_mode_masks(native, name):
    g = Golden(name)
    T = int(g.meta["train_Tmax"] * g.W * g.W)
    hist, paths, ts, ns, _ = _run_native(native, g.cost, g.start, g.goal, g.obst, g.g_ratio, T=T)
    np.testing.assert_array_equal(hist != 0, g.bits("train_hist_bits") != 0)
    np.testing.assert_array_equal(paths != 0, g.bits("train_path_bits") != 0)


def _random_problem(rng, B, H, W, p_obst, learned, unreachable_ok=True):
    obst = (rng.rand(B, 1, H, W) > p_obst).astype(np.float32)
    start = np.zeros((B, 1, H, W), np.float32)
    goal = np.zeros((B, 1, H, W), np.float32)
    for b in range(B):
        s, g_ = rng.randint(H * W, size=2)
        start[b, 0].flat[s] = 1
        goal[b, 0].flat[g_] = 1
        obst[b, 0].flat[s] = 1
        obst[b, 0].flat[g_] = 1
    if learned:
        cost = (1.0 / (1.0 + np.exp(-rng.randn(B, 1, H, W) * 2))).astype(np.float32) * np.float32(rng.choice([1.0, 10.0]))
    else:
        cost = obst.copy()
    return cost, start, goal, obst


SHAPES = [(32, 32), (12, 12), (1, 1), (1, 32), (32, 1), (5, 7), (31, 29), (16, 32), (32, 16), (3, 3), (20, 12), (12, 20),
          # engine 4 (nastar_warp64.cuh): up to 64x64, not both sides <= 32
          (33, 33), (1, 64), (64, 1), (2, 64), (64, 2), (32, 33), (33, 32), (40, 20), (63, 64), (47, 61),
          # generic engine: state in shared memory up to (131, 131), in the HBM workspace from (131, 132) on
          (65, 40), (1, 65), (70, 3), (97, 131), (131, 131), (131, 132), (144, 136)]


@pytest.mark.parametrize("learned", [False, True])
@pytest.mark.parametrize("H,W", SHAPES)
def test_random_vs_oracle(native, oracle, H, W, learned):
    """Every engine a shape selects (tests/test_abi_cpu.py pins the table).  Above 64x64 both cost kinds run on the
    generic engine: learned costs always do, and binary aliased planes do too because a trace is requested (engine 5
    records none).  When H > W the loop bound T = W*W is below N = H*W, so (64, 2) and (144, 136) also reach the step
    cap and the T-1 hop backtrack of unsolved maps."""
    rng = np.random.RandomState(1000 * H + 10 * W + int(learned))
    B = 24
    for p_obst, g_ratio in ((0.0, 0.5), (0.25, 0.5), (0.45, 0.5), (0.2, 0.8), (0.2, 0.3)):
        cost, start, goal, obst = _random_problem(rng, B, H, W, p_obst, learned)
        ref = oracle.forward(cost, start, goal, obst, g_ratio=g_ratio, mode="spec", want_trace=True)
        hist, paths, ts, ns, tr = _run_native(native, cost, start, goal, obst, g_ratio, trace=True, alias=not learned)
        np.testing.assert_array_equal(ts, ref.t_solve)
        np.testing.assert_array_equal(ns, ref.n_steps)
        np.testing.assert_array_equal(tr, ref.trace)
        np.testing.assert_array_equal(hist, ref.histories)
        np.testing.assert_array_equal(paths, ref.paths)


def test_step_cap_training(native, oracle):
    """Tmax < 1 in training mode caps the loop (differentiable_astar.py:200-202): capped maps report -1."""
    rng = np.random.RandomState(5)
    cost, start, goal, obst = _random_problem(rng, 64, 32, 32, 0.2, True)
    for Tmax in (0.25, 0.05, 1.0 / 1024):
        T = int(Tmax * 32 * 32)
        ref = oracle.forward(cost, start, goal, obst, Tmax=Tmax, training=True, mode="spec", want_trace=True)
        hist, paths, ts, ns, tr = _run_native(native, cost, start, goal, obst, 0.5, T=T, trace=True)
        np.testing.assert_array_equal(ts, ref.t_solve)
        np.testing.assert_array_equal(ns, ref.n_steps)
        np.testing.assert_array_equal(tr, ref.trace)
        np.testing.assert_array_equal(hist, ref.histories)
        np.testing.assert_array_equal(paths, ref.paths)
    assert (ts == -1).any()


def test_strided_and_multichannel_inputs(native, oracle):
    """Only channel 0 is searched (differentiable_astar.py:177-180); non-contiguous planes are accepted."""
    rng = np.random.RandomState(9)
    cost, start, goal, obst = _random_problem(rng, 8, 32, 32, 0.2, True)
    ref = oracle.forward(cost, start, goal, obst, mode="spec")
    c3 = torch.from_numpy(np.concatenate([cost, cost * 0 + 7, cost * 0 + 9], 1)).cuda()       # [B,3,H,W], stride 3*N
    big = torch.zeros((8, 1, 40, 40), device="cuda")
    big[:, :, 3:35, 5:37] = torch.from_numpy(obst).cuda()
    o_view = big[:, :, 3:35, 5:37]                                                            # non-contiguous rows
    hist, paths, ts, ns, _ = native.forward(c3, _dev(start), _dev(goal), o_view, 0.5, 1024, False)
    np.testing.assert_array_equal(hist.cpu().numpy(), ref.histories)
    np.testing.assert_array_equal(paths.cpu().numpy(), ref.paths)


def test_unreachable_goal_reports_exhausted(native):
    obst = np.ones((2, 1, 8, 8), np.float32)
    obst[:, 0, :, 4] = 0  # wall
    start = np.zeros_like(obst); start[:, 0, 0, 0] = 1
    goal = np.zeros_like(obst); goal[:, 0, 7, 7] = 1
    hist, paths, ts, ns, _ = _run_native(native, obst, start, goal, obst, alias=True)
    assert (ts == -2).all()          # NASTAR_TS_EXHAUSTED (the reference crashes here: NaN -> IndexError)
    assert hist.sum() == 2 * 8 * 4   # explored exactly the reachable half
    assert paths.sum() == 2          # only the goal cell is marked
    assert np.isfinite(hist).all()


LOWG = [n for n in NAMES if Golden(n).meta.get("lowg")]


@pytest.mark.parametrize("name", LOWG)
def test_low_g_ratio_batch_coupled_module_matches_reference(name):
    """g_ratio < 0.5 with B > 1: solved maps keep evolving until the slowest map is solved
    (differentiable_astar.py:251-252); the module reproduces the reference's masks and frame count."""
    from neural_astar.planner.differentiable_astar import DifferentiableAstar

    g = Golden(name)
    astar = DifferentiableAstar(g_ratio=g.g_ratio).cuda().eval()
    out = astar(_dev(g.cost), _dev(g.start), _dev(g.goal), _dev(g.obst), store_intermediate_results=True)
    np.testing.assert_array_equal(out.histories.cpu().numpy() != 0, g.bits("hist_bits") != 0)
    np.testing.assert_array_equal(out.paths.cpu().numpy() != 0, g.bits("path_bits") != 0)
    assert len(out.intermediate_results) == int(g.z["T_batch"]) + 1
    sel = torch.stack([f["paths"].reshape(g.B, -1).argmax(1) for f in out.intermediate_results[:-1]], 1)
    np.testing.assert_array_equal(sel.cpu().numpy(), g.z["trace"])


@pytest.mark.parametrize("H,W", [(32, 32), (12, 12), (64, 64), (20, 40), (65, 40), (144, 136)])
def test_no_early_exit_kernel_vs_oracle(native, oracle, H, W):
    """NASTAR_FWD_NO_EARLY_EXIT: exactly T steps per map, bit-exact trace vs the SPEC oracle in the same mode.  The
    batch-coupled path (g_ratio < 0.5) runs this mode on every engine, including the generic one ((65, 40) keeps its
    state in shared memory, (144, 136) in the HBM workspace)."""
    rng = np.random.RandomState(H + 3 * W)
    cost, start, goal, obst = _random_problem(rng, 12, H, W, 0.15, True)
    for g_ratio, T in ((0.0, 150), (0.3, 300), (0.5, 200)):
        T = min(T, W * W)
        ref = oracle.forward(cost, start, goal, obst, g_ratio=g_ratio, mode="spec", want_trace=True, T=T,
                             no_early_exit=True)
        hist, paths, ts, ns, tr = native.forward(_dev(cost), _dev(start), _dev(goal), _dev(obst), g_ratio, T, True, True)
        np.testing.assert_array_equal(tr.cpu().numpy(), ref.trace)
        np.testing.assert_array_equal(ts.cpu().numpy(), ref.t_solve)
        np.testing.assert_array_equal(ns.cpu().numpy(), ref.n_steps)
        np.testing.assert_array_equal(hist.cpu().numpy(), ref.histories)
        np.testing.assert_array_equal(paths.cpu().numpy(), ref.paths)
