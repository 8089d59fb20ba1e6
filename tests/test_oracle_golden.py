"""Pin the CPU oracle (oracle/astar_oracle.c) to the reference's own outputs.

Golden vectors come from running /root/reference's DifferentiableAstar on CPU
(tests/golden/make_golden.py).  Both restatements are checked:
  literal — the dense exp/softmax/first-argmax loop (differentiable_astar.py:203-252)
  spec    — the arg-min-over-(f, index) state machine the CUDA engine implements
Masks are compared bit-exactly; gradients to 1e-5 relative (north_star tolerance).
"""
import numpy as np
import pytest

from golden_util import Golden, all_names

NAMES = all_names()


def spec_batch_coupled(oracle, g):
    """SPEC form of the reference's batch-synchronous loop for g_ratio < 0.5 (the procedure the product's host
    side runs): step every map without early exit, find the first step at which ALL maps select their goal
    (differentiable_astar.py:219-220,251-252), then take the state after exactly that many steps."""
    T = g.W * g.W
    full = oracle.forward(g.cost, g.start, g.goal, g.obst, g_ratio=g.g_ratio, mode="spec", want_trace=True,
                          T=T, no_early_exit=True)
    at_goal = (full.trace == g.z["goal_idx"][:, None]).all(0)
    T_batch = int(np.argmax(at_goal)) + 1 if at_goal.any() else T
    o = oracle.forward(g.cost, g.start, g.goal, g.obst, g_ratio=g.g_ratio, mode="spec", want_trace=True,
                       T=T_batch, no_early_exit=True)
    return o, T_batch


def _run(oracle, g, mode, **kw):
    if mode == "spec" and g.meta.get("lowg"):
        o, T_batch = spec_batch_coupled(oracle, g)
        return o.histories, o.paths, T_batch
    if g.independent:
        outs = [oracle.forward(g.cost[i:i + 1], g.start[i:i + 1], g.goal[i:i + 1], g.obst[i:i + 1],
                               g_ratio=g.g_ratio, mode=mode, **kw) for i in range(g.B)]
        hist = np.concatenate([o.histories for o in outs])
        paths = np.concatenate([o.paths for o in outs])
        tb = np.array([o.T_batch for o in outs])
        return hist, paths, tb
    o = oracle.forward(g.cost, g.start, g.goal, g.obst, g_ratio=g.g_ratio, mode=mode, **kw)
    return o.histories, o.paths, o.T_batch


@pytest.mark.parametrize("mode", ["literal", "spec"])
@pytest.mark.parametrize("name", NAMES)
def test_forward_masks_match_reference(oracle, name, mode):
    g = Golden(name)
    hist, paths, tb = _run(oracle, g, mode)
    assert hist.dtype == np.float32 and paths.dtype == np.int64
    np.testing.assert_array_equal(hist != 0, g.bits("hist_bits") != 0)
    np.testing.assert_array_equal(paths != 0, g.bits("path_bits") != 0)
    assert set(np.unique(hist)) <= {0.0, 1.0}
    if g.independent:
        np.testing.assert_array_equal(tb, g.z["T_batch_each"])
    else:
        assert int(tb) == int(g.z["T_batch"])


@pytest.mark.parametrize("name", [n for n in NAMES if "trace" in Golden(n).z])
def test_selection_trace_matches_reference(oracle, name):
    """Step-by-step selected node indices vs the reference's.

    LITERAL must reproduce every step.  SPEC (arg-min over exact f, what the CUDA engine does) may
    only differ where the reference's fl(exp(-f/sqrt(W))) merges two DISTINCT f values into equal
    softmax weights and then breaks the "tie" by index (DESIGN.md "selection semantics"): such an
    event swaps two consecutive selections.  It occurs once in these vectors
    (mpd032_families_vanilla map 64, steps 135/136: f = 16.009552 vs 16.009553).
    """
    g = Golden(name)
    ref = g.z["trace"]  # [B, T_batch]
    lit = oracle.forward(g.cost, g.start, g.goal, g.obst, g_ratio=g.g_ratio, mode="literal", want_trace=True)
    np.testing.assert_array_equal(lit.trace[:, : ref.shape[1]], ref)
    if g.meta.get("lowg"):
        # batch-coupled: every step of every map is defined by the reference, post-solve steps included
        o, T_batch = spec_batch_coupled(oracle, g)
        assert T_batch == ref.shape[1]
        np.testing.assert_array_equal(o.trace, ref)
        return
    o = oracle.forward(g.cost, g.start, g.goal, g.obst, g_ratio=g.g_ratio, mode="spec", want_trace=True)
    swapped = 0
    for b in range(g.B):
        n = int(o.n_steps[b])
        diff = np.nonzero(o.trace[b, :n] != ref[b, :n])[0]
        if len(diff):
            # only adjacent transpositions are tolerated
            assert len(diff) % 2 == 0
            for i in range(0, len(diff), 2):
                a, c = diff[i], diff[i + 1]
                assert c == a + 1 and o.trace[b, a] == ref[b, c] and o.trace[b, c] == ref[b, a]
            swapped += len(diff) // 2
        # post-solve steps of the reference keep re-selecting the goal (SURVEY App. A.4)
        assert (ref[b, n:] == g.z["goal_idx"][b]).all()
    total = int(o.n_steps.sum())
    assert swapped <= max(1, total // 10000), f"{swapped} exp-collision swaps in {total} selections"


def test_adversarial_near_tie_is_the_documented_one_cell_deviation(oracle):
    """tests/golden/adversarial_neartie.npz: two open cells with f one ulp apart and equal rounded exp.  LITERAL (the
    reference's own selection rule) must reproduce the reference step for step; SPEC (arg-min over exact f — what the
    CUDA engine implements, DESIGN.md "Selection semantics") expands the smaller f first, reaches the goal one step
    earlier and leaves exactly ONE cell — (1,2) — out of `histories`; paths are identical."""
    g = Golden("adversarial_neartie")
    ref_h, ref_p = g.bits("hist_bits") != 0, g.bits("path_bits") != 0
    lit = oracle.forward(g.cost, g.start, g.goal, g.obst, mode="literal", want_trace=True)
    np.testing.assert_array_equal(lit.histories != 0, ref_h)
    np.testing.assert_array_equal(lit.paths != 0, ref_p)
    np.testing.assert_array_equal(lit.trace[:, : g.z["trace"].shape[1]], g.z["trace"])
    spec = oracle.forward(g.cost, g.start, g.goal, g.obst, mode="spec")
    np.testing.assert_array_equal(spec.paths != 0, ref_p)
    diff = (spec.histories != 0) != ref_h
    y, x = g.meta["extra_cell"]
    for b in range(g.B):
        assert diff[b].sum() == 1 and diff[b, 0, y, x] and ref_h[b, 0, y, x] and not spec.histories[b, 0, y, x]
    np.testing.assert_array_equal(spec.n_steps + 1, g.z["hist_sum"])       # one expansion fewer than the reference


@pytest.mark.parametrize("name", ["mazes032_neural_test", "warcraft12_synth"])
def test_training_mode_forward(oracle, name):
    g = Golden(name)
    for mode in ("literal", "spec"):
        o = oracle.forward(g.cost, g.start, g.goal, g.obst, g_ratio=g.g_ratio, Tmax=g.meta["train_Tmax"],
                           training=True, mode=mode)
        np.testing.assert_array_equal(o.histories != 0, g.bits("train_hist_bits") != 0)
        np.testing.assert_array_equal(o.paths != 0, g.bits("train_path_bits") != 0)
        assert o.T_batch == int(g.z["train_T_batch"])


def _relerr(a, b):
    return float(np.abs(a - b).max() / (np.abs(b).max() + 1e-30))


def test_backward_l1_training_grad(oracle):
    """dL/dcost of the L1 training loss (utils/training.py:58), Tmax=0.25, vs reference autograd."""
    g = Golden("mazes032_neural_test")
    hist = g.bits("train_hist_bits").astype(np.float32)
    opt = g.bits("opt_bits").astype(np.float32)
    G = np.sign(hist - opt) / hist.size
    gc = oracle.backward(g.cost, g.start, g.goal, g.obst, G, int(g.z["train_T_batch"]), g_ratio=g.g_ratio)
    assert _relerr(gc, g.plane("train_grad_cost")) < 1e-5


@pytest.mark.parametrize("name,T_key,G_key,out_key", [
    ("mazes032_lowg_gr00_cost10", "T_batch", "rand_G", "rand_grad_cost"),   # g_ratio < 0.5: post-solve steps matter
    ("mazes032_lowg_gr02", "T_batch", "rand_G", "rand_grad_cost"),
    ("mazes032_lowg_gr04_cost10", "T_batch", "rand_G", "rand_grad_cost"),
    ("mazes032_neural_test", "T_batch", "rand_G", "rand_grad_cost"),
    ("warcraft12_synth", "T_batch", "rand_G", "rand_grad_cost"),
    ("warcraft12_synth", "train_T_batch", "rand_G", "train_grad_cost"),
])
def test_backward_random_upstream(oracle, name, T_key, G_key, out_key):
    g = Golden(name)
    gc = oracle.backward(g.cost, g.start, g.goal, g.obst, g.plane(G_key), int(g.z[T_key]), g_ratio=g.g_ratio)
    assert _relerr(gc, g.plane(out_key)) < 1e-5


def test_mechanism_codes_match_the_header():
    """The bindings' mechanism codes are NASTAR_MECH_MOORE / NASTAR_MECH_NEWS of include/nastar_b200.h, and a name
    outside them is a ValueError in every binding."""
    import os
    import re

    from oracle import labels, wlabels
    from oracle import oracle as search

    header = open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include",
                               "nastar_b200.h")).read()
    defined = {m.lower(): int(v) for m, v in re.findall(r"#define NASTAR_MECH_(\w+)\s+(\d+)", header)}
    assert search.MECHANISMS == defined == {"moore": 0, "news": 1}
    plane = np.zeros((1, 1, 3, 3), np.float32)
    plane[0, 0, 0, 0] = 1
    with pytest.raises(ValueError, match="mechanism"):
        search.forward(plane, plane, plane, plane, mechanism="hex")
    with pytest.raises(ValueError, match="mechanism"):
        search.backward(plane, plane, plane, plane, plane, 1, mechanism="hex")
    with pytest.raises(ValueError, match="mechanism"):
        labels.opt_labels(plane, [0], mechanism="hex")
    with pytest.raises(ValueError, match="mechanism"):
        wlabels.weighted_labels(plane, [0], mechanism="hex")
