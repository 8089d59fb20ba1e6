"""GPU tests of the round-2 additions, all through the C ABI of libnastar_b200.so:

  * engine 5 (csrc/nastar_bin16.cuh, binary-cost maps, CTA per map) vs the SPEC oracle, incl. the maps it must
    hand back to the generic engine (non-binary aliased costs) and the edge cases of the other engines;
  * NASTAR_FWD_PAIR (validation pair in one launch) and the per-map counts;
  * the fused encoder hand-off: pack_inputs, NASTAR_COST_LOGIT / NASTAR_COST_TAPS prologues, sigmoid bit-exactness
    against torch.sigmoid, NeuralAstar's fused forward vs the unfused composition;
  * GraphedPlanner.replay_host and PipelinedPlanner vs the eager call;
  * validation metrics from one launch vs the two-call path and the reference's anchors.
"""
import os

import numpy as np
import pytest
import torch

import encoder_exact_oracle as eo
from golden_util import Golden

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def native():
    from neural_astar import _native

    _native.lib()
    return _native


def _cu(x):
    return torch.from_numpy(np.ascontiguousarray(x)).cuda()


def _corner_problem(rng, B, H, W, p_obst=0.2):
    obst = (rng.rand(B, 1, H, W) > p_obst).astype(np.float32)
    start = np.zeros((B, 1, H, W), np.float32)
    goal = np.zeros((B, 1, H, W), np.float32)
    for b in range(B):
        ys, xs = rng.randint(max(1, H // 4)), rng.randint(max(1, W // 4))
        yg, xg = H - 1 - rng.randint(max(1, H // 4)), W - 1 - rng.randint(max(1, W // 4))
        obst[b, 0, ys, xs] = obst[b, 0, yg, xg] = 1
        start[b, 0, ys, xs] = 1
        goal[b, 0, yg, xg] = 1
    return obst, start, goal


def _ckpt_planner():
    from neural_astar.planner import NeuralAstar

    state = np.load(os.path.join(ROOT, "tests", "golden", "mazes032_ckpt_planner_state.npz"))
    na = NeuralAstar(encoder_arch="CNN")
    na.load_state_dict({k: torch.from_numpy(state[k]) for k in state.files})
    return na.cuda().eval()


# ------------------------------------------------------------------------------------------------ engine 5
@pytest.mark.parametrize("H,W,B", [(256, 256, 6), (128, 128, 8), (97, 131, 4), (200, 300, 3), (65, 40, 5), (300, 70, 3)])
def test_bin16_engine_vs_oracle(native, oracle, H, W, B):
    """Binary aliased cost planes run on engine 5; outputs (incl. solve step and step count) equal the oracle's."""
    assert native.lib().nastar_b200_bin16_supported(H, W) == 1
    rng = np.random.RandomState(7 * H + W)
    obst, start, goal = _corner_problem(rng, B, H, W)
    ref = oracle.forward(obst, start, goal, obst, mode="spec")
    c = _cu(obst)
    before = native.launch_count()
    hist, paths, ts, ns, _, (ncl, plen) = native.forward(c, _cu(start), _cu(goal), c, 0.5, W * W, want_counts=True)
    assert native.launch_count() - before == 2          # engine 5 + the (empty) redo pass of the generic engine
    np.testing.assert_array_equal(ts.cpu().numpy(), ref.t_solve)
    np.testing.assert_array_equal(ns.cpu().numpy(), ref.n_steps)
    np.testing.assert_array_equal(hist.cpu().numpy(), ref.histories)
    np.testing.assert_array_equal(paths.cpu().numpy(), ref.paths)
    np.testing.assert_array_equal(ncl.cpu().numpy(), ref.histories.sum((1, 2, 3)).astype(np.int64))
    np.testing.assert_array_equal(plen.cpu().numpy(), ref.paths.sum((1, 2, 3)))


def test_bin16_sqrt_is_ieee_for_every_reachable_argument(native):
    """Engine 5 evaluates get_heuristic's sqrt with a branch-free sequence; it must equal the IEEE-rounded sqrtf for
    every integer dy^2 + dx^2 a map of up to 512 rows / 1024 columns can produce."""
    import ctypes

    n = 511 * 511 + 1023 * 1023 + 1
    bad = torch.zeros(1, dtype=torch.int32, device="cuda")
    st = native.lib().nastar_b200_selftest_sqrt(n, bad.data_ptr(), ctypes.c_void_p(torch.cuda.current_stream().cuda_stream))
    assert st == 0 and int(bad.item()) == 0


def test_bin16_edge_cases_and_redo(native, oracle):
    """Unreachable goal, start == goal, start on an obstacle cell, g_ratio != 0.5, a step cap, and a batch in which
    some maps carry non-binary costs (those are re-run by the generic engine inside the same call)."""
    H, W, B = 96, 128, 8
    rng = np.random.RandomState(5)
    obst, start, goal = _corner_problem(rng, B, H, W, p_obst=0.25)
    # map 0: goal walled in
    gy, gx = np.argwhere(goal[0, 0])[0]
    obst[0, 0, max(gy - 1, 0):gy + 2, max(gx - 1, 0):gx + 2] = 0
    obst[0, 0, gy, gx] = 1
    # map 1: start == goal
    goal[1] = start[1]
    # map 2: start on an obstacle cell (cost 0 there)
    sy, sx = np.argwhere(start[2, 0])[0]
    obst[2, 0, sy, sx] = 0
    # maps 5..7: non-binary values in the aliased plane -> handed to the generic engine
    cost = obst.copy()
    cost[5:] *= (0.5 + rng.rand(3, 1, H, W)).astype(np.float32)
    for g_ratio, T in ((0.5, W * W), (0.7, W * W), (0.5, 300)):
        ref = oracle.forward(cost, start, goal, cost, g_ratio=g_ratio, mode="spec", T=T)
        c = _cu(cost)
        hist, paths, ts, ns, _ = native.forward(c, _cu(start), _cu(goal), c, g_ratio, T)
        np.testing.assert_array_equal(ts.cpu().numpy(), ref.t_solve)
        np.testing.assert_array_equal(ns.cpu().numpy(), ref.n_steps)
        np.testing.assert_array_equal(hist.cpu().numpy(), ref.histories)
        solved = ref.t_solve != -2
        np.testing.assert_array_equal(paths.cpu().numpy()[solved], ref.paths[solved])
    assert ref.t_solve[0] == -2 or T == 300


def test_bin16_matches_generic_engine_on_config5_maps(native):
    """Config-5-style maps (256x256, 20 % obstacles, far apart start/goal): engine 5 and engine 3 agree bit for bit
    (the same inputs, non-aliased, take the generic path)."""
    H = W = 256
    rng = np.random.RandomState(11)
    obst, start, goal = _corner_problem(rng, 12, H, W)
    c, s, g = _cu(obst), _cu(start), _cu(goal)
    a = native.forward(c, s, g, c, 0.5, W * W)
    b = native.forward(c.clone(), s, g, c, 0.5, W * W)      # different pointer for cost: not aliased
    for x, y in zip(a[:4], b[:4]):
        assert torch.equal(x, y)


# ------------------------------------------------------------------------------------------------ pair + counts
@pytest.mark.parametrize("H,W", [(32, 32), (20, 12), (64, 64), (96, 80)])
def test_pair_launch_equals_two_calls(native, H, W):
    rng = np.random.RandomState(H * 3 + W)
    B = 9
    obst, start, goal = _corner_problem(rng, B, H, W)
    cost = (obst * (0.2 + rng.rand(B, 1, H, W))).astype(np.float32)
    c, s, g, o = _cu(cost), _cu(start), _cu(goal), _cu(obst)
    native.forward(c, s, g, o, 0.5, W * W)      # one-time table fill of the warp engines is a launch of its own
    before = native.launch_count()
    hist, paths, ts, ns, _, (ncl, plen) = native.forward(c, s, g, o, 0.5, W * W, pair=True, want_counts=True)
    n_launch = native.launch_count() - before
    if H <= 32 and W <= 32:
        assert n_launch == 1                      # both searches in ONE kernel launch
    learned = native.forward(c, s, g, o, 0.5, W * W)
    vanilla = native.forward(o, s, g, o, 0.5, W * W)
    assert hist.shape[0] == 2 * B
    for k in range(4):
        assert torch.equal((hist, paths, ts, ns)[k][:B], learned[k])
        assert torch.equal((hist, paths, ts, ns)[k][B:], vanilla[k])
    np.testing.assert_array_equal(ncl.cpu().numpy(), hist.sum((1, 2, 3)).long().cpu().numpy())
    np.testing.assert_array_equal(plen.cpu().numpy(), paths.sum((1, 2, 3)).cpu().numpy())


def test_validation_step_one_launch_matches_two_calls_and_reference_anchor():
    """SURVEY 8(f)-2: PlannerModule.validation_step issues ONE search launch for the learned + vanilla pair; its
    metrics equal the two-call formulas and the reference's checkpoint anchor (p_opt 0.80 / p_exp 0.445 / h_mean
    0.572 on the test split, SURVEY section 6)."""
    from types import SimpleNamespace

    from neural_astar import _native
    from neural_astar.planner import VanillaAstar
    from neural_astar.utils.training import PlannerModule, planner_metrics

    g = Golden("mazes032_vanilla_test")
    na = _ckpt_planner()
    mod = PlannerModule(na, SimpleNamespace(params=SimpleNamespace(lr=1e-3))).cuda().eval()
    maps, start, goal = (_cu(x) for x in (g.obst, g.start, g.goal))
    opt = torch.zeros_like(start)
    with torch.no_grad():
        mod.validation_step((maps, start, goal, opt), 0)          # warm-up (plan building, autotuning)
        before = _native.launch_count()
        mod.validation_step((maps, start, goal, opt), 0)
        # pack_inputs + head products + ONE search launch (both halves)
        assert _native.launch_count() - before == 3
        got = tuple(mod.logged[f"metrics/{k}"] for k in ("p_opt", "p_exp", "h_mean"))
        out = na(maps, start, goal)
        va = VanillaAstar().cuda()(maps, start, goal)
    want = planner_metrics(out, va)
    assert got == pytest.approx(want, abs=1e-9)
    assert abs(got[0] - 0.80) <= 0.03 and abs(got[1] - 0.445) <= 0.02 and abs(got[2] - 0.572) <= 0.02
    np.testing.assert_array_equal(va.histories.cpu().numpy() != 0, g.bits("hist_bits") != 0)


# ------------------------------------------------------------------------------------------------ fused hand-off
def test_sigmoid_prologue_is_bit_exact_with_torch(native):
    """NASTAR_COST_LOGIT / cost_from_taps reproduce torch.sigmoid(x) * const bit for bit (encoder.py:32-34)."""
    torch.manual_seed(0)
    B, H, W = 7, 32, 32
    x = torch.cat([torch.randn(B, 1, H, W) * 4, torch.tensor([0.0, -0.0, 88.0, -88.0, 104.0, -104.0, 1e-8, -20.0] * 128)
                   .reshape(1, 1, H, W)]).cuda()
    for scale in (1.0, 10.0, 0.37):
        want = torch.sigmoid(x) * scale
        taps = torch.zeros((B + 1, H, W, 9), device="cuda")
        taps[..., 4] = x[:, 0]
        got = native.cost_from_taps(taps, 0.0, scale)
        assert torch.equal(got, want)


def test_cost_kinds_equal_plane_search(native):
    rng = np.random.RandomState(3)
    for (H, W) in ((32, 32), (12, 12), (20, 31), (64, 64), (40, 57), (33, 64)):     # engine 1 and engine 4 shapes
        B = 6
        obst, start, goal = _corner_problem(rng, B, H, W, p_obst=0.1)
        s, g, o = _cu(start), _cu(goal), _cu(obst)
        logits = torch.from_numpy(rng.randn(B, 1, H, W).astype(np.float32) * 2).cuda()
        taps = torch.from_numpy(rng.randn(B, H, W, 9).astype(np.float32)).cuda()
        bias, scale = 0.3, 10.0
        # LOGIT
        plane = torch.sigmoid(logits) * scale
        a = native.forward(plane, s, g, o, 0.5, W * W)
        b = native.forward(logits, s, g, o, 0.5, W * W, cost_kind=native.COST_LOGIT, cost_scale=scale)
        for x, y in zip(a[:4], b[:4]):
            assert torch.equal(x, y)
        # TAPS: the glue kernel and the prologue share one device function; the gather itself is checked against
        # a plain PyTorch fp32 convolution of the same 9 one-hot taps
        plane = native.cost_from_taps(taps, bias, scale)
        w = torch.zeros(1, 9, 3, 3, device="cuda")
        for k in range(9):
            w[0, k, k // 3, k % 3] = 1.0
        with torch.backends.cudnn.flags(enabled=False):
            ref = torch.sigmoid(torch.nn.functional.conv2d(taps.permute(0, 3, 1, 2), w, padding=1) + bias) * scale
        assert float((plane - ref).abs().max()) <= 2e-5
        a = native.forward(plane, s, g, o, 0.5, W * W)
        b = native.forward(taps, s, g, o, 0.5, W * W, cost_kind=native.COST_TAPS, cost_scale=scale, cost_bias=bias)
        for x, y in zip(a[:4], b[:4]):
            assert torch.equal(x, y)
    with pytest.raises(RuntimeError):      # fused kinds are for H, W <= 64
        big = torch.zeros((1, 1, 80, 80), device="cuda")
        native.forward(big, big, big, big, 0.5, 80 * 80, cost_kind=native.COST_LOGIT)


@pytest.mark.parametrize("C,B,H", [(256, 7, 32), (128, 5, 12), (64, 3, 20), (32, 2, 9)])
def test_head_taps_kernel_matches_fp32_matmul(native, C, B, H):
    """Encoder head: per-pixel [C] x [C,9] products from the streaming kernel, bit-equal to the same fp32 operation
    sequence replayed on the CPU (eo.head_taps_replay: ascending channel, one fmaf per product)."""
    torch.manual_seed(C)
    x = torch.randn(B, C, H, H, device="cuda").contiguous(memory_format=torch.channels_last)
    w = torch.randn(C, 9, device="cuda") / C ** 0.5
    want = eo.head_taps_replay(x.permute(0, 2, 3, 1).reshape(-1, C).cpu().numpy(), w.cpu().numpy())
    got = native.head_taps(x, w.cpu().numpy())
    assert got.shape == (B, H, H, 9)
    assert np.array_equal(got.view(-1, 9).cpu().numpy(), want)
    buf = torch.empty_like(got)
    assert native.head_taps(x, w.cpu().numpy(), out=buf).data_ptr() == buf.data_ptr() and torch.equal(buf, got)


@pytest.mark.parametrize("B,H,W", [(7, 32, 32), (3, 20, 27), (2, 64, 64), (1, 5, 3)])
def test_conv1_marks_matches_torch_conv(native, B, H, W):
    """First encoder layer fused with the input assembly: relu(conv2d(cat(map, start + goal), w, b)), channels-last,
    bit-equal to the kernel's fp32 operation sequence replayed on the CPU (eo.conv1_marks_replay)."""
    torch.manual_seed(B * H + W)
    maps = (torch.rand(B, 1, H, W, device="cuda") > 0.2).float()
    start = torch.zeros(B, 1, H, W, device="cuda")
    goal = torch.zeros_like(start)
    for b in range(B):
        start[b, 0, b % H, (3 * b) % W] = 1
        goal[b, 0, H - 1 - b % H, W - 1] = 1
    w = torch.randn(32, 2, 3, 3, device="cuda") * 0.3
    bias = torch.randn(32, device="cuda") * 0.1
    wh = np.ascontiguousarray(w.permute(2, 3, 1, 0).reshape(9, 2, 32).cpu().numpy())
    bh = bias.cpu().numpy()
    want = eo.conv1_marks_replay(maps.cpu().numpy(), start.cpu().numpy(), goal.cpu().numpy(), wh, bh)
    got = native.conv1_marks(maps, start, goal, wh, bh)
    assert got.shape == (B, 32, H, W) and got.is_contiguous(memory_format=torch.channels_last)
    assert np.array_equal(got.permute(0, 2, 3, 1).cpu().numpy(), want)
    # strided one-hot planes (views into a stacked request buffer) are read in place
    stacked = torch.stack((maps, start, goal), 0)
    got2 = native.conv1_marks(stacked[0], stacked[1], stacked[2], wh, bh)
    assert torch.equal(got2, got)
    with pytest.raises(ValueError):
        native.conv1_marks(maps.repeat(1, 2, 1, 1), start, goal, wh, bh)


def test_first_layer_kernel_equals_packed_cudnn_path(native, monkeypatch):
    """NeuralAstar.forward with the engine's first-layer kernel vs the pack_inputs + cuDNN first layer (both fp32, other
    layers identical): the 9-tap products agree to fp32 rounding and the search masks are the same on this batch."""
    from neural_astar.planner import NeuralAstar, encoder

    torch.manual_seed(3)
    na = NeuralAstar(encoder_input="m+", encoder_arch="CNN", encoder_depth=4).cuda().eval()
    B, H = 24, 32
    x = (torch.rand(B, 1, H, H, device="cuda") > 0.15).float()
    s = torch.zeros(B, 1, H, H, device="cuda"); s[:, :, 0, 0] = 1
    g = torch.zeros_like(s); g[:, :, -1, -1] = 1
    x[:, :, 0, 0] = 1; x[:, :, -1, -1] = 1
    monkeypatch.setattr(encoder, "ALLOW_TF32", False)
    with torch.no_grad():
        assert na.encoder.head_taps_marks(x, s, g) is not None
        t_new = na._head_taps(x, s, g)[0].clone()
        out_new = na(x, s, g)
        monkeypatch.setattr(encoder, "CONV1_KERNEL", False)
        assert na.encoder.head_taps_marks(x, s, g) is None
        t_old = na._head_taps(x, s, g)[0].clone()
        out_old = na(x, s, g)
    assert float((t_new - t_old).abs().max()) < 1e-4
    assert int((out_new.histories != out_old.histories).flatten(1).any(1).sum()) <= 1
    assert int((out_new.paths != out_old.paths).flatten(1).any(1).sum()) <= 1


@pytest.mark.parametrize("C,Hm,H", [(1, 32, 32), (3, 96, 12), (2, 24, 12), (1, 64, 64)])
def test_pack_inputs_matches_torch(native, C, Hm, H):
    torch.manual_seed(C + Hm)
    B = 5
    maps = torch.rand(B, C, Hm, Hm, device="cuda")
    start = torch.zeros(B, 1, H, H, device="cuda")
    goal = torch.zeros_like(start)
    for b in range(B):
        start[b, 0, b % H, (3 * b) % H] = 1
        goal[b, 0, H - 1 - b % H, H - 1] = 1
    marks = start + goal
    if Hm != H:
        marks = torch.nn.functional.interpolate(marks, size=(Hm, Hm), mode="nearest")
    want = torch.cat((maps, marks), dim=1)
    got = native.pack_inputs(maps, start, goal)
    assert got.shape == want.shape and got.is_contiguous(memory_format=torch.channels_last)
    assert torch.equal(got, want)


@pytest.mark.parametrize("arch,inp,depth,const,shape,hw", [("CNN", "m+", 4, None, (16, 1, 32, 32), 32),
                                                            ("CNNDownSize", "rgb+", 3, 10.0, (8, 3, 96, 96), 12),
                                                            ("CNN", "m+", 4, None, (6, 1, 64, 64), 64),
                                                            ("CNN", "m+", 3, 5.0, (5, 1, 48, 48), 48)])
def test_fused_forward_equals_unfused_composition(native, arch, inp, depth, const, shape, hw):
    """NeuralAstar.forward in eval mode (pack kernel -> convs -> head GEMM -> search with the TAPS prologue) gives
    exactly the outputs of encode() followed by the plain search: the cost arithmetic is one shared device function."""
    from neural_astar.planner import NeuralAstar

    torch.manual_seed(1)
    na = NeuralAstar(encoder_input=inp, encoder_arch=arch, encoder_depth=depth, const=const,
                     learn_obstacles=(arch != "CNN")).cuda()
    x = (torch.rand(shape, device="cuda") > 0.15).float() if shape[1] == 1 else torch.rand(shape, device="cuda")
    s = torch.zeros((shape[0], 1, hw, hw), device="cuda"); s[:, :, 0, 0] = 1
    g = torch.zeros_like(s); g[:, :, -1, -1] = 1
    if shape[1] == 1:
        x[:, :, 0, 0] = 1; x[:, :, -1, -1] = 1
    na.train()
    for _ in range(2):
        na.encode(x, s, g)      # non-trivial BatchNorm statistics
    na.eval()
    with torch.no_grad():
        na(x, s, g)             # plan building
        before = native.launch_count()
        out = na(x, s, g, store_intermediate_results=False)
        assert native.launch_count() - before == 3          # first layer (or pack_inputs) + head products + search; the rest is cuDNN
        cost = na.encode(x, s, g)
        passable = torch.ones_like(s) if na.learn_obstacles else x
        want = na.perform_astar(cost, s, g, passable)
        frames = na(x, s, g, store_intermediate_results=True)
    assert torch.equal(out.histories, want.histories) and torch.equal(out.paths, want.paths)
    assert torch.equal(frames.histories, want.histories) and len(frames.intermediate_results) >= 2
    # the cost maps themselves agree with the module's own (slow, autograd) path to TF32 accuracy
    slow = na.encode(x, s, g)
    assert slow.requires_grad
    assert float((cost - slow).abs().max()) < 3e-3 * (1.0 if const is None else const)


def test_tf32_encoder_mask_differences_are_counted():
    """VERDICT r1 weak #5: how many of the 100 headline maps change their search masks because the encoder's convs
    run in TF32 (the fast path's default, like torch's own cuDNN default) instead of fp32 — against the reference's
    CPU outputs for the same checkpoint (mazes032_neural_test).  Prints the counts; bounds them loosely."""
    import neural_astar.planner.encoder as enc

    g = Golden("mazes032_vanilla_test")
    gn = Golden("mazes032_neural_test")
    na = _ckpt_planner()
    maps, start, goal = (_cu(x) for x in (g.obst, g.start, g.goal))
    res = {}
    old = enc.ALLOW_TF32
    try:
        for tf32 in (True, False):
            enc.ALLOW_TF32 = tf32
            with torch.no_grad():
                out = na(maps, start, goal)
                cost = na.encode(maps, start, goal)
            dh = (out.histories.cpu().numpy() != 0) != (gn.bits("hist_bits") != 0)
            dp = (out.paths.cpu().numpy() != 0) != (gn.bits("path_bits") != 0)
            res[tf32] = dict(maps_hist_differ=int(dh.reshape(100, -1).any(1).sum()),
                             maps_path_differ=int(dp.reshape(100, -1).any(1).sum()),
                             cells_hist_differ=int(dh.sum()),
                             max_cost_err=float((cost.cpu() - torch.from_numpy(gn.cost)).abs().max()))
    finally:
        enc.ALLOW_TF32 = old
    print("encoder precision vs reference masks (100 maps):", res)
    assert res[False]["max_cost_err"] < 1e-4 and res[True]["max_cost_err"] < 5e-3
    assert res[False]["maps_hist_differ"] <= 15 and res[True]["maps_hist_differ"] <= 60


def test_warp64_engine_on_the_whole_all064_test_split(native, oracle):
    """All 400 test problems of the reference's 64x64 dataset (all_064_moore_c16) through the warp-resident 64-wide
    engine: histories / paths bit-exact against the reference's own VanillaAstar outputs
    (tests/golden/inputs_all064_test400.npz); the CPU oracle is pinned to the same vectors on a sample."""
    g = Golden("inputs_all064_test400")
    c, s, gl = _cu(g.obst), _cu(g.start), _cu(g.goal)
    hist, paths, ts, ns, _ = native.forward(c, s, gl, c, 0.5, 64 * 64)
    np.testing.assert_array_equal(hist.cpu().numpy() != 0, g.bits("hist_bits") != 0)
    np.testing.assert_array_equal(paths.cpu().numpy() != 0, g.bits("path_bits") != 0)
    np.testing.assert_array_equal(ns.cpu().numpy(), g.z["hist_sum"])
    sl = slice(0, 400, 40)
    ref = oracle.forward(g.obst[sl], g.start[sl], g.goal[sl], g.obst[sl], mode="literal")
    np.testing.assert_array_equal(ref.histories != 0, g.bits("hist_bits")[sl] != 0)


def test_end_to_end_masks_on_all_1000_maps():
    """System-level parity on the whole mazes_032 dataset (800 train + 100 valid + 100 test problems): NeuralAstar
    with the shipped checkpoint through the engine's fused forward vs the masks the REFERENCE produced for the same
    inputs on CPU (tests/golden/inputs_mazes032_all1000.npz).  The search itself is bit-exact; what can differ is the
    cost map: the cuDNN encoder's TF32 convolutions perturb costs at the 5e-4 level (fp32 convs: 1e-6), which flips a
    near-tie selection in a few maps.  Both settings are counted, recorded and bounded (first measurement: TF32
    9 / 1000 maps differ in histories, 5 in paths)."""
    import neural_astar.planner.encoder as enc

    g = Golden("inputs_mazes032_all1000")
    na = _ckpt_planner()
    ref_h, ref_p = g.bits("neural_hist_bits") != 0, g.bits("neural_path_bits") != 0
    maps, start, goal = (_cu(x) for x in (g.obst, g.start, g.goal))
    res = {}
    old = enc.ALLOW_TF32
    try:
        for tf32 in (True, False):
            enc.ALLOW_TF32 = tf32
            dh = dp = 0
            with torch.no_grad():
                for i in range(0, 1000, 100):
                    out = na(maps[i:i + 100], start[i:i + 100], goal[i:i + 100])
                    h, p = out.histories.cpu().numpy() != 0, out.paths.cpu().numpy() != 0
                    dh += int((h != ref_h[i:i + 100]).reshape(100, -1).any(1).sum())
                    dp += int((p != ref_p[i:i + 100]).reshape(100, -1).any(1).sum())
            res["tf32" if tf32 else "fp32"] = {"maps": 1000, "maps_hist_differ": dh, "maps_path_differ": dp}
    finally:
        enc.ALLOW_TF32 = old
    print("end-to-end vs reference on 1000 maps:", res)
    assert res["fp32"]["maps_hist_differ"] <= 10 and res["fp32"]["maps_path_differ"] <= 10
    assert res["tf32"]["maps_hist_differ"] <= 40 and res["tf32"]["maps_path_differ"] <= 40


# ------------------------------------------------------------------------------------------------ graphs / pipeline
@pytest.mark.parametrize("fork", ["late", "early"])
def test_pipelined_and_host_graphs_match_eager(fork):
    from neural_astar.utils.inference import GraphedPlanner, PipelinedPlanner

    g = Golden("mazes032_vanilla_test")
    na = _ckpt_planner()
    maps, start, goal = (_cu(x) for x in (g.obst, g.start, g.goal))
    torch.manual_seed(0)
    batches = []
    for k in range(5):
        perm = torch.randperm(100, device="cuda")
        batches.append((maps[perm], start[perm], goal[perm]))
    with torch.no_grad():
        want = [na(*b) for b in batches]
    # device-resident pipeline
    pipe = PipelinedPlanner(na, maps, start, goal, fork=fork)
    got = []
    for b in batches:
        prev = pipe.submit(*b)
        if prev is not None:
            got.append((prev.histories.clone(), prev.paths.clone()))
    last = pipe.drain()
    got.append((last.histories.clone(), last.paths.clone()))
    assert len(got) == 5
    for (h, p), w in zip(got, want):
        assert torch.equal(h, w.histories) and torch.equal(p, w.paths)
    # stacked delivery (one copy per batch)
    prev = None
    for k, b in enumerate(batches[:3]):
        prev = pipe.submit_stacked(torch.stack(b))
        if k >= 1:
            assert torch.equal(prev.histories, want[k - 1].histories)
    last = pipe.drain()
    assert torch.equal(last.histories, want[2].histories) and torch.equal(last.paths, want[2].paths)
    # host pipeline (three stages: H2D(k) || encoder(k-1) || search(k-2) + D2H): pinned in, pinned out
    pipe = PipelinedPlanner(na, maps, start, goal, host=True, fork=fork)
    assert pipe.depth == 3 and len(pipe.host_inputs) == 3 and len(pipe.host_outputs) == 2
    results = []
    for k, b in enumerate(batches):
        torch.cuda.synchronize()                    # the staging buffer's previous batch has been consumed
        for dst, src in zip(pipe.host_inputs[k % 3], b):
            dst.copy_(src.cpu())
        out = pipe.submit()
        assert (out is None) == (k < 2)
        if k >= 2:
            torch.cuda.synchronize()
            assert torch.equal(out.histories, want[k - 2].histories)
            results.append(tuple(t.clone() for t in pipe.host_outputs[(k - 2) % 2]))
    last = pipe.drain()
    torch.cuda.synchronize()
    n = len(batches)
    assert torch.equal(last.histories, want[n - 1].histories)
    results.append(tuple(t.clone() for t in pipe.host_outputs[(n - 2) % 2]))
    results.append(tuple(t.clone() for t in pipe.host_outputs[(n - 1) % 2]))
    assert len(results) == n
    for (h, p), w in zip(results, want):
        assert torch.equal(h, w.histories.cpu()) and torch.equal(p, w.paths.cpu())
    # short runs: drain after one and after two batches
    for n_short in (1, 2):
        for k in range(n_short):
            for dst, src in zip(pipe.host_inputs[k % 3], batches[k]):
                dst.copy_(src.cpu())
            assert pipe.submit() is None
        last = pipe.drain()
        torch.cuda.synchronize()
        assert torch.equal(last.histories, want[n_short - 1].histories)
        for k in range(n_short):
            assert torch.equal(pipe.host_outputs[k % 2][1], want[k].paths.cpu())
    assert pipe.drain() is None
    # single-graph end-to-end replay
    fast = GraphedPlanner(na, maps, start, goal)
    for dst, src in zip(fast.host_inputs, batches[2]):
        dst.copy_(src.cpu())
    fast.replay_host()
    torch.cuda.synchronize()
    assert torch.equal(fast.host_outputs[0], want[2].histories.cpu())
    assert torch.equal(fast.host_outputs[1], want[2].paths.cpu())


def test_overlapped_planner_matches_direct_calls():
    """OverlappedPlanner: batches round-robin on several streams give exactly the direct call's outputs (engine 5 on
    136x144 binary maps, the warp engine on 32x32 learned costs)."""
    from neural_astar.planner import VanillaAstar
    from neural_astar.utils.inference import OverlappedPlanner

    rng = np.random.RandomState(7)
    va = VanillaAstar().cuda().eval()
    batches = []
    for k in range(6):
        H, W = (136, 144) if k % 2 == 0 else (40, 33)
        o = (rng.rand(5, 1, H, W) > 0.2).astype(np.float32)
        s = np.zeros_like(o); g = np.zeros_like(o)
        o[:, 0, 0, 0] = o[:, 0, -1, -1] = 1; s[:, 0, 0, 0] = 1; g[:, 0, -1, -1] = 1
        batches.append(tuple(_cu(x) for x in (o, s, g)))
    with torch.no_grad():
        want = [va(*b) for b in batches]
    over = OverlappedPlanner(va, n_streams=3, device="cuda")
    handles = [over.submit(*b) for b in batches]
    for h, w in zip(handles, want):
        out = h.result()
        assert torch.equal(out.histories, w.histories) and torch.equal(out.paths, w.paths)
    h = over.submit(*batches[0])
    over.wait_all()
    torch.cuda.synchronize()
    assert h.done() and torch.equal(h.result().paths, want[0].paths)
    na = _ckpt_planner()
    g_ = Golden("mazes032_vanilla_test")
    b = tuple(_cu(x) for x in (g_.obst, g_.start, g_.goal))
    with torch.no_grad():
        w = na(*b)
    outs = [OverlappedPlanner(na, n_streams=2).submit(*b).result() for _ in range(2)]
    assert all(torch.equal(o.histories, w.histories) for o in outs)


@pytest.mark.parametrize("host", [False, True])
def test_pipelined_planner_downsizing_encoder(host):
    """PipelinedPlanner on the WarCraft-shaped planner (rgb+ input packed by pack_inputs, CNNDownSize with pooling,
    learn_obstacles): same outputs as the eager call, late fork (hook before the last conv) and host staging."""
    from neural_astar.planner import NeuralAstar
    from neural_astar.utils.inference import PipelinedPlanner

    torch.manual_seed(5)
    na = NeuralAstar(encoder_input="rgb+", encoder_arch="CNNDownSize", encoder_depth=3, learn_obstacles=True,
                     const=10.0).cuda().eval()
    B = 16
    batches = []
    for k in range(4):
        maps = torch.rand(B, 3, 96, 96, device="cuda")
        s = torch.zeros(B, 1, 12, 12, device="cuda"); s[:, :, k, 0] = 1
        g = torch.zeros_like(s); g[:, :, 11, 11 - k] = 1
        batches.append((maps, s, g))
    with torch.no_grad():
        want = [na(*b) for b in batches]
    pipe = PipelinedPlanner(na, *batches[0], host=host, fork="late")
    got = []
    for k, b in enumerate(batches):
        if host:
            torch.cuda.synchronize()
            for dst, src in zip(pipe.host_inputs[k % 3], b):
                dst.copy_(src.cpu())
            out = pipe.submit()
        else:
            out = pipe.submit(*b)
        if out is not None:
            got.append((out.histories.clone(), out.paths.clone()))
    if host:                        # drain runs two steps: batch n-2, then batch n-1 (returned)
        last = pipe.drain()
        torch.cuda.synchronize()
        assert torch.equal(pipe.host_outputs[(len(batches) - 2) % 2][0], want[-2].histories.cpu())
        got.append((want[-2].histories, want[-2].paths))
    else:
        last = pipe.drain()
    got.append((last.histories.clone(), last.paths.clone()))
    assert len(got) == len(batches)
    for (h, p), w in zip(got, want):
        assert torch.equal(h, w.histories) and torch.equal(p, w.paths)


@pytest.mark.parametrize("hw", [32, 64])
def test_forward_pair_with_fused_handoff(hw):
    """NeuralAstar.forward_pair (validation pair with the TAPS prologue): learned half == NeuralAstar.forward, vanilla
    half == VanillaAstar, on the 32-wide engine (one launch) and the 64-wide engine (two halves back to back, the
    second one on the plain obstacle plane)."""
    from neural_astar.planner import NeuralAstar, VanillaAstar

    torch.manual_seed(hw)
    na = NeuralAstar(encoder_input="m+", encoder_arch="CNN", encoder_depth=4).cuda().eval()
    B = 5
    x = (torch.rand(B, 1, hw, hw, device="cuda") > 0.15).float()
    s = torch.zeros(B, 1, hw, hw, device="cuda"); s[:, :, 0, 0] = 1
    g = torch.zeros_like(s); g[:, :, -1, -1] = 1
    x[:, :, 0, 0] = 1; x[:, :, -1, -1] = 1
    with torch.no_grad():
        learned, vanilla, (ncl, plen) = na.forward_pair(x, s, g)
        want_l = na(x, s, g)
        want_v = VanillaAstar().cuda()(x, s, g)
    assert torch.equal(learned.histories, want_l.histories) and torch.equal(learned.paths, want_l.paths)
    assert torch.equal(vanilla.histories, want_v.histories) and torch.equal(vanilla.paths, want_v.paths)
    assert torch.equal(ncl[:B], want_l.histories.sum((1, 2, 3)).to(ncl.dtype))
    assert torch.equal(plen[B:], want_v.paths.sum((1, 2, 3)).to(plen.dtype))


def test_pipelined_planner_on_64_wide_grids():
    """PipelinedPlanner with the 64-wide engine's fused hand-off (48x48 and 64x64 planning grids)."""
    from neural_astar.planner import NeuralAstar
    from neural_astar.utils.inference import PipelinedPlanner

    for hw in (64, 48):
        torch.manual_seed(hw)
        na = NeuralAstar(encoder_input="m+", encoder_arch="CNN", encoder_depth=3).cuda().eval()
        batches = []
        for k in range(3):
            x = (torch.rand(6, 1, hw, hw, device="cuda") > 0.15).float()
            s = torch.zeros(6, 1, hw, hw, device="cuda"); s[:, :, k, 0] = 1
            g = torch.zeros_like(s); g[:, :, -1, -1 - k] = 1
            x[:, :, k, 0] = 1; x[:, :, -1, -1 - k] = 1
            batches.append((x, s, g))
        with torch.no_grad():
            want = [na(*b) for b in batches]
        pipe = PipelinedPlanner(na, *batches[0])
        got = [pipe.submit(*b) for b in batches]
        got = [(o.histories.clone(), o.paths.clone()) for o in got[1:]]
        last = pipe.drain()
        got.append((last.histories, last.paths))
        for (h, p), w in zip(got, want):
            assert torch.equal(h, w.histories) and torch.equal(p, w.paths)
