"""Persistent schedules and prologue / epilogue variants of the search engines and the encoder kernels, against the SPEC
oracle (oracle/astar_oracle.c) and fp64 references.

The other parity tests use batches smaller than a resident grid, so no persistent CTA there takes a second map and no
grid-stride loop takes a second round.  Here every batch is sized from the device's SM count to exceed the grid, so
the per-map resets, the engine-5 work queue, the redo pass and the grid-stride loops all run again on state a previous
map or round left behind.

Launch constants restated from the sources (each size below asserts that it exceeds the grid they give):
  * nastar_api.cu: kGlobalCtasPerSm = 8; generic_slots(B) = min(B, 8 x SMs) CTAs for engine 3's forward and every
    generic backward (engine 2's forward launches one CTA per map and does not loop);
  * nastar_bin16.cuh: kBin16Threads = 256 and __launch_bounds__(256, 1), so at most 2048 / 256 = 8 CTAs per SM;
  * nastar_api.cu launch_head: at most 16 CTAs per SM, nastar_glue.cuh kHeadWarps = 4 warps, one 32-pixel group per warp;
  * nastar_api.cu conv1_marks: at most 8 CTAs per SM, nastar_glue.cuh kConv1Warps = 8 warps of 32 pixels;
  * nastar_api.cu cost_from_taps / pack_inputs: at most 16 CTAs per SM of 256 threads, one pixel per thread.
"""
import numpy as np
import pytest
import torch

import encoder_exact_oracle as eo
from grad_bound import assert_within_bound
from test_gpu_convhead import _problem as _convhead_problem

pytestmark = pytest.mark.gpu
GENERIC_CTAS_PER_SM = 8
BIN16_CTAS_PER_SM = 2048 // 256
FOLLOWERS = ("short", "same", "unreachable", "capped")   # kinds of map that run second in a slot after a long search


@pytest.fixture(scope="module")
def native():
    from neural_astar import _native

    _native.lib()
    return _native


@pytest.fixture(scope="module")
def sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _dev(x):
    return torch.from_numpy(np.ascontiguousarray(x)).cuda()


def _problems(rng, kinds, H, W, p_obst=0.15):
    """One map per entry of `kinds`:
      long        start and goal in opposite corners;
      short       goal at most two cells from the start;
      same        start == goal;
      unreachable the start is walled in: the open set empties after one step (t_solve -2);
      capped      no obstacles but a walled-in goal: more reachable cells than T = W*W steps (t_solve -1)."""
    B = len(kinds)
    obst = (rng.rand(B, 1, H, W) > p_obst).astype(np.float32)
    start = np.zeros((B, 1, H, W), np.float32)
    goal = np.zeros((B, 1, H, W), np.float32)
    for b, kind in enumerate(kinds):
        sy, sx = rng.randint(H), rng.randint(W)
        if kind == "long":
            (sy, sx), (gy, gx) = (0, 0), (H - 1, W - 1)
        elif kind == "short":
            gy, gx = min(max(sy + rng.randint(-2, 3), 0), H - 1), min(max(sx + rng.randint(-2, 3), 0), W - 1)
        elif kind == "same":
            gy, gx = sy, sx
        elif kind == "unreachable":
            gy, gx = (sy + H // 2) % H, (sx + W // 2) % W
            obst[b, 0, max(sy - 1, 0):sy + 2, max(sx - 1, 0):sx + 2] = 0
        elif kind == "capped":
            (sy, sx), (gy, gx) = (0, 0), (H // 2, W // 2)
            obst[b] = 1
            obst[b, 0, gy - 1:gy + 2, gx - 1:gx + 2] = 0
        else:
            raise ValueError(kind)
        obst[b, 0, sy, sx] = obst[b, 0, gy, gx] = 1
        start[b, 0, sy, sx] = 1
        goal[b, 0, gy, gx] = 1
    return obst, start, goal


def _learned(rng, shape):
    return (1.0 / (1.0 + np.exp(-rng.randn(*shape)))).astype(np.float32)


def _forward_vs_oracle(native, oracle, planes, dev_planes, T, g_ratio=0.5, trace=True):
    """Forward on the device planes (cost, start, goal, obst) against the SPEC oracle on the host copies: every output
    and both per-map counts bit for bit.  Returns (t_solve, n_steps) on the device."""
    hist, paths, ts, ns, tr, (ncl, plen) = native.forward(*dev_planes, g_ratio, T, trace, want_counts=True)
    ref = oracle.forward(*planes, g_ratio=g_ratio, mode="spec", want_trace=trace, T=T)
    np.testing.assert_array_equal(ts.cpu().numpy(), ref.t_solve)
    np.testing.assert_array_equal(ns.cpu().numpy(), ref.n_steps)
    if trace:
        np.testing.assert_array_equal(tr.cpu().numpy(), ref.trace)
    np.testing.assert_array_equal(hist.cpu().numpy(), ref.histories)
    np.testing.assert_array_equal(paths.cpu().numpy(), ref.paths)
    np.testing.assert_array_equal(ncl.cpu().numpy(), ref.histories.sum((1, 2, 3)).astype(np.int64))
    np.testing.assert_array_equal(plen.cpu().numpy(), ref.paths.sum((1, 2, 3)))
    return ts, ns


def _backward_vs_oracle(native, oracle, planes, dev_planes, ts, ns, T, rng, g_ratio=0.5, T_batch=None):
    """Backward for the forward's T_batch, or for a given shorter T_batch: the oracle's replay costs B x T_batch x N,
    and one unsolved map would otherwise make T_batch = T for the whole batch."""
    cost, start, goal, obst = planes
    G = rng.randn(*cost.shape).astype(np.float32)
    if T_batch is None:
        Tb = native.batch_steps(ts, ns, T)
    else:
        Tb = torch.full((1,), T_batch, dtype=torch.int32, device="cuda")
    gc = native.backward(*dev_planes, _dev(G), Tb, ts, g_ratio).cpu().numpy()
    want, M = oracle.backward_with_bound(cost, start, goal, obst, G, int(Tb.item()), g_ratio=g_ratio)
    assert_within_bound(gc, want, M, (cost.shape, g_ratio, int(Tb.item())))


# ------------------------------------------------------------------------- engine 4 and generic prologue / epilogue
@pytest.mark.parametrize("H,W", [
    (48, 64),     # engine 4, W = 64: TMA prologue when every plane is 16-B aligned, 128-bit epilogue
    (50, 47),     # engine 4, W < 64: scalar prologue and epilogue
    (96, 64),     # engine 2, (W & 31) == 0: vectorised prologue and epilogue, TMA cost copy
    (96, 50),     # engine 2, W not a multiple of 32 (N % 4 == 0: TMA cost copy, scalar bit rows)
    (65, 41),     # engine 2, odd N: no TMA
    (160, 128),   # engine 3, (W & 31) == 0
])
@pytest.mark.parametrize("misaligned", [False, True])
def test_prologue_and_epilogue_variants_vs_oracle(native, oracle, H, W, misaligned):
    """Aligned planes take the TMA / 128-bit paths; the same planes one float past a 16-B boundary (views into a larger
    buffer) take the scalar ones.  Forward bit-exact with its trace, and for the generic engine the backward, whose
    engine-2 prologue refills the shared cost plane the same way."""
    rng = np.random.RandomState(H * 131 + W)
    B = 12
    kinds = [("long", "short", "long", "same")[b % 4] for b in range(B)]
    obst, start, goal = _problems(rng, kinds, H, W, p_obst=0.2)
    cost = _learned(rng, obst.shape) * np.float32(3.0)
    planes = (cost, start, goal, obst)
    dev = []
    for x in planes:
        if misaligned:
            buf = torch.zeros(x.size + 1, device="cuda")
            v = buf[1:1 + x.size].view(x.shape)
            v.copy_(torch.from_numpy(x))
            assert v.data_ptr() % 16 != 0
            dev.append(v)
        else:
            dev.append(_dev(x))
    ts, ns = _forward_vs_oracle(native, oracle, planes, dev, W * W)
    if native.lib().nastar_b200_engine_for(H, W) in (2, 3):
        _backward_vs_oracle(native, oracle, planes, dev, ts, ns, W * W, rng)


# ----------------------------------------------------------------------------------- generic engine: slot reuse
@pytest.mark.parametrize("H,W,engine", [(65, 40, 2), (144, 136, 3)])
def test_generic_slots_take_a_second_map(native, oracle, sms, H, W, engine):
    """B = 8 x SMs + 64 learned-cost maps: slot k runs map k, a long search, and then map k + slots, which is short,
    has start == goal, has an unreachable goal or is step-capped; every other map is short.  Forward with trace and
    counts bit-exact, backward (the per-map reset of V / ACC, and at 65x40 engine 2's TMA refill of the shared cost
    plane) within the oracle's bound."""
    assert native.lib().nastar_b200_engine_for(H, W) == engine
    slots = GENERIC_CTAS_PER_SM * sms
    B = slots + 64
    assert B > slots
    kinds = ["short"] * B
    for k in range(B - slots):
        kinds[k] = "long"
        kinds[k + slots] = FOLLOWERS[k % len(FOLLOWERS)]
    rng = np.random.RandomState(H + W)
    obst, start, goal = _problems(rng, kinds, H, W)
    planes = (_learned(rng, obst.shape), start, goal, obst)
    dev = [_dev(x) for x in planes]
    T = W * W
    ts, ns = _forward_vs_oracle(native, oracle, planes, dev, T)
    ts_h = ts.cpu().numpy()
    for kind, want in (("same", 0), ("unreachable", -2), ("capped", -1)):
        assert (ts_h[[b for b in range(slots, B) if kinds[b] == kind]] == want).all(), kind
    # 256 steps: the long maps run that long or finish, and the capped ones replay all of them
    _backward_vs_oracle(native, oracle, planes, dev, ts, ns, T, rng, T_batch=256)


def test_engine3_workspace_left_by_a_previous_call(native, oracle):
    """Two calls with the same (B, H, W) on engine 3: the caching allocator hands the second call the workspace block
    that holds the first call's g / f / parent planes and backward sums.  Both calls match the oracle."""
    H, W, B = 144, 136, 16
    assert native.lib().nastar_b200_engine_for(H, W) == 3
    rng = np.random.RandomState(31)
    for kinds in (["long"] * B, [FOLLOWERS[b % len(FOLLOWERS)] for b in range(B)]):
        obst, start, goal = _problems(rng, kinds, H, W)
        planes = (_learned(rng, obst.shape), start, goal, obst)
        dev = [_dev(x) for x in planes]
        ts, ns = _forward_vs_oracle(native, oracle, planes, dev, W * W)
        _backward_vs_oracle(native, oracle, planes, dev, ts, ns, W * W, rng, T_batch=1024)


# --------------------------------------------------------------------------------------------- engine 5: queue
@pytest.mark.parametrize("H,W", [(65, 40), (256, 256)])
def test_bin16_queue_and_redo_pass_beyond_the_grid(native, oracle, sms, H, W):
    """Binary aliased planes, B = 8 x SMs + 64: more maps than engine 5 can hold resident (at most 8 CTAs per SM; at
    256x256 Bin16Layout::smem_bytes = 16384 + 1024 + 1024 + 131072 + 65536 + 8192 + 64 = 223296 B allows one), so CTAs
    take further maps from the queue onto planes the previous map left.  Long and short maps are interleaved.  A few
    maps carry non-binary costs in the aliased plane and go to the redo pass; at 256x256 that pass runs on
    min(B, 8 x SMs) engine-3 slots, and maps k and k + slots are both redone by slot k."""
    L = native.lib()
    assert L.nastar_b200_bin16_supported(H, W) == 1
    slots = GENERIC_CTAS_PER_SM * sms
    B = slots + 64
    assert B > BIN16_CTAS_PER_SM * sms and B > slots
    kinds = ["long" if b % 8 == 3 else "short" for b in range(B)]
    redo = [5, 5 + slots, 40, 40 + slots, 61]
    for b in redo[::2]:
        kinds[b] = "long"
    rng = np.random.RandomState(H * W)
    obst, start, goal = _problems(rng, kinds, H, W, p_obst=0.2)
    obst[redo] *= (0.5 + rng.rand(len(redo), 1, H, W)).astype(np.float32)
    c = _dev(obst)
    before = native.launch_count()
    _forward_vs_oracle(native, oracle, (obst, start, goal, obst), (c, _dev(start), _dev(goal), c), W * W, trace=False)
    assert native.launch_count() - before == 2          # engine 5, then the generic engine's redo pass


# --------------------------------------------------------------------------------------- glue kernels: grid stride
@pytest.mark.parametrize("C", [32, 256])
def test_head_taps_beyond_the_grid(native, sms, C):
    """More 32-pixel groups than the capped grid has warps: each warp prefetches its next group's first slice while it
    finishes the current group.  P is not a multiple of 32 (ragged last group).  Bit-equal to the kernel's fp32
    operation sequence (eo.head_taps_replay) on 2 048 sampled pixels and the last 40."""
    cap = sms * 16 * 4 * 32
    H = W = 61
    B = cap // (H * W) + 2
    B += 1 - B % 2                                       # odd B: P = B * 3721 is odd
    P = B * H * W
    assert P > cap and P % 32
    torch.manual_seed(C)
    x = torch.randn(B, C, H, W, device="cuda").contiguous(memory_format=torch.channels_last)
    w = torch.randn(C, 9, device="cuda") / C ** 0.5
    got = native.head_taps(x, w.cpu().numpy()).view(P, 9)
    idx = torch.from_numpy(np.unique(np.concatenate([np.random.RandomState(C).randint(0, P, 2048),
                                                     np.arange(P - 40, P)]))).cuda()
    want = eo.head_taps_replay(x.permute(0, 2, 3, 1).reshape(P, C)[idx].cpu().numpy(), w.cpu().numpy())
    assert np.array_equal(got[idx].cpu().numpy(), want)


def test_conv1_marks_beyond_the_grid(native, sms):
    cap = sms * 8 * 8 * 32
    H, W = 37, 53
    B = cap // (H * W) + 2
    assert B * H * W > cap
    torch.manual_seed(1)
    maps = (torch.rand(B, 1, H, W, device="cuda") > 0.2).float()
    start = torch.zeros(B, 1, H, W, device="cuda")
    goal = torch.zeros_like(start)
    b = torch.arange(B, device="cuda")
    start[b, 0, b % H, (3 * b) % W] = 1
    goal[b, 0, H - 1 - b % H, (5 * b) % W] = 1
    w = torch.randn(32, 2, 3, 3, device="cuda") * 0.3
    bias = torch.randn(32, device="cuda") * 0.1
    wh = np.ascontiguousarray(w.permute(2, 3, 1, 0).reshape(9, 2, 32).cpu().numpy())
    got = native.conv1_marks(maps, start, goal, wh, bias.cpu().numpy()).permute(0, 2, 3, 1).reshape(-1, 32)
    # bit-equal to the kernel's fp32 operation sequence (eo.conv1_marks_replay) on 2 048 sampled pixels and the last 40
    idx = np.unique(np.concatenate([np.random.RandomState(1).randint(0, B * H * W, 2048),
                                    np.arange(B * H * W - 40, B * H * W)]))
    want = eo.conv1_marks_replay(maps.cpu().numpy(), start.cpu().numpy(), goal.cpu().numpy(), wh, bias.cpu().numpy(),
                                 pix=idx)
    assert np.array_equal(got[torch.from_numpy(idx).cuda()].cpu().numpy(), want)


def test_cost_from_taps_beyond_the_grid(native, sms):
    """Bit-exact against the same fp32 operation sequence in PyTorch: bias plus the 9 taps in ascending k with zero
    padding, then torch.sigmoid(x) * scale (bit-equal to the kernel's sigmoid, test_sigmoid_prologue_is_bit_exact)."""
    cap = sms * 16 * 256
    H, W = 37, 53
    B = cap // (H * W) + 2
    assert B * H * W > cap
    torch.manual_seed(2)
    taps = torch.randn(B, H, W, 9, device="cuda")
    bias, scale = 0.3, 10.0
    padded = torch.nn.functional.pad(taps, (0, 0, 1, 1, 1, 1))
    acc = torch.full((B, H, W), bias, device="cuda")
    for k in range(9):
        acc = acc + padded[:, k // 3:k // 3 + H, k % 3:k % 3 + W, k]
    want = (torch.sigmoid(acc) * scale)[:, None]
    got = native.cost_from_taps(taps, bias, scale)
    assert torch.equal(got, want)


@pytest.mark.parametrize("C", [1, 3])
def test_pack_inputs_beyond_the_grid(native, sms, C):
    cap = sms * 16 * 256
    Hm, Wm, H, W = 74, 106, 37, 53
    B = cap // (Hm * Wm) + 2
    assert B * Hm * Wm > cap
    torch.manual_seed(C)
    maps = torch.rand(B, C, Hm, Wm, device="cuda")
    start = torch.zeros(B, 1, H, W, device="cuda")
    goal = torch.zeros_like(start)
    b = torch.arange(B, device="cuda")
    start[b, 0, b % H, (3 * b) % W] = 1
    goal[b, 0, H - 1 - b % H, W - 1] = 1
    marks = torch.nn.functional.interpolate(start + goal, size=(Hm, Wm), mode="nearest")
    want = torch.cat((maps, marks), dim=1)
    assert torch.equal(native.pack_inputs(maps, start, goal), want)


# ------------------------------------------------------------------------------ fused conv + head: tile schedule
@pytest.mark.parametrize("Wp,ragged", [(8, (17, 5)), (16, (9, 12)), (32, (5, 27)), (64, (3, 50))])
def test_fused_taps_tile_schedule_sweep(native, Wp, ragged):
    """conv3x3_head_taps over every tile count of the cluster schedule (ch_tile): full rounds, a half-tile tail, and a
    tail of more than half a round that runs as a full extra round.  (128 / Wp, Wp) maps are one tile each, so tiles
    = B, and B = 1..400 gives three rounds for any cluster count up to 66.  The ragged shape (R + 1 rows, W < Wp) has
    two tiles per map, the second with one valid row, so half tiles and partial columns land past the map's edge.
    Each result is within the fp32-accumulation bound of the fp64 taps of its TF32 operands (eo.tf32_taps_and_bound),
    every pixel is written and nothing after the output is."""
    R = 128 // Wp
    assert ragged[0] == R + 1 and Wp // 2 < ragged[1] < Wp
    for (H, W), Bmax in (((R, Wp), 400), (ragged, 200)):
        x, w, b, hw = _convhead_problem(Bmax, H, W, seed=Wp * 1000 + W)
        want, bound = eo.tf32_taps_and_bound(x, w, b, hw)
        n = H * W * 9
        buf = torch.empty(Bmax * n + 64, device="cuda")
        ok = []
        for B in range(1, Bmax + 1):
            buf.fill_(float("nan"))
            out = buf[:B * n].view(B, H, W, 9)
            native.conv3x3_head_taps(x[:B], w, b, hw, out=out)
            within = ((out.double() - want[:B]).abs() <= bound[:B]).all()   # NaN (not written) compares False
            ok.append(within & torch.isnan(buf[B * n:]).all())
        bad = [B for B, v in zip(range(1, Bmax + 1), torch.stack(ok).tolist()) if not v]
        assert not bad, f"{H}x{W}: wrong or missing taps, or writes past the output, at B = {bad}"


# ------------------------------------------------------------------ batch-coupled path (g_ratio < 0.5) on 4, 2, 3
@pytest.mark.parametrize("H,W,B", [(48, 40, 8), (64, 64, 6), (100, 72, 4), (144, 136, 3)])
@pytest.mark.parametrize("g_ratio", [0.0, 0.3])
@pytest.mark.parametrize("train", [False, True])
def test_coupled_low_g_ratio_module_vs_oracle(oracle, H, W, B, g_ratio, train):
    """DifferentiableAstar with g_ratio < 0.5 and B > 1 steps every map until all of them select their goal in the same
    step.  Restated here from the SPEC oracle's no-exit trace: T_batch = the first step at which every map selects its
    goal (T if there is none), and a goal is clamped when its map selects it at least twice within T_batch steps.
    Frame count, masks and per-frame selections must equal the oracle run for exactly T_batch steps, and cost.grad its
    closed form within its bound."""
    from neural_astar.planner.differentiable_astar import DifferentiableAstar

    rng = np.random.RandomState(H * W + int(g_ratio * 10) + 7 * train)
    obst = (rng.rand(B, 1, H, W) > 0.15).astype(np.float32)
    start = np.zeros_like(obst)
    goal = np.zeros_like(obst)
    for b in range(B):
        sy, sx = rng.randint(H // 4), rng.randint(W // 4)
        gy, gx = H - 1 - rng.randint(H // 4), W - 1 - rng.randint(W // 4)
        obst[b, 0, sy, sx] = obst[b, 0, gy, gx] = 1
        start[b, 0, sy, sx] = 1
        goal[b, 0, gy, gx] = 1
    cost = _learned(rng, obst.shape) * np.float32(10.0)
    G = rng.randn(B, 1, H, W).astype(np.float32)
    T = int((0.25 if train else 1.0) * W * W)

    full = oracle.forward(cost, start, goal, obst, g_ratio=g_ratio, mode="spec", want_trace=True, T=T,
                          no_early_exit=True)
    gidx = goal.reshape(B, -1).argmax(1)
    at_goal = full.trace == gidx[:, None]
    every = at_goal.all(0)
    T_batch = int(every.argmax()) + 1 if every.any() else T
    clamped = at_goal[:, :T_batch].sum(1) >= 2
    if not train:   # these seeds reach both sides of the clamp (in training the capped loop often solves no map)
        assert clamped.any() and not clamped.all(), clamped
    ref = oracle.forward(cost, start, goal, obst, g_ratio=g_ratio, mode="spec", want_trace=True, T=T_batch,
                         no_early_exit=True)

    astar = DifferentiableAstar(g_ratio=g_ratio, Tmax=0.25).cuda().train(train)
    c = _dev(cost).requires_grad_(True)
    out = astar(c, _dev(start), _dev(goal), _dev(obst), store_intermediate_results=True)
    assert len(out.intermediate_results) == T_batch + 1
    np.testing.assert_array_equal(out.histories.detach().cpu().numpy(), ref.histories)
    np.testing.assert_array_equal(out.paths.cpu().numpy(), ref.paths)
    sel = torch.stack([f["paths"].reshape(B, -1).argmax(1) for f in out.intermediate_results[:-1]], 1)
    np.testing.assert_array_equal(sel.cpu().numpy(), np.where(ref.trace < 0, gidx[:, None], ref.trace))
    (out.histories * _dev(G)).sum().backward()
    want, M = oracle.backward_with_bound(cost, start, goal, obst, G, T_batch, g_ratio=g_ratio)
    assert_within_bound(c.grad.cpu().numpy(), want, M, (T_batch, clamped.tolist()))
