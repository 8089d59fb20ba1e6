"""The Unet encoder on the H100: the upsample-concat and 16-channel head kernels, the fused forward into the search,
graph replay, the pipeline, the validation pair and graphed training."""
from types import SimpleNamespace

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from golden_util import Golden

pytestmark = pytest.mark.gpu

DEC = [256, 128, 64, 32, 16]
STAGE_OUT = [64, 128, 256, 512, 512, 512]


def _decoder_shapes(d, side):
    """(h, Cd, Cs) of every decoder block of depth d on side x side inputs."""
    head = STAGE_OUT[d]
    ins = [head] + DEC[:d - 1]
    skips = [STAGE_OUT[k] for k in range(d - 1, 0, -1)] + [0]
    return [(side >> (d - i), ci, cs) for i, (ci, cs) in enumerate(zip(ins, skips))]


def _grid_cap_items():
    # the launcher caps the grid at 16 CTAs of 256 threads per SM: beyond this many float4 items the loop turns again
    return torch.cuda.get_device_properties(0).multi_processor_count * 16 * 256


@pytest.mark.parametrize("side", [32, 64])
@pytest.mark.parametrize("d", [1, 2, 3, 4, 5])
def test_upsample_concat_bit_equal(d, side):
    from neural_astar import _native

    g = torch.Generator(device="cuda").manual_seed(d * 100 + side)
    for h, cd, cs in _decoder_shapes(d, side):
        per_map = h * h * cd // 4 + 4 * h * h * cs // 4
        B = 2 * _grid_cap_items() // per_map + 1           # at least two turns of the grid-stride loop
        dec = torch.randn(B, cd, h, h, device="cuda", generator=g).contiguous(memory_format=torch.channels_last)
        skip = None
        if cs:
            skip = torch.randn(B, cs, 2 * h, 2 * h, device="cuda", generator=g)
            skip = skip.contiguous(memory_format=torch.channels_last)
        got = _native.upsample_concat(dec, skip)
        ref = F.interpolate(dec, scale_factor=2, mode="nearest")
        if skip is not None:
            ref = torch.cat((ref, skip), 1)
        assert got.is_contiguous(memory_format=torch.channels_last)
        assert torch.equal(got, ref), (d, side, h, cd, cs)


def test_head_taps_16_channels():
    from neural_astar import _native

    torch.manual_seed(0)
    B, H, W = 37, 31, 33                                    # P = 37851: a ragged last 32-pixel group of 27
    x = torch.randn(B, 16, H, W, device="cuda").contiguous(memory_format=torch.channels_last)
    w = np.random.RandomState(0).randn(16, 9).astype(np.float32)
    taps = _native.head_taps(x, w)
    ref = x.permute(0, 2, 3, 1).double().reshape(-1, 16) @ torch.from_numpy(w).double().cuda()
    torch.testing.assert_close(taps.double().reshape(-1, 9), ref, atol=1e-5, rtol=1e-5)


def _inputs(n=100):
    g = Golden("mazes032_vanilla_test")
    return [torch.from_numpy(a[:n]).cuda() for a in (g.obst, g.start, g.goal)]


def _calibrate(planner, maps, starts, goals):
    """Seeded weights with BatchNorm statistics from one batch, so that the logits are O(1) rather than saturated."""
    x = planner._encoder_input(maps, starts, goals)
    bns = [m for m in planner.encoder.modules() if isinstance(m, torch.nn.BatchNorm2d)]
    for m in bns:
        m.momentum = None
    planner.train()
    with torch.no_grad():
        planner.encoder.model(x)
    for m in bns:
        m.momentum = 0.1
    planner.eval()


def _planner(d, inp, mech="moore", seed=0):
    from neural_astar.planner import NeuralAstar

    torch.manual_seed(seed)
    p = NeuralAstar(encoder_arch="Unet", encoder_depth=d, encoder_input=inp, mechanism=mech).cuda()
    _calibrate(p, *_inputs())
    return p


@pytest.mark.parametrize("mech", ["moore", "news"])
@pytest.mark.parametrize("inp", ["m", "m+"])
@pytest.mark.parametrize("d", [4, 5])
def test_fused_forward_matches_encode_then_search(d, inp, mech):
    from neural_astar import _native

    maps, starts, goals = _inputs()
    p = _planner(d, inp, mech)
    with torch.no_grad():
        before = _native.launch_count()
        out = p(maps, starts, goals)
        torch.cuda.synchronize()
        assert _native.launch_count() - before >= d + 2     # upsample-concat per block, head, search
        cost = p.encode(maps, starts, goals)
        ref = p.perform_astar(cost, starts, goals, maps)
    assert torch.equal(out.histories, ref.histories)
    assert torch.equal(out.paths, ref.paths)
    assert 0.05 < float(cost.mean()) < 0.95, "logits saturated: the comparison would be vacuous"


ENCODE_CASES = [(d, inp, head) for head in ("kernel", "mm") for d in (4, 5) for inp in ("m", "m+")]


@pytest.mark.parametrize("d,inp,head", ENCODE_CASES,
                         ids=[f"{d}-{inp}" + ("" if head == "kernel" else "-mm") for d, inp, head in ENCODE_CASES])
def test_encode_matches_eager_module(d, inp, head, monkeypatch):
    """encode() against the eager module, with the head's products from the head kernel or, with
    NASTAR_B200_HEAD_KERNEL=0, from torch.mm."""
    from neural_astar import _native
    from neural_astar.planner import encoder

    maps, starts, goals = _inputs()
    p = _planner(d, inp)
    monkeypatch.setattr(encoder, "HEAD_KERNEL", head == "kernel")
    if head == "mm":
        monkeypatch.setattr(_native, "head_taps", lambda *a, **k: pytest.fail("head kernel ran with HEAD_KERNEL off"))
    x = p._encoder_input(maps, starts, goals)
    old = torch.backends.cudnn.allow_tf32
    try:
        torch.backends.cudnn.allow_tf32 = False
        with torch.no_grad():
            eager = torch.sigmoid(p.encoder.model(x.contiguous())) * p.encoder.const
            monkeypatch.setattr(encoder, "ALLOW_TF32", False)
            fp32 = p.encode(maps, starts, goals)
            monkeypatch.setattr(encoder, "ALLOW_TF32", True)
            tf32 = p.encode(maps, starts, goals)
    finally:
        torch.backends.cudnn.allow_tf32 = old
    # 21 convolutions deep, with BatchNorm folded on one side and not on the other and different cuDNN algorithms:
    # fp32 re-association alone moved the costs by 2.4e-5 .. 3.8e-5 on an H100 80GB HBM3 (700 W)
    torch.testing.assert_close(fp32, eager, atol=1e-4, rtol=0)
    diff = float((tf32 - eager).abs().max())
    print(f"\nUnet d={d} {inp} {head}: max |encode() - eager| = {float((fp32 - eager).abs().max()):.3g} (fp32), "
          f"{diff:.3g} (TF32)")
    assert diff < 5e-2


def test_bad_sides_on_the_fast_path():
    p = _planner(4, "m+")
    maps = torch.ones(2, 1, 24, 32, device="cuda")
    marks = torch.zeros_like(maps)
    with torch.no_grad(), pytest.raises(ValueError, match="divisible by 2\\*\\*4"):
        p(maps, marks, marks)


def test_graphs_pipeline_and_pair():
    from neural_astar.utils.inference import GraphedPlanner, PipelinedPlanner

    maps, starts, goals = _inputs()
    p = _planner(4, "m+")
    with torch.no_grad():
        ref = p(maps, starts, goals)
        ref2 = p(maps.flip(-1).contiguous(), starts.flip(-1).contiguous(), goals.flip(-1).contiguous())
        pair = p.forward_pair(maps, starts, goals)
    assert pair is not None
    assert torch.equal(pair[0].histories, ref.histories) and torch.equal(pair[0].paths, ref.paths)

    graphed = GraphedPlanner(p, maps, starts, goals)
    out = graphed.replay()
    assert torch.equal(out.histories, ref.histories) and torch.equal(out.paths, ref.paths)
    assert graphed.native_launches_per_replay >= 4 + 2

    pipe = PipelinedPlanner(p, maps, starts, goals)
    assert pipe.submit(maps, starts, goals) is None
    first = pipe.submit(maps.flip(-1).contiguous(), starts.flip(-1).contiguous(), goals.flip(-1).contiguous())
    h1, p1 = first.histories.clone(), first.paths.clone()
    second = pipe.drain()
    assert torch.equal(h1, ref.histories) and torch.equal(p1, ref.paths)
    assert torch.equal(second.histories, ref2.histories) and torch.equal(second.paths, ref2.paths)


def test_graphed_train_step_matches_eager():
    from neural_astar.planner import NeuralAstar
    from neural_astar.utils.training import GraphedTrainStep, PlannerModule

    g = Golden("mazes032_neural_test")
    batch = [torch.from_numpy(a).cuda() for a in (g.obst, g.start, g.goal, g.bits("opt_bits").astype(np.float32))]

    def make():
        torch.manual_seed(1234)
        planner = NeuralAstar(encoder_input="m+", encoder_arch="Unet", encoder_depth=4, Tmax=0.25)
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
    assert step_fn.replays == 3
    np.testing.assert_allclose(graph_losses, eager_losses, rtol=2e-3)
    pe = float(sum(p.detach().abs().sum() for p in eager.planner.parameters()))
    pg = float(sum(p.detach().abs().sum() for p in graphed.planner.parameters()))
    assert pg == pytest.approx(pe, rel=1e-3)
