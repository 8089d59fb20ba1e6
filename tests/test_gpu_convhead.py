"""The fused last-conv + head kernel (csrc/nastar_convhead.cuh): TF32 128 -> 256 3x3 convolution, bias, ReLU and the
head's 9 per-pixel products in one launch.  Checked against fp64 taps of its TF32 operands within a bound on fp32
accumulation alone, against the cuDNN TF32 conv + head_taps path it replaces, for determinism, and for staying out of
the fp32 path.  tests/test_gpu_encoder_exact.py checks it bit for bit."""
import os

import numpy as np
import pytest
import torch

import encoder_exact_oracle as eo
from golden_util import Golden

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
# TF32 keeps 10 explicit mantissa bits: reading an fp32 operand as TF32 changes it by less than 2^-10 relatively, so
# each product x*w is off by less than 2^-9 |x||w|.  The fused kernel's tensor cores truncate (observed on an H100 SXM,
# test_gpu_encoder_exact.py::test_tf32_operand_conversion_mode); cuDNN's conversion is not assumed, so this bound, used
# for cuDNN and the encoder references, covers rounding as well.
U_TF32 = 2.0 ** -10
PROD = 2 * U_TF32 + U_TF32 ** 2


@pytest.fixture(scope="module")
def native():
    from neural_astar import _native

    _native.lib()
    return _native


def _ckpt_planner():
    from neural_astar.planner import NeuralAstar

    state = np.load(os.path.join(ROOT, "tests", "golden", "mazes032_ckpt_planner_state.npz"))
    na = NeuralAstar(encoder_arch="CNN")
    na.load_state_dict({k: torch.from_numpy(state[k]) for k in state.files})
    return na.cuda().eval()


def _problem(B, H, W, seed):
    g = torch.Generator(device="cpu").manual_seed(seed)
    x = torch.rand(B, 128, H, W, generator=g) * (torch.rand(B, 128, H, W, generator=g) > 0.4)   # ReLU-like input
    w = torch.randn(256, 128, 3, 3, generator=g) * 0.03 + 0.01
    b = torch.randn(256, generator=g) * 0.1
    hw = (torch.randn(256, 9, generator=g) * 0.05 + 0.05).numpy().astype(np.float32)
    return (x.cuda().contiguous(memory_format=torch.channels_last), w.cuda().contiguous(memory_format=torch.channels_last),
            b.cuda(), hw)


def _fp64_taps_and_bound(x, w, b, hw):
    """taps = relu(conv(x, w) + b) . hw in fp64, and a per-output bound on the error of a TF32-operand / fp32-accumulate
    evaluation: the pre-activation error is at most PROD * sum|x||w| plus fp32 accumulation (K = 1152 terms) and the
    bias add; ReLU does not enlarge it; the fp32 head sum over 256 channels adds at most 2^-15 sum|a||hw|."""
    xd, wd, bd = x.double(), w.double(), b.double()
    hwd = torch.from_numpy(hw).double().cuda()
    a = torch.relu(torch.nn.functional.conv2d(xd, wd, bd, padding=1))
    s = torch.nn.functional.conv2d(xd.abs(), wd.abs(), None, padding=1) + bd.abs().view(1, -1, 1, 1)
    taps = torch.einsum("bchw,ck->bhwk", a, hwd)
    pre_err = (PROD + 1152 * 2.0 ** -24) * s
    bound = torch.einsum("bchw,ck->bhwk", pre_err, hwd.abs()) + 2.0 ** -15 * torch.einsum("bchw,ck->bhwk", a, hwd.abs())
    return taps, bound + 1e-12


@pytest.mark.parametrize("B,H,W", [(1, 32, 32), (7, 32, 32), (100, 32, 32), (3, 64, 64), (5, 20, 27), (4, 5, 3),
                                   (100, 64, 64), (1000, 32, 32)])   # production batches: 3200 and 8000 tiles
def test_fused_taps_within_tf32_bound_of_fp64(native, B, H, W):
    """Against fp64 taps of the TF32 operands the tensor cores read (eo.tf32_taps_and_bound): the bound covers only
    the fp32 accumulation, the bias add and the head sum, and is at least 10x tighter than the a-priori bound of
    _fp64_taps_and_bound, which also has to cover the operand conversion."""
    x, w, b, hw = _problem(B, H, W, seed=B * 1000 + H * 10 + W)
    got = native.conv3x3_head_taps(x, w, b, hw)
    torch.cuda.synchronize()
    want, bound = eo.tf32_taps_and_bound(x, w, b, hw)
    err = (got.double() - want).abs()
    assert got.shape == (B, H, W, 9)
    assert bool(torch.isfinite(got).all())
    worst = float((err / bound).max())
    tighter = float((bound / _fp64_taps_and_bound(x, w, b, hw)[1]).max())
    print(f"B={B} {H}x{W}: max error / TF32-emulated bound = {worst:.4f}; bound / a-priori TF32 bound <= {tighter:.4f}")
    assert worst <= 1.0, f"error exceeds the TF32-emulated bound by {worst:.3f}x"
    assert tighter <= 0.1
    # the bound is not vacuous: it is a small fraction of the outputs it bounds
    assert float(bound.median()) < 0.002 * float(want.abs().median())


def test_fused_taps_leave_the_rest_of_out_untouched(native):
    """Every pixel of the map is written exactly once; nothing outside [B,H,W,9] is touched."""
    x, w, b, hw = _problem(3, 20, 27, seed=5)
    buf = torch.full((3 * 20 * 27 * 9 + 64,), float("nan"), device="cuda")
    out = buf[:3 * 20 * 27 * 9].view(3, 20, 27, 9)
    native.conv3x3_head_taps(x, w, b, hw, out=out)
    torch.cuda.synchronize()
    assert bool(torch.isfinite(out).all())
    assert bool(torch.isnan(buf[3 * 20 * 27 * 9:]).all())


def test_fused_taps_are_deterministic(native):
    x, w, b, hw = _problem(100, 32, 32, seed=11)
    t1 = native.conv3x3_head_taps(x, w, b, hw)
    t2 = native.conv3x3_head_taps(x, w, b, hw)
    assert torch.equal(t1, t2)


def _flagship_inputs():
    g = Golden("mazes032_vanilla_test")
    return tuple(torch.from_numpy(np.ascontiguousarray(v)).cuda() for v in (g.obst, g.start, g.goal))


def _conv3_output(na, maps, start, goal):
    from neural_astar import _native
    from neural_astar.planner import encoder as enc

    plan = na.encoder._inference_plan(maps.device)
    with enc._conv_flags():
        x = enc._run_layers(plan.body[1:], _native.conv1_marks(maps, start, goal, *plan.conv1))
    return plan, x.contiguous(memory_format=torch.channels_last)


def test_fused_taps_match_cudnn_tf32_last_conv_and_head(native):
    """Flagship batch (100 maps of 32x32, shipped checkpoint): the fused taps against cuDNN's TF32 conv4 followed by
    head_taps.  Both carry TF32 operand error, so they may differ by up to twice the bound; the cost maps stay within
    the 3e-3 the module's own path tolerance allows."""
    from neural_astar.planner import encoder as enc

    assert enc.ALLOW_TF32
    na = _ckpt_planner()
    maps, start, goal = _flagship_inputs()
    with torch.no_grad():
        plan, x3 = _conv3_output(na, maps, start, goal)
        w, b = plan.last.w, plan.last.b
        fused = native.conv3x3_head_taps(x3, w, b, plan.head_w)
        with torch.backends.cudnn.flags(enabled=True, allow_tf32=True):
            a4 = torch.cudnn_convolution_relu(x3, *plan.last[:5], 1).contiguous(memory_format=torch.channels_last)
        old = native.head_taps(a4, plan.head_w)
        _, bound = _fp64_taps_and_bound(x3, w, b, plan.head_w)
        bias, scale = plan.head_b, plan.const
        c_new = native.cost_from_taps(fused, bias, scale)
        c_old = native.cost_from_taps(old, bias, scale)
    diff = (fused.double() - old.double()).abs()
    print("fused vs cuDNN TF32 taps: max |diff| %.3g, max diff/bound %.3f, max cost diff %.3g"
          % (float(diff.max()), float((diff / bound).max()), float((c_new - c_old).abs().max())))
    assert float((diff / (2 * bound)).max()) <= 1.0
    assert float((c_new - c_old).abs().max()) < 3e-3


def test_head_step_selects_fused_kernel_only_with_tf32(native, monkeypatch):
    """With TF32 allowed the encoder runs the fused kernel in place of cuDNN conv4 + head_taps; with ALLOW_TF32 off the
    taps are bit-identical to cuDNN fp32 conv4 followed by head_taps (the fused kernel is not selected)."""
    from neural_astar.planner import encoder as enc

    na = _ckpt_planner()
    maps, start, goal = _flagship_inputs()
    calls = []
    real = native.conv3x3_head_taps
    monkeypatch.setattr(native, "conv3x3_head_taps", lambda *a, **k: calls.append(1) or real(*a, **k))
    monkeypatch.setattr(torch.backends.cudnn, "deterministic", True)    # one cuDNN algorithm for both fp32 evaluations
    with torch.no_grad():
        t_tf32 = na.encoder.head_taps_marks(maps, start, goal)[0]
        assert len(calls) == 1
        monkeypatch.setattr(enc, "ALLOW_TF32", False)
        t_fp32 = na.encoder.head_taps_marks(maps, start, goal)[0].clone()
        assert len(calls) == 1
        plan, x3 = _conv3_output(na, maps, start, goal)
        with enc._conv_flags():
            a4 = torch.cudnn_convolution_relu(x3, *plan.last[:5], 1).contiguous(memory_format=torch.channels_last)
        want = native.head_taps(a4, plan.head_w)
    assert torch.equal(t_fp32, want)
    assert not torch.equal(t_tf32, t_fp32)
