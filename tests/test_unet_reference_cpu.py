"""Pin NeuralAstar's U-Net encoder to the reference's own NeuralAstar run in float64, stage by stage.

The staged reference builds its U-Net through `segmentation_models_pytorch.Unet`, which is not installed: while it is
built, `StandInUnet` takes that name.  The stand-in is smp 0.3.1's vgg16_bn U-Net in float64 with smp's module names
(tests/test_unet_cpu.py `expected_layout`) and smp's forward; it asserts the exact arguments the reference passes, and
equals a real smp where one is importable.  Each configuration's reference has seeded weights (95 % of every conv's
positive, as tests/test_encoder_reference_cpu.py `build_reference` draws them) and BatchNorm statistics set by
`randomise_one_batchnorm` during one float64 calibration forward.

An end-to-end bound says nothing for a network 26 convolutions deep, so `stage_ratios` checks the product one stage at a
time: every stage is evaluated in float64 on the product's own recorded outputs of the stages that feed it in the
reference's graph, and held to a bound on that stage's own rounding only (see `stage_ratios`).  A miswired skip, a wrong
fold, a dropped bias or a wrong kernel index misses its stage's bound by orders of magnitude.  Checked here, without a
GPU:
  state dicts   both directions load with every key matched and every value kept;
  stand-in      the reference's encode() is the stand-in's forward on the reference's encoder input, which equals
                tests/test_unet_cpu.py `functional_unet` wherever that runs (sides divisible by 32);
  module path   the product's encode() in fp32 on the CPU (nn.Module path), recorded through forward hooks, meets every
                stage's fp32 bound; no conv stage's median bound exceeds 1 % of its median |pre-activation| in fp32, or
                5 % with TF32 operands.

tests/test_gpu_unet_reference.py records the eval fast path on the GPU (pack_inputs, the folded cuDNN plan, max pools,
upsample_concat, head_taps or torch.mm, cost_from_taps) and holds it to the same stage bounds.
"""
from __future__ import annotations

import zlib
from typing import List, NamedTuple, Optional, Tuple

import numpy as np
import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

import test_encoder_reference_cpu as er
from test_encoder_reference_cpu import FOLD, POSITIVE, SIGMOID, _f32, gamma
from test_gpu_convhead import PROD, U_TF32
from test_unet_cpu import CFG, DEC, STAGE_OUT, expected_layout, functional_unet

HEAD_STD = 1.0          # std of the head's logits on the calibration batch: costs far from both saturation and const / 2
VACUOUS_FP32 = 0.01     # largest median conv-stage bound / median |pre-activation| allowed in fp32 ...
VACUOUS_TF32 = 0.05     # ... and with TF32 operands


# ------------------------------------------------------------------------------------------------- the stand-in
def _cbr(cin: int, cout: int, bias: bool = False) -> nn.Sequential:
    return nn.Sequential(nn.Conv2d(cin, cout, 3, padding=1, bias=bias), nn.BatchNorm2d(cout), nn.ReLU(inplace=True))


class StandInUnet(nn.Module):
    """smp 0.3.1's `Unet(encoder_name="vgg16_bn", encoder_weights=None, classes=1, encoder_depth=depth)`: torchvision's
    vgg16_bn features as the encoder (biased convs), a two-block center (vgg encoders get one in smp), one decoder
    block per depth level (nearest x2 upsample, concat of the skip, two bias-less conv + BatchNorm + ReLU), a 3x3
    segmentation head.  PyTorch's default initialisation."""

    def __init__(self, in_channels: int, depth: int):
        super().__init__()
        self.depth = depth
        features, cin = [], in_channels
        for v in CFG:
            if v == "M":
                features.append(nn.MaxPool2d(kernel_size=2, stride=2))
            else:
                features += list(_cbr(cin, v, bias=True))
                cin = v
        self.encoder = nn.Module()
        self.encoder.features = nn.Sequential(*features)
        head = STAGE_OUT[depth]
        self.decoder = nn.Module()
        self.decoder.center = nn.Sequential(_cbr(head, head), _cbr(head, head))
        ins = [head] + DEC[:depth - 1]
        skips = [STAGE_OUT[k] for k in range(depth - 1, 0, -1)] + [0]
        self.decoder.blocks = nn.ModuleList()
        for ci, cs, co in zip(ins, skips, DEC[:depth]):
            block = nn.Module()
            block.conv1, block.conv2 = _cbr(ci + cs, co), _cbr(co, co)
            self.decoder.blocks.append(block)
        self.segmentation_head = nn.Sequential(nn.Conv2d(DEC[depth - 1], 1, kernel_size=3, padding=1))

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        # smp's VGGEncoder: the feature stack split before every max pool; stages 0..depth
        stages, cur = [], []
        for m in self.encoder.features:
            if isinstance(m, nn.MaxPool2d):
                stages.append(cur)
                cur = []
            cur.append(m)
        stages.append(cur)
        feats = []
        for stage in stages[:self.depth + 1]:
            for m in stage:
                x = m(x)
            feats.append(x)
        # smp's UnetDecoder: the full-resolution stage 0 is dropped, the deepest stage enters the center
        feats = feats[1:][::-1]
        x = self.decoder.center(feats[0])
        for i, block in enumerate(self.decoder.blocks):
            x = F.interpolate(x, scale_factor=2, mode="nearest")
            if i < len(feats) - 1:
                x = torch.cat([x, feats[i + 1]], dim=1)
            x = block.conv2(block.conv1(x))
        return self.segmentation_head(x)


def stand_in_unet(*args, **kw) -> StandInUnet:
    """What the reference's `smp.Unet(...)` call builds here; asserts the call is the one the reference makes."""
    d = kw.get("encoder_depth")
    assert not args and kw == dict(encoder_name="vgg16_bn", encoder_weights=None, classes=1,
                                   in_channels=kw.get("in_channels"), encoder_depth=d, decoder_channels=DEC[:d]), kw
    return StandInUnet(kw["in_channels"], d)


# ------------------------------------------------------------------------------------------------- the configurations
class UConfig(NamedTuple):
    inp: str                   # encoder_input: "m", "m+" or "rgb+"
    depth: int                 # encoder_depth
    grid: Tuple[int, int]      # H, W of the maps, the marks and the cost maps
    const: Optional[float] = None
    learn_obstacles: bool = False

    @property
    def id(self):
        extra = ("" if self.const is None else f"-c{self.const:g}") + ("-lo" if self.learn_obstacles else "")
        return f"Unet-{self.inp}-d{self.depth}-{self.grid[0]}x{self.grid[1]}{extra}"

    @property
    def seed(self):
        return zlib.crc32(self.id.encode())

    @property
    def B(self):
        """2 to 6 maps"""
        return 2 + self.seed % 5

    @property
    def image(self):
        return self.grid

    @property
    def head_channels(self):
        return DEC[self.depth - 1]


GRIDS = ((32, 32), (64, 64), (32, 96), (96, 32))
CONFIGS = ([UConfig(inp, d, hw) for d in (1, 2, 3, 4, 5) for inp in ("m", "m+")
            for hw in GRIDS + ((2 ** d, 2 ** (d + 1)),)]                       # the smallest legal grid of each depth
           + [UConfig("rgb+", 3, (32, 32), learn_obstacles=True)]                # as the reference's WarCraft setup
           + [UConfig("m+", 4, (32, 32), const=5.0, learn_obstacles=lo) for lo in (False, True)]
           + [UConfig("m+", 4, (128, 128))])                                    # above TAPS_MAX_SIDE


# ------------------------------------------------------------------------------------------------- the reference
def build_reference(ref_astar, cfg: UConfig, seed: int, device="cpu"):
    """The reference's NeuralAstar of `cfg` around a StandInUnet, its weights drawn from `seed` with 95 % of every conv's
    positive, its BatchNorms randomised during one float64 calibration forward of a batch of the configuration, its
    head scaled and shifted so that the logits of that batch have mean 0 and std HEAD_STD; float64, eval mode, every
    value fp32-representable, on `device`."""
    with torch.random.fork_rng(), pytest.MonkeyPatch.context() as mp:
        mp.setattr(ref_astar.encoder.smp, "Unet", stand_in_unet)
        torch.manual_seed(seed)
        ref = ref_astar.NeuralAstar(encoder_input=cfg.inp, encoder_arch="Unet", encoder_depth=cfg.depth,
                                    learn_obstacles=cfg.learn_obstacles, const=cfg.const)
    model = ref.encoder.model
    assert isinstance(model, StandInUnet)
    rng = np.random.RandomState(seed % 2 ** 32)
    with torch.no_grad():
        for m in model.modules():
            if isinstance(m, nn.Conv2d):
                positive = torch.from_numpy(rng.rand(*m.weight.shape) < POSITIVE)
                m.weight.copy_(torch.where(positive, m.weight.abs(), -m.weight.abs()))
    ref = ref.double().eval().to(device)
    x, _ = er.encoder_input(ref, *(torch.from_numpy(a).double().to(device) for a in er.inputs(cfg, seed + 1)))
    hooks = [m.register_forward_pre_hook(lambda mod, args: er.randomise_one_batchnorm(mod, args[0], rng))
             for m in model.modules() if isinstance(m, nn.BatchNorm2d)]
    try:
        with torch.no_grad():
            logits = model(x)
    finally:
        for h in hooks:
            h.remove()
    head = model.segmentation_head[0]
    with torch.no_grad():
        k = HEAD_STD / float(logits.std())
        head.weight.copy_((head.weight * k).float().double())
        head.bias.copy_(((head.bias - logits.mean()) * k).float().double())
    return ref


def build_product(ref, cfg: UConfig, **kw):
    """The product's NeuralAstar of `cfg` (and keyword arguments `kw`) holding the reference's state (fp32), in eval
    mode on the CPU."""
    from neural_astar.planner import NeuralAstar

    na = NeuralAstar(encoder_input=cfg.inp, encoder_arch="Unet", encoder_depth=cfg.depth,
                     learn_obstacles=cfg.learn_obstacles, const=cfg.const, **kw)
    result = na.load_state_dict(ref.state_dict())
    assert not result.missing_keys and not result.unexpected_keys, result
    return na.eval()


def const_of(ref) -> float:
    const = ref.encoder.const
    return float(const) if isinstance(const, float) else float(const.detach())


# ------------------------------------------------------------------------------------------------- the graph
class Node(NamedTuple):
    name: str                       # the reference module the stage computes (smp's name)
    kind: str                       # conv | pool | upcat | taps | cost (fast path) | head | sigmoid (module path)
    src: Tuple[int, ...]            # the nodes whose outputs feed it; -1 is the encoder input
    conv: Optional[nn.Conv2d] = None
    bn: Optional[nn.BatchNorm2d] = None


def reference_graph(model: StandInUnet, fast: bool) -> List[Node]:
    """The reference's U-Net as a list of stages in the order smp's forward runs them.  fast: the head ends in the
    eval fast path's per-pixel [C] x [C,9] products and their 9-tap gather into sigmoid(.) * const; otherwise in the
    head convolution and the sigmoid, as the module path computes them."""
    nodes: List[Node] = []

    def add(*a, **k) -> int:
        nodes.append(Node(*a, **k))
        return len(nodes) - 1

    mods, d = list(model.encoder.features), model.depth
    feats, cur, stage = [], -1, 0
    for i, m in enumerate(mods):
        if isinstance(m, nn.MaxPool2d):
            feats.append(cur)
            stage += 1
            if stage > d:
                break
            cur = add(f"encoder.features.{i}", "pool", (cur,))
        elif isinstance(m, nn.Conv2d):
            cur = add(f"encoder.features.{i}", "conv", (cur,), m, mods[i + 1])
    else:
        feats.append(cur)
    skips = feats[1:d][::-1]                # s_{d-1} .. s_1
    for j, blk in enumerate(model.decoder.center):
        cur = add(f"decoder.center.{j}", "conv", (cur,), blk[0], blk[1])
    for b, blk in enumerate(model.decoder.blocks):
        cur = add(f"decoder.blocks.{b}", "upcat", (cur,) + tuple(skips[b:b + 1]))
        cur = add(f"decoder.blocks.{b}.conv1", "conv", (cur,), blk.conv1[0], blk.conv1[1])
        cur = add(f"decoder.blocks.{b}.conv2", "conv", (cur,), blk.conv2[0], blk.conv2[1])
    head = model.segmentation_head[0]
    if fast:
        cur = add("segmentation_head.0", "taps", (cur,), head)
        add("cost", "cost", (cur,))
    else:
        cur = add("segmentation_head.0", "head", (cur,), head)
        add("sigmoid", "sigmoid", (cur,))
    return nodes


# ------------------------------------------------------------------------------------------------- the stage checker
class Stage(NamedTuple):
    name: str
    kind: str
    ratio: float                  # worst |product - float64| / bound: within the bound iff <= 1
    rel: Optional[float] = None   # conv: median (conv(|a|, |W|) + bmag) / median |pre-activation|
    K: Optional[int] = None       # conv: rounded fp32 operations per output, the bias included


def conv_c(u_op: float, K: int) -> float:
    """The relative factor of the conv + BatchNorm stage bound (tests/test_encoder_reference_cpu.py
    reference_and_bound): the fold, operands read with relative error u_op, K rounded operations."""
    return (1 + FOLD) * (1 + (PROD if u_op else 0.0)) * (1 + gamma(K)) - 1


def _ratio(got: torch.Tensor, want: torch.Tensor, bound: torch.Tensor) -> float:
    err = (got.double() - want).abs()
    return float(torch.where(err == 0, torch.zeros_like(err), err / bound).max())


def _exact(got: torch.Tensor, want: torch.Tensor) -> float:
    return 0.0 if got.shape == want.shape and torch.equal(got.double(), want) else float("inf")


def _gather(taps: torch.Tensor) -> torch.Tensor:
    """[B,H,W,9] -> [B,1,H,W]: sum over k = ky*3+kx of taps[y+ky-1][x+kx-1][k], zero outside the grid."""
    B, H, W, _ = taps.shape
    t = F.pad(taps.permute(0, 3, 1, 2), (1, 1, 1, 1))
    return sum(t[:, 3 * ky + kx, ky:ky + H, kx:kx + W] for ky in range(3) for kx in range(3)).unsqueeze(1)


def stage_ratios(ref, x: torch.Tensor, outs: List[torch.Tensor], fast: bool, u_op: float) -> List[Stage]:
    """Every stage of the reference's graph (`reference_graph`) evaluated in float64 on the product's recorded outputs
    `outs` (one per stage, in the graph's order) of the stages that feed it, x (the reference's encoder input) for the
    first, against the product's own output of the stage.  Tensors on any one device; ref's must be on it too.  The
    bounds, for the stage's own rounding alone:
      conv    conv + BatchNorm (+ ReLU): conv_c(u_op, K) (conv(|a|, |W|) + bmag), K = 9 C_in + 1, with the folded
              weights W = w s and bmag = |s| (|b_conv| + |mu|) + |beta| (reference_and_bound's terms);
      pool, upcat   exact;
      taps    the head's per-pixel products in C fp32 FMAs, in any order: gamma_C sum_c |a_c| |w_ck|;
      cost    sigmoid(bias + 9-tap gather) * const as nastar_common.cuh cost_from_taps computes it: the bias and 9
              fp32 additions, e = gamma_9 (|bias| + sum |taps|), then |const| (e / 4 + SIGMOID (sigmoid + e / 4));
      head    the module path's head conv: gamma_{9C+1} (conv(|a|, |w|) + |b|);
      sigmoid the module path's sigmoid(logit) * const: |const| SIGMOID sigmoid.
    A stage whose product output has another shape fails (ratio inf)."""
    graph = reference_graph(ref.encoder.model, fast)
    assert len(outs) == len(graph), (len(outs), [n.kind for n in graph])
    const = const_of(ref)
    res = []
    with torch.no_grad():
        for node, got in zip(graph, outs):
            a = [x if s < 0 else outs[s].double() for s in node.src]
            if node.kind == "conv":
                conv, bn = node.conv, node.bn
                s = bn.weight / torch.sqrt(bn.running_var + bn.eps)
                Wabs = (conv.weight * s.view(-1, 1, 1, 1)).abs()
                bmag = s.abs() * ((0 if conv.bias is None else conv.bias.abs()) + bn.running_mean.abs()) + bn.bias.abs()
                pre = F.batch_norm(F.conv2d(a[0], conv.weight, conv.bias, padding=1), bn.running_mean,
                                   bn.running_var, bn.weight, bn.bias, False, 0.0, bn.eps)
                mag = F.conv2d(a[0].abs(), Wabs, bmag, padding=1)
                K = 9 * conv.in_channels + 1
                ratio = _ratio(got, F.relu(pre), conv_c(u_op, K) * mag) if got.shape == pre.shape else float("inf")
                res.append(Stage(node.name, "conv", ratio, float(mag.median() / pre.abs().median()), K))
                continue
            if node.kind == "pool":
                ratio = _exact(got, F.max_pool2d(a[0], 2))
            elif node.kind == "upcat":
                ratio = _exact(got, torch.cat([F.interpolate(a[0], scale_factor=2, mode="nearest")] + a[1:], 1))
            elif node.kind == "taps":
                B, C, H, W = a[0].shape
                w = node.conv.weight[0].reshape(C, 9)
                got = got.reshape(B, H, W, 9)
                want = torch.einsum("bchw,ck->bhwk", a[0], w)
                ratio = _ratio(got, want, gamma(C) * torch.einsum("bchw,ck->bhwk", a[0].abs(), w.abs()))
            elif node.kind == "cost":
                bias = float(graph[node.src[0]].conv.bias)
                taps = a[0].reshape(got.shape[0], got.shape[2], got.shape[3], 9)      # torch.mm's are [P, 9]
                logit = bias + _gather(taps)
                e = gamma(9) * (abs(bias) + _gather(taps.abs()))
                sig = torch.sigmoid(logit)
                ratio = _ratio(got, sig * const, abs(const) * (e / 4 + SIGMOID * (sig + e / 4)))
            elif node.kind == "head":
                conv = node.conv
                want = F.conv2d(a[0], conv.weight, conv.bias, padding=1)
                mag = F.conv2d(a[0].abs(), conv.weight.abs(), conv.bias.abs(), padding=1)
                ratio = _ratio(got, want, gamma(9 * conv.in_channels + 1) * mag)
            else:
                assert node.kind == "sigmoid"
                sig = torch.sigmoid(a[0])
                ratio = _ratio(got, sig * const, abs(const) * SIGMOID * sig)
            res.append(Stage(node.name, node.kind, ratio))
    return res


# ------------------------------------------------------------------------------------------------- the module path
def record_module_path(na, maps, start, goal):
    """(encoder input, per-stage outputs) of the product's encode() on the CPU, recorded by hooks on the product's
    own modules, in reference_graph(fast=False)'s order."""
    model = na.encoder.model
    seen, outs, hooks = [], [], []
    convs = [m for m in model.modules() if isinstance(m, nn.Conv2d)]
    block_conv1 = {blk.conv1[0] for blk in model.decoder.blocks}

    def conv_in(mod, args):
        if mod in block_conv1:
            outs.append(args[0].clone())                    # the decoder block's upsample + concat
    hooks.append(model.register_forward_pre_hook(lambda mod, args: seen.append(args[0].clone())))
    for m in model.modules():
        if isinstance(m, nn.Conv2d):
            hooks.append(m.register_forward_pre_hook(conv_in))
        if isinstance(m, (nn.ReLU, nn.MaxPool2d)):
            hooks.append(m.register_forward_hook(lambda mod, args, out: outs.append(out.clone())))
    hooks.append(convs[-1].register_forward_hook(lambda mod, args, out: outs.append(out.clone())))
    try:
        with torch.no_grad():
            cost = na.encode(maps, start, goal)
    finally:
        for h in hooks:
            h.remove()
    return seen[0], outs + [cost]


# ------------------------------------------------------------------------------------------------- the tests
_REFERENCES = {}    # config id -> float64 reference (never mutated)
WORST = {}          # config id -> worst |error| / bound over the module path's stages
SHARES = {}         # config id -> (fp32, TF32) largest median conv-stage bound / median |pre-activation|


@pytest.fixture(scope="module")
def ref_astar():
    mod = er.staged_encoder_reference()
    if mod is None:
        pytest.skip("the reference's astar.py / encoder.py are not staged in oracle/_ref/ (build() stages them)")
    return mod


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    for key in sorted(WORST):
        f32, t32 = SHARES.get(key, (float("nan"), float("nan")))
        print(f"\n{key}: worst |error| / bound {WORST[key]:.4f}, largest median bound / |pre-activation| "
              f"{100 * f32:.3f} % (fp32) {100 * t32:.3f} % (TF32)")


def reference(ref_astar, cfg: UConfig):
    if cfg.id not in _REFERENCES:
        _REFERENCES[cfg.id] = build_reference(ref_astar, cfg, cfg.seed)
    return _REFERENCES[cfg.id]


def test_stand_in_matches_smp():
    """Where segmentation_models_pytorch is importable, the stand-in is its Unet: the same state dict layout, and the
    same logits once either's state is loaded into the other."""
    smp = pytest.importorskip("segmentation_models_pytorch")
    for d in (1, 4, 5):
        torch.manual_seed(d)
        theirs = smp.Unet(encoder_name="vgg16_bn", encoder_weights=None, classes=1, in_channels=2, encoder_depth=d,
                          decoder_channels=DEC[:d]).double().eval()
        ours = StandInUnet(2, d).double().eval()
        ours.load_state_dict(theirs.state_dict(), strict=True)
        x = torch.rand(2, 2, 64, 64, dtype=torch.float64)
        with torch.no_grad():
            torch.testing.assert_close(ours(x), theirs(x), atol=1e-12, rtol=0)


@pytest.mark.parametrize("d", [1, 2, 3, 4, 5])
def test_stand_in_layout(d):
    """smp 0.3.1's names and shapes, as tests/test_unet_cpu.py lists them."""
    got = {k: tuple(v.shape) for k, v in StandInUnet(4, d).state_dict().items()}
    assert got == expected_layout(4, d)


@pytest.mark.parametrize("cfg", CONFIGS, ids=[c.id for c in CONFIGS])
def test_state_dicts_interchange(ref_astar, cfg):
    """The reference's float64 state dict loads into the product with every key matched, and the product's into a fresh
    reference; every value survives both ways."""
    ref = reference(ref_astar, cfg)
    na = build_product(ref, cfg)
    for k, v in ref.state_dict().items():
        assert torch.equal(na.state_dict()[k].double(), v), k
    with pytest.MonkeyPatch.context() as mp:
        mp.setattr(ref_astar.encoder.smp, "Unet", stand_in_unet)
        fresh = ref_astar.NeuralAstar(encoder_input=cfg.inp, encoder_arch="Unet", encoder_depth=cfg.depth,
                                      learn_obstacles=cfg.learn_obstacles, const=cfg.const)
    result = fresh.load_state_dict(na.state_dict())
    assert not result.missing_keys and not result.unexpected_keys, result
    for k, v in na.state_dict().items():
        assert torch.equal(fresh.state_dict()[k], v), k


@pytest.mark.parametrize("cfg", CONFIGS, ids=[c.id for c in CONFIGS])
def test_module_path_within_stage_bounds(ref_astar, cfg):
    """The reference's encode() is the stand-in's forward, which is functional_unet; its costs are not saturated.  The
    product's fp32 module path on the CPU meets every stage's fp32 bound, and the bounds are not vacuous."""
    ref = reference(ref_astar, cfg)
    maps, start, goal = (torch.from_numpy(v) for v in er.inputs(cfg, cfg.seed))
    x, cost = er.encoder_input(ref, maps.double(), start.double(), goal.double())
    model = ref.encoder.model
    const = const_of(ref)
    with torch.no_grad():
        assert torch.equal(cost, torch.sigmoid(model(x)) * const)
        if cfg.grid[0] % 32 == 0 and cfg.grid[1] % 32 == 0:      # functional_unet runs all five of vgg16's pools
            sd = model.state_dict()
            torch.testing.assert_close(model(x), functional_unet(x, sd, cfg.depth), atol=1e-12, rtol=0)
    spread = float((cost - const / 2).abs().median())
    assert 0.02 * const / 2 < spread < 0.5 * const / 2, ("costs flat or saturated", spread)

    na = build_product(ref, cfg)
    got_x, outs = record_module_path(na, maps, start, goal)
    assert torch.equal(got_x.double(), x)
    stages = stage_ratios(ref, x, outs, fast=False, u_op=0.0)
    WORST[cfg.id] = max(s.ratio for s in stages)
    for s in stages:
        assert s.ratio <= 1.0, (cfg.id, s)
    convs = [s for s in stages if s.kind == "conv"]
    assert len(convs) == [4, 7, 10, 13, 13][cfg.depth - 1] + 2 + 2 * cfg.depth
    f32 = max(conv_c(0.0, s.K) * s.rel for s in convs)
    t32 = max(conv_c(U_TF32, s.K) * s.rel for s in convs)
    SHARES[cfg.id] = (f32, t32)
    assert f32 < VACUOUS_FP32 and t32 < VACUOUS_TF32, (cfg.id, f32, t32)
