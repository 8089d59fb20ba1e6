"""Cost-map encoders (plain PyTorch; the north star keeps them on cuDNN).

Same classes, constructor arguments and state-dict layout as
/root/reference/src/neural_astar/planner/encoder.py:12-97 so reference checkpoints load:
`model.{0,3,6,...}` are 3x3 convs, `model.{1,4,7,...}` BatchNorms, ReLU (and MaxPool for
CNNDownSize) in between, trailing activation(s) dropped; output = sigmoid(model(x)) * const.
"""
from __future__ import annotations

import os
from typing import List, NamedTuple, Optional

import numpy as np
import torch
import torch.nn as nn
import torch.nn.functional as F

from .. import _native

# Precision of the eval fast path's 3x3 convolutions: TF32 tensor-core math (what torch's own default
# `torch.backends.cudnn.allow_tf32 = True` gives the reference on any Ampere+ GPU) or full fp32.  The head
# (last, single-output-channel conv) is always fp32.  bench.py states this in its `dtype` field;
# tests/test_gpu_module_api.py counts how many search masks differ between the two settings.
ALLOW_TF32 = os.environ.get("NASTAR_B200_ENCODER_TF32", "1") != "0"
# The head's per-pixel [C] x [C,9] product: the engine's streaming kernel (csrc/nastar_glue.cuh head_taps_kernel, fp32
# FMA, weights in the constant bank) or, with NASTAR_B200_HEAD_KERNEL=0, torch.mm (cuBLAS SGEMM on this skinny
# shape).  Same sums up to fp32 re-association.
HEAD_KERNEL = os.environ.get("NASTAR_B200_HEAD_KERNEL", "1") != "0"
# First layer of the "m+" CNN (2 -> 32 channels, 18 multiply-adds per output): the engine's kernel that also forms the
# start+goal channel and the concat on the fly (csrc/nastar_glue.cuh conv1_marks_kernel, fp32 FMA), or, with
# NASTAR_B200_CONV1_KERNEL=0, the pack_inputs kernel followed by cuDNN's (also fp32, generic NHWC) convolution.
CONV1_KERNEL = os.environ.get("NASTAR_B200_CONV1_KERNEL", "1") != "0"


class _Layer(NamedTuple):
    """A conv + BatchNorm (running statistics) block folded into one convolution: cuDNN's conv + bias (+ ReLU) op,
    then the block's max-pool if it has one."""
    w: torch.Tensor              # folded weights, channels-last
    b: torch.Tensor              # folded bias
    stride: tuple
    padding: tuple
    dilation: tuple
    relu: bool
    pool: Optional[nn.MaxPool2d]


class _Plan(NamedTuple):
    """An encoder's eval fast path: BatchNorm folded into every conv, ready for channels-last cuDNN convolutions."""
    body: object                 # what the class's _run_body runs up to the last conv (CNN: a list of _Layer)
    last: Optional[_Layer]       # the last conv before the head, run by cuDNN or the fused conv + head kernel (None
                                 # for a CNN of depth 0, whose head reads the input)
    head_w: np.ndarray           # the head's [C,9] weights on the host (a parameter of the head kernels)
    head_wm: torch.Tensor        # the same on the device, for torch.mm
    head_b: float                # the head's bias
    const: float
    conv1: Optional[tuple]       # host ([9,2,32], [32]) weights of conv1_marks for a 2 -> 32 first layer, else None


def _fold(conv: nn.Conv2d, bn: nn.BatchNorm2d, relu: bool = True, pool: Optional[nn.MaxPool2d] = None) -> _Layer:
    """One plan layer; a conv without bias gets a zero one.  The op order fixes the folded weights' bits."""
    scale = bn.weight / torch.sqrt(bn.running_var + bn.eps)
    w = (conv.weight * scale.view(-1, 1, 1, 1)).contiguous(memory_format=torch.channels_last)
    bias = conv.bias if conv.bias is not None else torch.zeros_like(bn.running_mean)
    b = ((bias - bn.running_mean) * scale + bn.bias).contiguous()
    return _Layer(w, b, conv.stride, conv.padding, conv.dilation, relu, pool)


def _host(t: torch.Tensor) -> np.ndarray:
    return t.cpu().numpy().astype("float32", order="C")


def _head_fields(w: torch.Tensor, b: torch.Tensor):
    """(head_w, head_wm, head_b) of a single-output-channel 3x3 head with weights [1,C,3,3] and bias [1]."""
    wm = w[0].reshape(w.shape[1], 9).contiguous()
    return _host(wm), wm, float(b.reshape(-1)[0])


def _conv(layer: _Layer, x: torch.Tensor) -> torch.Tensor:
    w, b, stride, padding, dilation, relu, pool = layer
    if relu:
        x = torch.cudnn_convolution_relu(x, w, b, stride, padding, dilation, 1)
    else:
        x = F.conv2d(x, w, b, stride, padding, dilation, 1)
    return pool(x) if pool is not None else x


def _run_layers(layers, x: torch.Tensor) -> torch.Tensor:
    for layer in layers:
        x = _conv(layer, x)
    return x


def _conv_flags():
    """cuDNN settings of the eval fast path.  Inference shapes are static, so cuDNN may time its candidates once
    per shape instead of trusting the heuristic (which can pick a much slower kernel for a layer) —
    unless the user asked for determinism (set_global_seeds(), utils/training.py): autotuned algorithm choice can
    differ run to run, so `torch.backends.cudnn.deterministic = True` is honoured and turns autotuning off."""
    det = bool(torch.backends.cudnn.deterministic)
    return torch.backends.cudnn.flags(enabled=True, benchmark=not det, deterministic=det, allow_tf32=ALLOW_TF32)


def _fuses(last: _Layer, x: torch.Tensor) -> bool:
    """The engine's fused last conv + head kernel covers this conv: TF32 convolutions allowed, the head kernel on,
    a 3x3 / pad 1 / stride 1 128 -> 256 conv with ReLU and no pooling, maps up to 64x64."""
    return (ALLOW_TF32 and HEAD_KERNEL and last.relu and last.pool is None
            and tuple(last.w.shape) == (_native.CONVHEAD_CHANNELS[1], _native.CONVHEAD_CHANNELS[0], 3, 3)
            and tuple(last.stride) == (1, 1) and tuple(last.padding) == (1, 1) and tuple(last.dilation) == (1, 1)
            and x.is_cuda and x.dtype == torch.float32 and x.shape[1] == _native.CONVHEAD_CHANNELS[0]
            and x.shape[-2] <= _native.CONVHEAD_MAX_SIDE and x.shape[-1] <= _native.CONVHEAD_MAX_SIDE)


class EncoderBase(nn.Module):
    def __init__(self, input_dim: int, encoder_depth: int = 4, const: Optional[float] = None):
        super().__init__()
        self.model = self.construct_encoder(input_dim, encoder_depth)
        # learnable scale when given (reference :25-28); plain 1.0 otherwise
        self.const = nn.Parameter(torch.ones(1) * const) if const is not None else 1.0
        self._plan = None       # cached _Plan of the eval fast path
        self._plan_key = None
        self._nhwc = False      # conv weights converted to channels-last (done lazily on the first CUDA batch)

    def construct_encoder(self, input_dim: int, encoder_depth: int) -> nn.Module:
        raise NotImplementedError

    def _fold_plan(self) -> Optional[_Plan]:
        """The modules folded into a _Plan (called without autograd), or None when they do not fold."""
        raise NotImplementedError

    def _run_body(self, plan: _Plan, x: torch.Tensor) -> torch.Tensor:
        """plan.body on the channels-last input x: the activation that plan.last takes."""
        raise NotImplementedError

    def fast_path_ok(self, x: torch.Tensor) -> bool:
        """Eval-mode, no-grad, fp32 CUDA input: the folded cuDNN plan (and the fused hand-off) may be used."""
        return (not self.training) and x.is_cuda and not torch.is_grad_enabled() and x.dtype == torch.float32

    def prepare_channels_last(self) -> None:
        """One-off, explicit: store the conv weights channels-last (cuDNN's tensor-core convolutions are
        NHWC-native).  Pure memory-format change: the Parameter objects,
        shapes and state-dict contents are unchanged.  Call it once after moving the module to the GPU — before
        wrapping it in DDP or capturing a CUDA graph.  forward() calls it on the first CUDA batch otherwise."""
        if not self._nhwc:
            self.model.to(memory_format=torch.channels_last)
            self._nhwc = True

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        if self.fast_path_ok(x):
            head = self.head_taps(x)
            if head is not None:
                # sigmoid(.)*const finished by the engine's glue kernel: the very arithmetic the fused search
                # prologue performs (NASTAR_COST_TAPS), so encode() and the fused forward agree bit for bit
                return _native.cost_from_taps(*head)
        if x.is_cuda and x.dim() == 4:
            self.prepare_channels_last()
            x = x.contiguous(memory_format=torch.channels_last)
        return torch.sigmoid(self.model(x)) * self.const

    def head_taps(self, x: torch.Tensor, out: Optional[torch.Tensor] = None, on_last_conv=None):
        """Eval fast path up to (not including) the 9-tap gather of the single-output-channel head:
        returns (taps [B,H,W,9] fp32 contiguous, folded bias, const) as (tensor, float, float), or None when the
        encoder does not fold.  bias/const are cached Python floats (no host sync per call)."""
        plan = self._inference_plan(x.device)
        if plan is None:
            return None
        with _conv_flags():
            x = self._run_body(plan, x.contiguous(memory_format=torch.channels_last))
            return self._head_step(plan, x, plan.last, out, on_last_conv)

    def head_taps_marks(self, map_designs: torch.Tensor, start_maps: torch.Tensor, goal_maps: torch.Tensor,
                        out: Optional[torch.Tensor] = None, on_last_conv=None):
        """head_taps() of the "m+" input cat(map_designs, start_maps + goal_maps) without materialising it: the first
        layer reads the three planes directly (one kernel instead of pack_inputs + cuDNN's conv1).  None when the
        encoder's first layer is not the 2->32 3x3/ReLU block, the maps are not one-channel or the marks live on a
        different grid; callers then pack the input and use head_taps()."""
        if not CONV1_KERNEL or map_designs.shape[1] != 1 or map_designs.shape[-2:] != start_maps.shape[-2:]:
            return None
        plan = self._inference_plan(map_designs.device)
        if plan is None or plan.conv1 is None:
            return None
        x = _native.conv1_marks(map_designs, start_maps, goal_maps, *plan.conv1)
        with _conv_flags():
            if not plan.body:       # conv1 is the last conv itself
                return self._head_step(plan, x, None, out, on_last_conv)
            # only a CNN has conv1 weights, and its body is a list of layers: conv1_marks computed the first
            return self._head_step(plan, _run_layers(plan.body[1:], x), plan.last, out, on_last_conv)

    def _head_step(self, plan: _Plan, x: torch.Tensor, last: Optional[_Layer], out: Optional[torch.Tensor],
                   on_last_conv):
        """The conv `last` on x (None: x is already its output) and the head's products, written into `out` if given.
        `on_last_conv`, if given, is called once, before the last (widest) conv is enqueued: PipelinedPlanner forks the
        previous batch's search there (see its docstring)."""
        if on_last_conv is not None:
            on_last_conv()
        if last is not None and _fuses(last, x):
            # the last conv and the head products in one TF32 tensor-core kernel: its activation never reaches HBM
            x = x.contiguous(memory_format=torch.channels_last)
            return _native.conv3x3_head_taps(x, last.w, last.b, plan.head_w, out=out), plan.head_b, plan.const
        if last is not None:
            x = _conv(last, x)
        x = x.contiguous(memory_format=torch.channels_last)
        B, C, H, W = x.shape
        if HEAD_KERNEL and C in _native.HEAD_CHANNELS:
            taps = _native.head_taps(x, plan.head_w, out=out)
        else:   # torch.mm writes straight into a caller-owned [B,H,W,9] buffer
            a = x.permute(0, 2, 3, 1).reshape(-1, C)
            taps = torch.mm(a, plan.head_wm, out=None if out is None else out.view(-1, 9)).view(B, H, W, 9)
        return taps, plan.head_b, plan.const

    # ---- eval-mode cuDNN fast path (SURVEY 8(f) rank 3: encoder -> search hand-off) -----------------
    # Still plain PyTorch/cuDNN: BatchNorm (running stats) is folded into the preceding conv, activations
    # run channels-last (no NCHW<->NHWC transposes), and conv+bias+ReLU is one cuDNN fused op.  Same math
    # as self.model(x) up to fp32 re-association of the BN scale; training / autograd use self.model.
    def _inference_plan(self, device) -> Optional[_Plan]:
        """The _Plan of the current weights, rebuilt (one host sync) when a parameter or buffer has changed."""
        # the weights' layout first: the key then stays put between a warm-up and a captured call
        self.prepare_channels_last()
        tensors = list(self.model.parameters()) + list(self.model.buffers())
        if isinstance(self.const, torch.Tensor):
            tensors.append(self.const)
        key = (str(device),) + tuple((t.data_ptr(), t._version) for t in tensors)
        if key != self._plan_key:
            with torch.no_grad():
                self._plan, self._plan_key = self._fold_plan(), key
        return self._plan

    def _const(self) -> float:
        return float(self.const) if not isinstance(self.const, float) else self.const


def _conv_stack(widths: List[int], pool: bool) -> nn.Sequential:
    layers: List[nn.Module] = []
    tail = 2 if pool else 1  # modules to drop after the last BatchNorm
    for cin, cout in zip(widths[:-1], widths[1:]):
        layers += [nn.Conv2d(cin, cout, kernel_size=3, stride=1, padding=1), nn.BatchNorm2d(cout), nn.ReLU()]
        if pool:
            layers.append(nn.MaxPool2d((2, 2)))
    return nn.Sequential(*layers[:-tail])


class CNN(EncoderBase):
    CHANNELS = [32, 64, 128, 256]

    def construct_encoder(self, input_dim: int, encoder_depth: int) -> nn.Module:
        return _conv_stack([input_dim] + self.CHANNELS[:encoder_depth] + [1], pool=False)

    def _fold_plan(self) -> Optional[_Plan]:
        """Conv, BatchNorm[, ReLU][, MaxPool] blocks; the last one, without ReLU or pool, a 3x3 one-output head."""
        mods, layers, i = list(self.model), [], 0
        while i < len(mods):
            conv = mods[i]
            if not (isinstance(conv, nn.Conv2d) and conv.groups == 1 and i + 1 < len(mods)
                    and isinstance(mods[i + 1], nn.BatchNorm2d)):
                return None
            bn = mods[i + 1]
            i += 2
            relu = i < len(mods) and isinstance(mods[i], nn.ReLU)
            i += 1 if relu else 0
            pool = mods[i] if i < len(mods) and isinstance(mods[i], nn.MaxPool2d) else None
            i += 1 if pool is not None else 0
            layers.append(_fold(conv, bn, relu, pool))
        head = layers.pop()
        if not (head.w.shape[:1] == (1,) and head.w.shape[2:] == (3, 3) and tuple(head.stride) == (1, 1)
                and tuple(head.padding) == (1, 1) and tuple(head.dilation) == (1, 1) and not head.relu
                and head.pool is None):
            return None
        conv1 = None
        if layers:
            w0, b0, st0, pad0, dil0, relu0, pool0 = layers[0]
            if (tuple(w0.shape) == (32, 2, 3, 3) and tuple(st0) == (1, 1) and tuple(pad0) == (1, 1)
                    and tuple(dil0) == (1, 1) and relu0 and pool0 is None and w0.is_cuda and w0.dtype == torch.float32):
                conv1 = (_host(w0.permute(2, 3, 1, 0).reshape(9, 2, 32)), _host(b0))   # [tap, cin, cout]
        last = layers.pop() if layers else None
        return _Plan(layers, last, *_head_fields(head.w, head.b), self._const(), conv1)

    def _run_body(self, plan: _Plan, x: torch.Tensor) -> torch.Tensor:
        return _run_layers(plan.body, x)


class CNNDownSize(CNN):
    def construct_encoder(self, input_dim: int, encoder_depth: int) -> nn.Module:
        return _conv_stack([input_dim] + self.CHANNELS[:encoder_depth] + [1], pool=True)


# torchvision's vgg16_bn feature stack (cfg "D"): 13 conv/BatchNorm/ReLU blocks and 5 max-pools, modules 0..43.  The
# U-Net's encoder stages split it at each pool, the pool opening the next stage: module ranges [start, end) of s0..s5.
_VGG16 = [64, 64, "M", 128, 128, "M", 256, 256, 256, "M", 512, 512, 512, "M", 512, 512, 512, "M"]
_VGG16_STAGES = [(0, 6), (6, 13), (13, 23), (23, 33), (33, 43), (43, 44)]
_VGG16_STAGE_CHANNELS = [64, 128, 256, 512, 512, 512]


def _check_sides(x: torch.Tensor, depth: int) -> None:
    m = 2 ** depth
    if x.shape[-2] % m or x.shape[-1] % m:
        raise ValueError(f"Unet with encoder_depth={depth} needs input sides divisible by 2**{depth} = {m}, "
                         f"got {tuple(x.shape[-2:])}")


def _conv2d_relu(cin: int, cout: int) -> nn.Sequential:
    return nn.Sequential(nn.Conv2d(cin, cout, 3, padding=1, bias=False), nn.BatchNorm2d(cout), nn.ReLU(inplace=True))


class _VggEncoder(nn.Module):
    def __init__(self, input_dim: int, depth: int):
        super().__init__()
        layers: List[nn.Module] = []
        cin = input_dim
        for v in _VGG16:
            if v == "M":
                layers.append(nn.MaxPool2d(kernel_size=2, stride=2))
            else:
                layers += [nn.Conv2d(cin, v, kernel_size=3, padding=1), nn.BatchNorm2d(v), nn.ReLU(inplace=True)]
                cin = v
        self.features = nn.Sequential(*layers)
        self.depth = depth

    def forward(self, x: torch.Tensor) -> List[torch.Tensor]:
        """Outputs of stages s0..s_depth."""
        feats = []
        for a, b in _VGG16_STAGES[:self.depth + 1]:
            for m in self.features[a:b]:
                x = m(x)
            feats.append(x)
        return feats


class _DecoderBlock(nn.Module):
    def __init__(self, cin: int, cskip: int, cout: int):
        super().__init__()
        self.conv1 = _conv2d_relu(cin + cskip, cout)
        self.attention1 = nn.Identity()
        self.conv2 = _conv2d_relu(cout, cout)
        self.attention2 = nn.Identity()

    def forward(self, x: torch.Tensor, skip: Optional[torch.Tensor]) -> torch.Tensor:
        x = F.interpolate(x, scale_factor=2, mode="nearest")
        if skip is not None:
            x = torch.cat([x, skip], dim=1)
        return self.attention2(self.conv2(self.conv1(self.attention1(x))))


class _UnetDecoder(nn.Module):
    def __init__(self, stage_channels: List[int], decoder_channels: List[int]):
        super().__init__()
        enc = stage_channels[1:][::-1]          # s_d .. s1: the full-resolution s0 is not a skip
        head = enc[0]
        ins = [head] + decoder_channels[:-1]
        skips = enc[1:] + [0]
        self.center = nn.Sequential(_conv2d_relu(head, head), _conv2d_relu(head, head))
        self.blocks = nn.ModuleList([_DecoderBlock(i, s, o) for i, s, o in zip(ins, skips, decoder_channels)])

    def forward(self, feats: List[torch.Tensor]) -> torch.Tensor:
        feats = feats[1:][::-1]
        x = self.center(feats[0])
        skips = feats[1:]
        for i, block in enumerate(self.blocks):
            x = block(x, skips[i] if i < len(skips) else None)
        return x


class _UnetModel(nn.Module):
    """smp 0.3.1's `Unet(encoder_name="vgg16_bn", classes=1)` in plain torch.nn: same modules, names and shapes."""

    def __init__(self, input_dim: int, decoder_channels: List[int]):
        super().__init__()
        depth = len(decoder_channels)
        self.depth = depth
        self.encoder = _VggEncoder(input_dim, depth)
        self.decoder = _UnetDecoder(_VGG16_STAGE_CHANNELS[:depth + 1], decoder_channels)
        self.segmentation_head = nn.Sequential(nn.Conv2d(decoder_channels[-1], 1, kernel_size=3, padding=1))
        # smp's initialisation: torchvision's VGG init, except that the first conv is re-created for input_dim != 3
        # and keeps PyTorch's default init; kaiming-uniform decoder convs; a xavier head with a zero bias
        for i, m in enumerate(self.encoder.features):
            if isinstance(m, nn.Conv2d) and not (i == 0 and input_dim != 3):
                nn.init.kaiming_normal_(m.weight, mode="fan_out", nonlinearity="relu")
                nn.init.zeros_(m.bias)
        for m in self.decoder.modules():
            if isinstance(m, nn.Conv2d):
                nn.init.kaiming_uniform_(m.weight, mode="fan_in", nonlinearity="relu")
        for m in self.modules():
            if isinstance(m, nn.BatchNorm2d):
                nn.init.ones_(m.weight)
                nn.init.zeros_(m.bias)
        nn.init.xavier_uniform_(self.segmentation_head[0].weight)
        nn.init.zeros_(self.segmentation_head[0].bias)

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        _check_sides(x, self.depth)
        return self.segmentation_head(self.decoder(self.encoder(x)))


class Unet(EncoderBase):
    """U-Net with a VGG-16-BN backbone: the network of segmentation_models_pytorch 0.3.1's
    `Unet(encoder_name="vgg16_bn", encoder_weights=None, classes=1, in_channels=input_dim, encoder_depth=d,
    decoder_channels=DECODER_CHANNELS[:d])` (reference :37-57), built from torch.nn so that state dicts load in either
    direction.  Input sides must be divisible by 2**encoder_depth.

    Eval fast path (`head_taps`): BatchNorm folded into every conv, channels-last cuDNN convolutions, each decoder
    block's upsample + concat as one kernel (`_native.upsample_concat`), and the head's per-pixel [C] x [C,9] products
    handed to the search's NASTAR_COST_TAPS prologue like the CNN's."""

    DECODER_CHANNELS = [256, 128, 64, 32, 16]

    def construct_encoder(self, input_dim: int, encoder_depth: int) -> nn.Module:
        if encoder_depth not in range(1, 6):
            raise ValueError(f"Unet needs encoder_depth in 1..5, got {encoder_depth}")
        return _UnetModel(input_dim, self.DECODER_CHANNELS[:encoder_depth])

    def _fold_plan(self) -> _Plan:
        """body = (encoder stages, center, decoder blocks): stages and center lists of layers, each block its convs; the
        last block's conv2 is plan.last."""
        feats = self.model.encoder.features
        stages = []
        for a, b in _VGG16_STAGES[:self.model.depth + 1]:
            mods = list(feats[a:b])
            stages.append([_fold(c, n) for c, n in zip(mods, mods[1:]) if isinstance(c, nn.Conv2d)])
        dec = self.model.decoder
        center = [_fold(blk[0], blk[1]) for blk in dec.center]
        blocks = [[_fold(blk.conv1[0], blk.conv1[1]), _fold(blk.conv2[0], blk.conv2[1])] for blk in dec.blocks]
        last = blocks[-1].pop()
        head = self.model.segmentation_head[0]
        return _Plan((stages, center, blocks), last, *_head_fields(head.weight, head.bias), self._const(), None)

    def _run_body(self, plan: _Plan, x: torch.Tensor) -> torch.Tensor:
        _check_sides(x, self.model.depth)
        stages, center, blocks = plan.body
        feats = []
        for i, stage in enumerate(stages):
            if i:
                x = F.max_pool2d(x, 2)
            x = _run_layers(stage, x)
            feats.append(x)
        skips = feats[1:-1][::-1] + [None]
        x = _run_layers(center, x)
        cl = torch.channels_last
        for layers, skip in zip(blocks, skips):
            x = _native.upsample_concat(x.contiguous(memory_format=cl),
                                        None if skip is None else skip.contiguous(memory_format=cl))
            x = _run_layers(layers, x)
        return x
