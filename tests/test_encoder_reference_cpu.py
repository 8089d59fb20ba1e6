"""Pin NeuralAstar's CNN encoders to the reference's own NeuralAstar run in float64, element by element.

The staged reference (oracle/_ref/neural_astar/planner/{astar,encoder}.py, byte for byte, put there by build()) builds
each configuration of `CONFIGS` with a seed.  Its BatchNorms get statistics far from the identity (`randomise_batchnorm`),
it is converted to float64, and its state dict is loaded into the product's NeuralAstar.  `reference_and_bound` then
walks the reference's own nn.Sequential in float64, module by module, and carries an element-wise bound on |product -
reference| for an fp32 evaluation whose layers round as `layer_rounding` says.  Checked here, without a GPU:
  state dicts   both directions load with every key matched and every value kept;
  module path   the product's encode() in fp32 on the CPU (nn.Sequential, BatchNorm unfolded) is within the bound with
                fp32 operands, for every configuration;
  bound         the bound is not vacuous: in fp32 its median is under 1 % of the median distance of the cost from
                const / 2, and with TF32 operands in every layer (its loosest form) under that distance.

tests/test_gpu_encoder_reference.py runs the same matrix through the eval fast path (folded plan, conv1_marks, cuDNN,
the fused 128 -> 256 conv + head kernel, head_taps, cost_from_taps and the search's TAPS prologue) on the GPU.
"""
from __future__ import annotations

import importlib
import importlib.util
import os
import sys
import types
import zlib
from typing import List, NamedTuple, Optional, Tuple

import numpy as np
import pytest
import scipy.ndimage
import torch
import torch.nn as nn
import torch.nn.functional as F

from test_gpu_convhead import PROD, U_TF32

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF_ROOT = os.path.join(ROOT, "oracle", "_ref")
REF_PLANNER = os.path.join(REF_ROOT, "neural_astar", "planner")
REF_FILES = ("astar.py", "encoder.py", "differentiable_astar.py", "pq_astar.py")
REF_STUBS = ("segmentation_models_pytorch", "pqdict")   # staged next to the planner; the CNN encoders never use them
REF_PACKAGE = "_ref_encoder_planner"

U = 2.0 ** -24          # fp32 unit roundoff
FOLD = 10 * U           # BatchNorm in fp32, folded or not: see reference_and_bound
SIGMOID = 8 * U         # sigmoid(x) * const in fp32: see reference_and_bound
CHANNELS = [32, 64, 128, 256]
POSITIVE = 0.95        # share of the conv weights made positive: see build_reference


# ------------------------------------------------------------------------------------------------- the reference
def staged_encoder_reference():
    """The staged reference's `astar` module (its NeuralAstar, with `encoder` beside it), imported under a private package
    name so that it meets neither this project's `neural_astar` nor the `_ref_planner` package other tests import with
    their own `pqdict`; None where oracle/_ref/ is not staged.  The two stub modules it imports are registered from their
    staged files for the import only, so that no other test sees them."""
    if not (all(os.path.isfile(os.path.join(REF_PLANNER, f)) for f in REF_FILES)
            and all(os.path.isfile(os.path.join(REF_ROOT, s, "__init__.py")) for s in REF_STUBS)):
        return None
    if REF_PACKAGE + ".astar" in sys.modules:
        return sys.modules[REF_PACKAGE + ".astar"]
    pkg = types.ModuleType(REF_PACKAGE)
    pkg.__path__ = [REF_PLANNER]
    sys.modules[REF_PACKAGE] = pkg
    saved = {name: sys.modules.get(name) for name in REF_STUBS}
    try:
        for name in REF_STUBS:
            spec = importlib.util.spec_from_file_location(name, os.path.join(REF_ROOT, name, "__init__.py"))
            stub = importlib.util.module_from_spec(spec)
            spec.loader.exec_module(stub)
            sys.modules[name] = stub
        return importlib.import_module(REF_PACKAGE + ".astar")
    finally:
        for name, mod in saved.items():
            if mod is None:
                sys.modules.pop(name, None)
            else:
                sys.modules[name] = mod


@pytest.fixture(scope="module")
def ref_astar():
    mod = staged_encoder_reference()
    if mod is None:
        pytest.skip("the reference's astar.py / encoder.py are not staged in oracle/_ref/ (build() stages them)")
    return mod


# ------------------------------------------------------------------------------------------------- the configurations
class Config(NamedTuple):
    arch: str                  # "CNN" or "CNNDownSize"
    inp: str                   # encoder_input: "m", "m+", "rgb" or "rgb+"
    depth: int                 # encoder_depth
    image: Tuple[int, int]     # map_designs' H, W
    grid: Tuple[int, int]      # the planning grid: start / goal maps and cost maps
    const: Optional[float]
    learn_obstacles: bool

    @property
    def id(self):
        (hm, wm), (h, w) = self.image, self.grid
        side = f"{hm}x{wm}" if self.image == self.grid else f"{hm}x{wm}to{h}x{w}"
        extra = ("" if self.const is None else f"-c{self.const:g}") + ("-lo" if self.learn_obstacles else "")
        return f"{self.arch}-{self.inp}-d{self.depth}-{side}{extra}"

    @property
    def seed(self):
        return zlib.crc32(self.id.encode())

    @property
    def B(self):
        """2 to 6 maps"""
        return 2 + self.seed % 5

    @property
    def conv1_marks(self):
        """The "m+" CNN reads the map and the marks in its first layer's kernel (EncoderBase.head_taps_marks)."""
        return self.arch == "CNN" and self.inp == "m+" and self.image == self.grid

    @property
    def head_channels(self):
        return CHANNELS[self.depth - 1]

    @property
    def fused(self):
        """The last body layer is an unpooled 128 -> 256 conv: the fused conv + head kernel's layer."""
        return self.arch == "CNN" and self.depth == 4


def _cnn(inp, depth, H, W, const=None, learn_obstacles=False):
    return Config("CNN", inp, depth, (H, W), (H, W), const, learn_obstacles)


def _down(inp, depth, side):
    """CNNDownSize pools after every block but the head's: the grid is side / 2**depth.  learn_obstacles on, as the
    reference's WarCraft configuration has it."""
    return Config("CNNDownSize", inp, depth, (side, side), (side >> depth, side >> depth), None, True)


SHAPES = ((32, 32), (64, 64), (20, 48), (48, 20), (5, 3))
CONFIGS = ([_cnn("m+", d, H, W) for d in (1, 2, 3, 4) for H, W in SHAPES]
           + [_cnn("m", d, H, W) for d in (2, 4) for H, W in ((32, 32), (20, 48))]
           + [_cnn("m+", 4, 32, 32, const=5.0, learn_obstacles=lo) for lo in (False, True)]
           + [_down("rgb+", d, side) for d, side in ((1, 48), (2, 48), (3, 96), (4, 64))]
           + [_down("rgb", 3, 96)])
LARGEST = _cnn("m+", 4, 64, 64)


def inputs(cfg: Config, seed: int):
    """(map_designs, start_maps, goal_maps) float32 NumPy arrays: binary obstacle maps (a quarter blocked) or RGB images
    in [0, 1), and one-hot starts and goals on passable cells of the grid, each goal reachable from its start; map 0 has
    start == goal."""
    rng = np.random.RandomState(seed)
    B, (Hm, Wm), (H, W) = cfg.B, cfg.image, cfg.grid
    if cfg.inp.startswith("rgb"):
        maps = rng.rand(B, 3, Hm, Wm).astype(np.float32)
        passable = np.ones((B, H, W), np.float32)
    else:
        maps = (rng.rand(B, 1, H, W) > 0.25).astype(np.float32)
        maps[:, 0, 0, 0] = 1
        passable = maps[:, 0]
    start = np.zeros((B, 1, H, W), np.float32)
    goal = np.zeros_like(start)
    for b in range(B):
        s = rng.choice(np.flatnonzero(passable[b]))
        # the goal in the start's 8-connected region: the reference's backtrack fails on an unreachable goal
        labels, _ = scipy.ndimage.label(passable[b], structure=np.ones((3, 3), int))
        g = s if b == 0 else rng.choice(np.flatnonzero(labels == labels.flat[s]))
        start[b, 0].flat[s] = 1
        goal[b, 0].flat[g] = 1
    return maps, start, goal


def _f32(x: np.ndarray) -> torch.Tensor:
    """float64 tensor of fp32-representable values, so that the product holds exactly what the reference holds."""
    return torch.from_numpy(np.asarray(x, np.float64).astype(np.float32).astype(np.float64))


def encoder_input(ref, maps, start, goal):
    """(the input the reference's encode() hands its encoder, encode()'s output), both from the reference's own code."""
    seen = []
    hook = ref.encoder.model.register_forward_pre_hook(lambda mod, args: seen.append(args[0]))
    try:
        with torch.no_grad():
            cost = ref.encode(maps, start, goal)
    finally:
        hook.remove()
    return seen[0], cost


def randomise_batchnorm(ref, x: torch.Tensor, rng: np.random.RandomState) -> None:
    """Give every BatchNorm of the float64 reference statistics far from the identity: running variances log-uniform over
    1e-3 .. 10 (eps = 1e-5 is 1 % of the smallest), gamma of both signs, beta != 0 and running means of either sign.
    gamma sets the folded scale s = gamma / sqrt(var + eps) to a log-uniform 0.3 .. 3 over the channel's rms on the
    calibration input x, and the running mean is half that rms times a normal draw: the activations stay of order one
    whatever the variance (so |gamma| ranges over about 0.01 .. 30), without cancelling most of the channel's mean, which
    would amplify every rounding of the convolution by the ratio of its mean to its spread.  The head's scale is 3 over
    its rms, so the costs are neither saturated nor flat.  Every value is fp32-representable."""
    with torch.no_grad():
        for m in ref.encoder.model:
            if isinstance(m, nn.BatchNorm2d):
                randomise_one_batchnorm(m, x, rng)
            x = m(x)


def randomise_one_batchnorm(m: nn.BatchNorm2d, x: torch.Tensor, rng: np.random.RandomState) -> None:
    """randomise_batchnorm's statistics for one BatchNorm whose input, on the calibration batch, is x."""
    with torch.no_grad():
        C = m.num_features
        rms = x.pow(2).mean((0, 2, 3)).sqrt().clamp_min(1e-3).cpu().numpy()
        var = 10.0 ** rng.uniform(-3, 1, C)
        scale = (3.0 if C == 1 else 10.0 ** rng.uniform(-0.5, 0.5, C)) / rms
        gamma = rng.choice([-1.0, 1.0], C) * scale * np.sqrt(var + m.eps)
        m.running_var.copy_(_f32(var))
        m.running_mean.copy_(_f32(0.5 * rms * rng.randn(C)))
        m.weight.copy_(_f32(gamma))
        m.bias.copy_(_f32(rng.randn(C) * 0.5))


def build_reference(ref_astar, cfg: Config, seed: int):
    """The reference's NeuralAstar of `cfg`, its weights drawn from `seed`, its BatchNorms randomised on a calibration
    batch of the configuration, in float64 and eval mode.  The convolutions keep the magnitudes of the reference's own
    initialisation, but 95 % of their weights are made positive (a trained encoder's filters are not sign-balanced
    either): with sign-balanced weights an element-wise worst-case bound grows by about sqrt(9 C) a layer against the
    activations it bounds, and says nothing at depth 3 or 4.  One weight in 20 stays negative, so that a kernel that
    lost a sign still fails."""
    with torch.random.fork_rng():
        torch.manual_seed(seed)
        ref = ref_astar.NeuralAstar(encoder_input=cfg.inp, encoder_arch=cfg.arch, encoder_depth=cfg.depth,
                                    learn_obstacles=cfg.learn_obstacles, const=cfg.const)
    rng = np.random.RandomState(seed % 2 ** 32)
    with torch.no_grad():
        for m in ref.encoder.model:
            if isinstance(m, nn.Conv2d):
                positive = torch.from_numpy(rng.rand(*m.weight.shape) < POSITIVE)
                m.weight.copy_(torch.where(positive, m.weight.abs(), -m.weight.abs()))
    ref = ref.double().eval()
    x, _ = encoder_input(ref, *(torch.from_numpy(a).double() for a in inputs(cfg, seed + 1)))
    randomise_batchnorm(ref, x, rng)
    return ref


def build_product(ref, cfg: Config):
    """The product's NeuralAstar of `cfg` holding the reference's state (fp32), in eval mode on the CPU."""
    from neural_astar.planner import NeuralAstar

    na = NeuralAstar(encoder_input=cfg.inp, encoder_arch=cfg.arch, encoder_depth=cfg.depth,
                     learn_obstacles=cfg.learn_obstacles, const=cfg.const)
    result = na.load_state_dict(ref.state_dict())
    assert not result.missing_keys and not result.unexpected_keys, result
    return na.eval()


# ------------------------------------------------------------------------------------------------- the bound
class Rounding(NamedTuple):
    u_op: float    # relative error of reading one operand: U_TF32 for TF32 operands, 0 for fp32
    K: int         # rounded fp32 additions (or FMAs) summed into one output, the bias included


def layer_rounding(cfg: Config, mode: str) -> List[Rounding]:
    """How the product evaluates each conv (+ BatchNorm) of `cfg` in `mode`:
      cpu     the module path on the CPU: fp32 convolutions with the bias added, BatchNorm after them;
      module  the module path on CUDA under autograd: cuDNN with torch's default TF32, the head conv included;
      tf32    the eval fast path (default): cuDNN TF32 convolutions (or the fused TF32 128 -> 256 kernel); conv1_marks
              for the "m+" CNN (18 fp32 FMAs onto the bias); the head as fp32 [C] x [C,9] products (head_taps, or
              torch.mm with the head kernel off) followed by the bias and 9 fp32 adds of the tap gather;
      fp32    the fast path with TF32 off: the same with fp32 cuDNN convolutions;
      nohead  the fast path with the head kernel off (torch.mm): rounds as tf32 does."""
    chans = [len(cfg.inp)] + CHANNELS[:cfg.depth] + [1]
    out = []
    for i, cin in enumerate(chans[:-1]):
        tf32 = U_TF32 if mode in ("module", "tf32", "nohead") else 0.0
        if mode in ("cpu", "module"):
            out.append(Rounding(tf32, 9 * cin + 1))
        elif i == cfg.depth:
            out.append(Rounding(0.0, cin + 9))
        elif i == 0 and cfg.conv1_marks:
            out.append(Rounding(0.0, 18))
        else:
            out.append(Rounding(tf32, 9 * cin + 1))
    return out


def gamma(K: int) -> float:
    """gamma_K = K u / (1 - K u): relative error bound of K rounded fp32 operations, in any order."""
    return K * U / (1 - K * U)


class Walk(NamedTuple):
    steps: List[Tuple[str, torch.Tensor, torch.Tensor]]   # (module, reference activation, element-wise error bound)
    cost: torch.Tensor                                    # the reference's cost maps, float64
    bound: torch.Tensor                                   # element-wise bound on |product cost - cost|


def reference_and_bound(ref, x: torch.Tensor, rounding: List[Rounding]) -> Walk:
    """Walk the float64 reference's nn.Sequential on its encoder input x, module by module, and carry an element-wise
    bound e on |product - reference| of each activation.  A Conv2d and its BatchNorm are one step (the product folds
    them, or rounds them as if it had: see below), recorded at the BatchNorm.

    conv + BatchNorm.  With s = gamma / sqrt(var + eps), the folded weights W = w s and bias b = (b_conv - mu) s + beta
    are exact in float64, and
        e_out = conv(e_in, |W|) + c * (conv(|a_in| + e_in, |W|) + |s| (|b_conv| + |mu|) + |beta|),
        c = (1 + FOLD) (1 + PROD(u_op)) (1 + gamma_K) - 1.
    Every product x w of the sum reads two operands each off by at most u_op relatively (PROD = 2 u_op + u_op^2, the
    convention of tests/test_gpu_convhead.py; 0 in fp32) and the sum rounds K times (gamma_K, any order).  FOLD: the
    fp32 fold computes eps, var + eps, the square root and the division (s off by at most 3.5 u), then w * s (W off by
    4.5 u) and ((b_conv - mu) * s) + beta (off by 7.5 u of |s| (|b_conv| + |mu|) + |beta|).  The module path rounds
    the unfolded BatchNorm ((y - mu) * invstd * gamma + beta, or y * alpha + (beta - mu * alpha)) in as many
    operations, with at most 4 u in a reciprocal square root; 10 u covers both.  The magnitude of the bias term is
    taken before mu cancels, so that the unfolded form, which subtracts mu after the convolution, is covered too.
    ReLU is 1-Lipschitz: e passes unchanged.  MaxPool: e_out = maxpool(e_in).

    sigmoid(x) * const.  sigmoid' <= 1/4, and the fp32 evaluation (expf at most 2 ulp = 4 u off as CUDA documents it,
    1 + E rounded, an IEEE division, the separately rounded product: nastar_common.cuh sigmoid_scaled, ATen's sigmoid)
    is off by at most 7 u relatively, 8 u with the second-order terms:
        bound = |const| (e / 4 + SIGMOID (sigmoid(a) + e / 4)).
    The float64 reference's own rounding (about 1e-16 relatively) is far below every term."""
    steps, e, K = [], torch.zeros_like(x), iter(rounding)
    mods = list(ref.encoder.model)
    a = x
    for i, m in enumerate(mods):
        if isinstance(m, nn.Conv2d):
            conv, bn = m, mods[i + 1]
            assert isinstance(bn, nn.BatchNorm2d) and conv.kernel_size == (3, 3) and conv.padding == (1, 1)
            r = next(K)
            with torch.no_grad():
                s = bn.weight / torch.sqrt(bn.running_var + bn.eps)
                Wabs = (conv.weight * s.view(-1, 1, 1, 1)).abs()
                bmag = s.abs() * (conv.bias.abs() + bn.running_mean.abs()) + bn.bias.abs()
                c = (1 + FOLD) * (1 + (PROD if r.u_op else 0.0)) * (1 + gamma(r.K)) - 1
                e = F.conv2d((1 + c) * e + c * a.abs(), Wabs, c * bmag, padding=1)
                a = bn(conv(a))
            continue
        if isinstance(m, nn.BatchNorm2d):
            steps.append((f"{i - 1}+{i} conv+bn", a, e))
            continue
        with torch.no_grad():
            a = m(a)
            if isinstance(m, nn.MaxPool2d):
                e = m(e)
            else:
                assert isinstance(m, nn.ReLU)
        steps.append((f"{i} {type(m).__name__}", a, e))
    assert next(K, None) is None
    const = ref.encoder.const
    k = float(abs(const)) if isinstance(const, float) else float(const.detach().abs())
    with torch.no_grad():
        sig = torch.sigmoid(a)
        cost = sig * const
    bound = k * (e / 4 + SIGMOID * (sig + e / 4))
    return Walk(steps, cost, bound)


def reference_case(ref, cfg: Config, maps, start, goal, mode: str) -> Walk:
    """The walk of the reference on the case's NumPy inputs, checked against the reference's own encode()."""
    x, cost = encoder_input(ref, *(torch.from_numpy(v).double() for v in (maps, start, goal)))
    walk = reference_and_bound(ref, x, layer_rounding(cfg, mode))
    assert torch.equal(walk.cost, cost), "the walk does not follow the reference's forward"
    return walk


def bound_ratio(got: np.ndarray, walk: Walk) -> float:
    """Worst |got - reference| / bound: the product is within the bound iff <= 1."""
    err = np.abs(got.astype(np.float64) - walk.cost.numpy())
    return float((err / walk.bound.numpy()).max())


# Largest median bound / median |cost - const / 2| allowed.  fp32 bounds stay below 0.003 of the spread over the whole
# matrix.  A TF32 bound is loose by construction: every layer adds 2^-9 of sum |x| |w| in the worst case, and that is
# carried through up to four more layers by |W|; the fast path's reaches 0.70 of the spread with the "m" CNN at depth
# 4 (its first conv reads TF32 operands too), cuDNN's TF32 module path 0.71.
VACUOUS_FP32 = 0.01
VACUOUS_TF32 = 1.0


def assert_not_vacuous(walk: Walk, const: float, what, frac: float) -> float:
    """The median bound is a fraction `frac` of the median |cost - const / 2| (the cost's distance from the sigmoid's
    midpoint) at most; returns that fraction."""
    spread = float((walk.cost - const / 2).abs().median())
    share = float(walk.bound.median()) / spread
    assert share < frac, (what, share)
    return share


def const_of(cfg: Config) -> float:
    return 1.0 if cfg.const is None else cfg.const


# ------------------------------------------------------------------------------------------------- the tests
WORST = {}          # (config id, mode) -> worst |error| / bound


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    for key in sorted(WORST):
        print(f"\nworst |error| / bound {key[0]} {key[1]}: {WORST[key]:.3f}")


@pytest.mark.parametrize("cfg", CONFIGS, ids=[c.id for c in CONFIGS])
def test_state_dicts_interchange(ref_astar, cfg):
    """The reference's float64 state dict loads into the product with every key matched, and the product's into a fresh
    reference; every value survives both ways."""
    ref = build_reference(ref_astar, cfg, cfg.seed)
    na = build_product(ref, cfg)
    for k, v in ref.state_dict().items():
        assert torch.equal(na.state_dict()[k].double(), v), k
    fresh = ref_astar.NeuralAstar(encoder_input=cfg.inp, encoder_arch=cfg.arch, encoder_depth=cfg.depth,
                                  learn_obstacles=cfg.learn_obstacles, const=cfg.const)
    result = fresh.load_state_dict(na.state_dict())
    assert not result.missing_keys and not result.unexpected_keys, result
    for k, v in na.state_dict().items():
        assert torch.equal(fresh.state_dict()[k], v), k


@pytest.mark.parametrize("cfg", CONFIGS, ids=[c.id for c in CONFIGS])
def test_module_path_within_fp32_bound(ref_astar, cfg):
    """The product's encode() in fp32 on the CPU against the float64 reference, element by element.  The bound is not
    vacuous, in its fp32 form or in its loosest one (TF32 operands in every layer)."""
    ref = build_reference(ref_astar, cfg, cfg.seed)
    na = build_product(ref, cfg)
    maps, start, goal = inputs(cfg, cfg.seed)
    with torch.no_grad():
        got = na.encode(*(torch.from_numpy(v) for v in (maps, start, goal))).numpy()
    walk = reference_case(ref, cfg, maps, start, goal, "cpu")
    ratio = bound_ratio(got, walk)
    WORST[(cfg.id, "cpu")] = ratio
    assert ratio <= 1.0, ratio
    assert_not_vacuous(walk, const_of(cfg), cfg.id, VACUOUS_FP32)
    assert_not_vacuous(reference_case(ref, cfg, maps, start, goal, "module"), const_of(cfg), cfg.id, VACUOUS_TF32)


def test_bound_holds_with_a_margin_on_the_largest_configuration(ref_astar):
    """Depth 4 on 64x64 maps: fp32 on the CPU stays under a quarter of the bound, so the bound is not tuned to the edge of
    what it bounds; the ratio is printed."""
    cfg = LARGEST
    ref = build_reference(ref_astar, cfg, cfg.seed)
    na = build_product(ref, cfg)
    maps, start, goal = inputs(cfg, cfg.seed)
    with torch.no_grad():
        got = na.encode(*(torch.from_numpy(v) for v in (maps, start, goal))).numpy()
    ratio = bound_ratio(got, reference_case(ref, cfg, maps, start, goal, "cpu"))
    print(f"\n{cfg.id}: worst |error| / fp32 bound on the CPU = {ratio:.4f}")
    assert ratio <= 0.25, ratio
