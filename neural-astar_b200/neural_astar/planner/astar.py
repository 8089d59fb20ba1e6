"""VanillaAstar / NeuralAstar — the reference's nn.Module API on top of the H100 search engine.

API contract mirrored from /root/reference/src/neural_astar/planner/astar.py (:17-102 VanillaAstar,
:105-213 NeuralAstar): constructor keywords, the `.astar` / `.encoder` attributes, `encode()`,
`perform_astar()` and `forward()` returning `AstarOutput`.  `use_differentiable_astar=False` selects
`pq_astar`, the reference's heap A*: by default served by the dense GPU search (identical for uniform costs, which is
what the reference's own test pins, tests/astar_test.py:33-42), or with `pq_semantics="reference"` by a GPU heap A*
that reproduces the reference's results for any costs; see planner/pq_astar.py.

Inference hand-off (SURVEY.md 8(f)-3): in eval / no-grad mode on CUDA, `NeuralAstar.forward` runs
the input assembly (start+goal add, nearest upsample, concat, NHWC) as one kernel — folded into the first
convolution for the "m+" CNN (`conv1_marks`), a separate `pack_inputs` otherwise -> the encoder's cuDNN convs ->
the head's per-pixel products (`head_taps`) -> the search kernel, whose prologue finishes the encoder (9-tap
gather + bias, sigmoid, * const: encoder.py:32-34) — no ATen glue launches in between.
"""
from __future__ import annotations

from typing import Optional

import torch
import torch.nn as nn
import torch.nn.functional as F

from .. import _native
from . import encoder as _encoders
from .differentiable_astar import AstarOutput, BlackboxAstar, DifferentiableAstar, TakesMechanism, _mech_kw, batch_coupled
from .pq_astar import _check_semantics, pq_astar  # noqa: F401  pq_astar re-exported, like the reference module does


class TakesPlannerKeywords(TakesMechanism):
    """Metaclass of the planners: TakesMechanism's route for one more keyword-only argument, `pq_semantics` ("engine",
    the default, or "reference"): the semantics of `pq_astar` when `use_differentiable_astar=False` (see
    planner/pq_astar.py).  Every __init__ keeps the reference's signature.  An unknown value is a ValueError raised
    before anything is built; "reference" with `use_differentiable_astar=True` is a ValueError too, since it would
    select nothing."""

    def __call__(cls, *args, pq_semantics: str = "engine", **kwargs):
        _check_semantics(pq_semantics)
        planner = super().__call__(*args, **kwargs)
        if pq_semantics != "engine" and planner.use_differentiable_astar:
            raise ValueError(f"pq_semantics={pq_semantics!r} applies to use_differentiable_astar=False only")
        planner.pq_semantics = pq_semantics
        return planner


class VanillaAstar(nn.Module, metaclass=TakesPlannerKeywords):
    """A* on the given map: cost == obstacles == map design (reference :93-94).

    Keyword-only `mechanism` = "moore" (default, 8-connected) or "news" (4-connected with the Manhattan heuristic, for
    the planning-datasets generator's NEWS datasets); see DifferentiableAstar.  Keyword-only `pq_semantics` =
    "engine" (default) or "reference" (the reference's heap A* exactly), for `use_differentiable_astar=False`; see
    planner/pq_astar.py.

    >>> out = VanillaAstar()(map_designs, start_maps, goal_maps)   # out.histories, out.paths
    """

    def __init__(self, g_ratio: float = 0.5, use_differentiable_astar: bool = True):
        super().__init__()
        self._configure_search(g_ratio, 1.0, use_differentiable_astar)

    def _configure_search(self, g_ratio: float, Tmax: float, use_differentiable_astar: bool) -> None:
        self.astar = DifferentiableAstar(g_ratio=g_ratio, Tmax=Tmax)
        self.g_ratio = g_ratio
        self.use_differentiable_astar = use_differentiable_astar
        self.pq_semantics = "engine"

    def _select_mechanism(self, mechanism: str) -> None:
        if not self.use_differentiable_astar:
            raise NotImplementedError("pq_astar (use_differentiable_astar=False) searches Moore neighbourhoods only")
        self.astar._select_mechanism(mechanism)

    def perform_astar(self, map_designs: torch.Tensor, start_maps: torch.Tensor, goal_maps: torch.Tensor,
                      obstacles_maps: torch.Tensor, store_intermediate_results: bool = False) -> AstarOutput:
        """Positional contract of the seam (reference :48-71): (cost, start, goal, obstacles, store)."""
        if self.use_differentiable_astar:
            return self.astar(map_designs, start_maps, goal_maps, obstacles_maps, store_intermediate_results)
        return pq_astar(map_designs, start_maps, goal_maps, obstacles_maps, store_intermediate_results,
                        g_ratio=self.g_ratio, semantics=self.pq_semantics)

    def forward(self, map_designs: torch.Tensor, start_maps: torch.Tensor, goal_maps: torch.Tensor,
                store_intermediate_results: bool = False) -> AstarOutput:
        # the same tensor is passed as cost and as obstacles; the engine notices the alias and reads it once
        return self.perform_astar(map_designs, start_maps, goal_maps, map_designs, store_intermediate_results)


class NeuralAstar(VanillaAstar):
    """Neural A*: an encoder predicts the cost map, the differentiable search runs on it (reference :105-213).

    Args (same names and defaults as the reference):
        g_ratio: weight of g(v) against h(v); 0 = best-first.
        Tmax: fraction of W*W steps explored in training mode (use 0.25 when training).
        encoder_input: "m" = map only, "m+" = map + (start+goal) channel, "rgb+" = RGB + that channel.
        encoder_arch: class name in `planner.encoder` ("CNN", "CNNDownSize", "Unet").
        encoder_depth: number of conv blocks.
        learn_obstacles: hide the obstacle map from the search (all cells passable).
        const: learnable multiplier on the predicted cost (None = 1).
        use_differentiable_astar: False runs `pq_astar`, see module docstring.
        mechanism (keyword-only): "moore" (default) or "news": the search's neighbourhood and heuristic, see
            DifferentiableAstar.
        pq_semantics (keyword-only): "engine" (default) or "reference": which `pq_astar` runs when
            use_differentiable_astar is False, see planner/pq_astar.py.
    """

    def __init__(self, g_ratio: float = 0.5, Tmax: float = 1.0, encoder_input: str = "m+", encoder_arch: str = "CNN",
                 encoder_depth: int = 4, learn_obstacles: bool = False, const: Optional[float] = None,
                 use_differentiable_astar: bool = True):
        super().__init__()
        self._configure_search(g_ratio, Tmax, use_differentiable_astar)
        self.encoder_input = encoder_input
        self.encoder = getattr(_encoders, encoder_arch)(len(encoder_input), encoder_depth, const)
        self.learn_obstacles = learn_obstacles
        if learn_obstacles:
            print("WARNING: learn_obstacles has been set to True")

    def encode(self, map_designs: torch.Tensor, start_maps: torch.Tensor, goal_maps: torch.Tensor) -> torch.Tensor:
        """Cost maps from the encoder; with a "+" input the start/goal marks ride along as an extra channel,
        nearest-upsampled when the image is larger than the planning grid (reference :154-180)."""
        return self._cost(self._head_taps(map_designs, start_maps, goal_maps), map_designs, start_maps, goal_maps)

    def _cost(self, head, map_designs: torch.Tensor, start_maps: torch.Tensor, goal_maps: torch.Tensor) -> torch.Tensor:
        """Cost maps from _head_taps()'s result (the same arithmetic as the search's TAPS prologue), or from the
        module path when there is none."""
        if head is not None:
            return _native.cost_from_taps(*head)
        return self.encoder(self._encoder_input(map_designs, start_maps, goal_maps))

    def _encoder_input(self, map_designs: torch.Tensor, start_maps: torch.Tensor, goal_maps: torch.Tensor) -> torch.Tensor:
        if "+" not in self.encoder_input:
            return map_designs
        marks = start_maps + goal_maps
        if marks.shape[-1] != map_designs.shape[-1]:
            marks = F.interpolate(marks, size=map_designs.shape[-2:], mode="nearest")
        return torch.cat((map_designs, marks), dim=1)

    def _head_taps(self, map_designs: torch.Tensor, start_maps: torch.Tensor, goal_maps: torch.Tensor, out=None,
                   on_last_conv=None):
        """The eval fast path from the un-assembled inputs to the 9-tap products of the encoder's head
        (EncoderBase.head_taps): the "m+" CNN reads the three planes in its first layer's kernel, other "+" encoders
        get them packed by one kernel.  None when the fast path does not apply: training, autograd, inputs other than
        fp32 CUDA, or an encoder the plan cannot fold."""
        if not self.encoder.fast_path_ok(map_designs):
            return None
        if "+" not in self.encoder_input:
            return self.encoder.head_taps(map_designs, out=out, on_last_conv=on_last_conv)
        if not (start_maps.is_cuda and start_maps.dtype == torch.float32):
            return None
        head = self.encoder.head_taps_marks(map_designs, start_maps, goal_maps, out=out, on_last_conv=on_last_conv)
        if head is None:
            head = self.encoder.head_taps(_native.pack_inputs(map_designs, start_maps, goal_maps), out=out,
                                          on_last_conv=on_last_conv)
        return head

    @staticmethod
    def _searchable(head, start_maps: torch.Tensor) -> bool:
        """The search's TAPS prologue can read these taps: fp32 CUDA marks on the taps' grid, at most
        TAPS_MAX_SIDE on a side."""
        H, W = start_maps.shape[-2:]
        return (head is not None and start_maps.is_cuda and start_maps.dtype == torch.float32
                and tuple(head[0].shape[1:3]) == (H, W) and H <= _native.TAPS_MAX_SIDE and W <= _native.TAPS_MAX_SIDE)

    def forward(self, map_designs: torch.Tensor, start_maps: torch.Tensor, goal_maps: torch.Tensor,
                store_intermediate_results: bool = False) -> AstarOutput:
        """In eval mode without autograd the encoder runs once, up to its head's 9-tap products.  The search kernel
        consumes them directly (NASTAR_COST_TAPS), so no cost plane, sigmoid, bias add or layout conversion is
        launched, unless the taps do not fit its prologue or the search does not take them: pq_astar, and g_ratio < 0.5
        batches outside CUDA-graph capture, which keep the host procedure of DifferentiableAstar.forward (under capture
        search_from_taps couples the batch on the device).  Those search the cost plane of the same taps."""
        passable = torch.ones_like(start_maps) if self.learn_obstacles else map_designs
        head = self._head_taps(map_designs, start_maps, goal_maps)
        if (self._searchable(head, start_maps) and self.use_differentiable_astar and passable.dtype == torch.float32
                and (not batch_coupled(self.g_ratio, start_maps.shape[0]) or torch.cuda.is_current_stream_capturing())):
            return self.astar.search_from_taps(*head, start_maps, goal_maps, passable, store_intermediate_results)
        cost_maps = self._cost(head, map_designs, start_maps, goal_maps)
        return self.perform_astar(cost_maps, start_maps, goal_maps, passable, store_intermediate_results)

    def forward_pair(self, map_designs: torch.Tensor, start_maps: torch.Tensor, goal_maps: torch.Tensor,
                     vanilla_g_ratio: float = 0.5):
        """Validation pair (reference utils/training.py:63-87) in one search launch: returns
        (outputs of this planner, outputs of VanillaAstar on the same batch with this planner's mechanism,
        (n_closed [2B], path_len [2B]))
        or None when the single-launch form does not apply (autograd on, CPU tensors, learn_obstacles, different
        g_ratio for the baseline, g_ratio < 0.5 batches, pq_astar).  Inference only."""
        B = start_maps.shape[0]
        if (torch.is_grad_enabled() or not start_maps.is_cuda or self.learn_obstacles or map_designs.shape[1] != 1
                or not self.use_differentiable_astar or float(vanilla_g_ratio) != float(self.g_ratio)
                or (float(self.g_ratio) < 0.5 and B > 1) or map_designs.shape[-2:] != start_maps.shape[-2:]
                or map_designs.dtype != torch.float32 or start_maps.dtype != torch.float32):
            return None
        T = self.astar.num_steps(start_maps.shape[-1])
        kw = _mech_kw(self.astar.mechanism)
        head = self._head_taps(map_designs, start_maps, goal_maps)
        if self._searchable(head, start_maps):
            cost, bias, scale = head
            kw.update(cost_kind=_native.COST_TAPS, cost_bias=bias, cost_scale=scale)
        else:
            cost = self._cost(head, map_designs, start_maps, goal_maps)
        hist, paths, _, _, _, counts = _native.forward(cost, start_maps, goal_maps, map_designs, float(self.g_ratio), T,
                                                       pair=True, want_counts=True, **kw)
        return (AstarOutput(hist[:B], paths[:B], []), AstarOutput(hist[B:], paths[B:], []), tuple(counts))


class BBAstar(NeuralAstar):
    """BB-A*: Neural A*'s encoder trained through a non-differentiable A*, with the black-box gradient of Vlastelica
    et al., "Differentiation of Blackbox Combinatorial Solvers" (ICLR 2020).  The learned baseline that the Neural A*
    paper (Yonetani et al., ICML 2021) sets against Neural A*.

    The forward is NeuralAstar's, output for output.  The backward takes the incoming gradient g = dL/dhistories,
    searches again on the perturbed costs w' = fl(w + fl(lambda * g)) (same g_ratio, step bound, mechanism and
    obstacles; w' may be negative) and returns dL/dcost = (histories(w') - histories(w)) / lambda, every cell 0 or
    +-fl(1/lambda); only channel 0 of a multi-channel cost gets a gradient.  Below g_ratio 0.5 a batch of more than one
    map is searched batch-coupled in both searches, each with its own T_batch decided on the device.  The backward is
    one search launch (three when coupled) and never synchronises with the host, so GraphedTrainStep captures it.

    The default bbastar_lambda = 20.0 is the value Vlastelica et al. use in their shortest-path experiments, and the
    formula follows the two papers.  Neither is checked against the Neural A* authors' own BB-A* code, which is not
    part of the reference this project follows.

    Args: NeuralAstar's, plus
        bbastar_lambda: the interpolation strength lambda, a finite float32 > 0 (ValueError otherwise).
    use_differentiable_astar=False is a ValueError: pq_astar has no black-box gradient.  The state dict is
    NeuralAstar's key for key (lambda is not a buffer), so checkpoints load either way.
    """

    def __init__(self, g_ratio: float = 0.5, Tmax: float = 1.0, encoder_input: str = "m+", encoder_arch: str = "CNN",
                 encoder_depth: int = 4, learn_obstacles: bool = False, const: Optional[float] = None,
                 use_differentiable_astar: bool = True, bbastar_lambda: float = 20.0):
        if not use_differentiable_astar:
            raise ValueError("BBAstar needs use_differentiable_astar=True: pq_astar has no black-box gradient")
        astar = BlackboxAstar(g_ratio=g_ratio, Tmax=Tmax, bbastar_lambda=bbastar_lambda)
        super().__init__(g_ratio, Tmax, encoder_input, encoder_arch, encoder_depth, learn_obstacles, const,
                         use_differentiable_astar)
        self.astar = astar

    @property
    def bbastar_lambda(self) -> float:
        return self.astar.bbastar_lambda
