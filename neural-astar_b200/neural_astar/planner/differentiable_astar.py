"""Differentiable A* — H100-native engine behind the reference's module surface.

Mirrors /root/reference/src/neural_astar/planner/differentiable_astar.py:
  AstarOutput (:16-23), get_heuristic (:26-52), DifferentiableAstar (:128-267).
The T-step Python loop (:203-252), `expand` (:77-93), `_st_softmax_noexp` (:55-74) and
`backtrack` (:96-125) do not exist here as Python: they run inside one persistent sm_90a kernel
per map batch (csrc/nastar_{warp32,warp64,bin16,generic}.cuh) reached through the C ABI in include/nastar_b200.h.
Autograd (only cost -> h -> f -> softmax -> histories is live in the reference, :237-243) is a
second kernel evaluating the closed form of SURVEY.md App. B.
"""
from __future__ import annotations

import contextvars
from typing import List, NamedTuple, Optional

import torch
import torch.nn as nn

from .. import _native
from .._native import check_steps


class AstarOutput(NamedTuple):
    """Output structure of A* search planners (reference :16-23)."""

    histories: torch.Tensor
    paths: torch.Tensor
    intermediate_results: Optional[List[dict]] = None


class SearchRecord(NamedTuple):
    """What the frames of a search are made of, handed out in place of the frame list while `recording_search` is on:
    T_batch is the batch-coupled step count, or None when the search exited per map."""

    histories: torch.Tensor
    paths: torch.Tensor
    goal_maps: torch.Tensor
    t_solve: torch.Tensor
    trace: torch.Tensor
    T: int
    T_batch: Optional[int]


# None: forward returns frames.  "batch": forward returns a SearchRecord of the search it runs.  "each": the same, and
# the batch is never coupled, so each map's record is that of the map searched alone.  Set by utils.data.search_gifs.
_recording = contextvars.ContextVar("recording_search", default=None)


def batch_coupled(g_ratio: float, B: int) -> bool:
    """Whether a batch of B maps is searched batch-coupled (the reference's loop, g_ratio < 0.5)."""
    return float(g_ratio) < 0.5 and B > 1 and _recording.get() != "each"


def get_heuristic(goal_maps: torch.Tensor, tb_factor: float = 0.001) -> torch.Tensor:
    """Chebyshev distance + tb_factor * Euclidean distance to the goal (reference :26-52).

    Kept for API compatibility (`DifferentiableAstar.get_heuristic`); the engine evaluates the same
    expression on-chip (csrc/nastar_common.cuh: heuristic()).
    """
    B, H, W = goal_maps.shape[0], goal_maps.shape[-2], goal_maps.shape[-1]
    flat = goal_maps.reshape(B, -1)
    ys = torch.arange(H, device=goal_maps.device, dtype=goal_maps.dtype).repeat_interleave(W)
    xs = torch.arange(W, device=goal_maps.device, dtype=goal_maps.dtype).repeat(H)
    gy = (flat * ys).sum(-1, keepdim=True)
    gx = (flat * xs).sum(-1, keepdim=True)
    dy, dx = (ys - gy).abs(), (xs - gx).abs()
    cheb = (dy + dx) - torch.minimum(dy, dx)
    euc = torch.sqrt(dy * dy + dx * dx)
    return (cheb + tb_factor * euc).reshape_as(goal_maps)


def get_news_heuristic(goal_maps: torch.Tensor, tb_factor: float = 0.001) -> torch.Tensor:
    """Manhattan distance + tb_factor * Euclidean distance to the goal: the planning-datasets generator's
    NorthEastWestSouth.get_heuristic (planning_datasets_utils/mechanism.py:124-131), for any H x W.

    `DifferentiableAstar(mechanism="news").get_heuristic`; the engine evaluates the same expression on-chip
    (csrc/nastar_common.cuh: heuristic_news()).
    """
    B, H, W = goal_maps.shape[0], goal_maps.shape[-2], goal_maps.shape[-1]
    flat = goal_maps.reshape(B, -1)
    ys = torch.arange(H, device=goal_maps.device, dtype=goal_maps.dtype).repeat_interleave(W)
    xs = torch.arange(W, device=goal_maps.device, dtype=goal_maps.dtype).repeat(H)
    gy = (flat * ys).sum(-1, keepdim=True)
    gx = (flat * xs).sum(-1, keepdim=True)
    dy, dx = (ys - gy).abs(), (xs - gx).abs()
    euc = torch.sqrt(dy * dy + dx * dx)
    return ((dy + dx) + tb_factor * euc).reshape_as(goal_maps)


def neighbor_filter_of(mechanism: str) -> torch.Tensor:
    """The 3x3 neighbour filter [1,1,3,3] of a mechanism: Moore = all but the centre (reference :139-143), NEWS = N,
    W, E, S (NorthEastWestSouth.get_neighbor_filter, mechanism.py:113-121)."""
    _check_mechanism(mechanism)
    if mechanism == "news":
        f = torch.zeros(1, 1, 3, 3)
        f[0, 0, 0, 1] = f[0, 0, 1, 0] = f[0, 0, 1, 2] = f[0, 0, 2, 1] = 1
    else:
        f = torch.ones(1, 1, 3, 3)
        f[0, 0, 1, 1] = 0
    return f


MECHANISMS = ("moore", "news")   # the planning-datasets generator's --mechanism values


def _check_mechanism(mechanism: str) -> None:
    if mechanism not in MECHANISMS:
        raise ValueError(f"mechanism must be one of {list(MECHANISMS)} (got {mechanism!r})")


def _mech_kw(mechanism: str) -> dict:
    """Keyword arguments of the _native search calls for a mechanism: none for Moore, the engine's default."""
    return {} if mechanism == "moore" else {"mechanism": mechanism}


class TakesMechanism(type):
    """Metaclass of the planners: `Planner(*args, mechanism="news", **kwargs)` runs __init__ with the other arguments,
    then `planner._select_mechanism(mechanism)`.  So the keyword-only `mechanism` ("moore", the default, or "news")
    exists while every __init__ keeps the reference's signature, which positional callers and checkpoint tooling rely
    on.  Any other value is a ValueError, raised before anything is built."""

    def __call__(cls, *args, mechanism: str = "moore", **kwargs):
        _check_mechanism(mechanism)
        planner = super().__call__(*args, **kwargs)
        if mechanism != "moore":
            planner._select_mechanism(mechanism)
        return planner


def _search(cost_maps, start_maps, goal_maps, obstacles_maps, g_ratio, T, want_trace, goal_clamped, mechanism,
            device_coupled):
    """The search of _AstarSearch.forward: (histories, paths, t_solve, n_steps, trace, T_batch, goal_clamp).
    goal_clamped is given only on the batch-coupled path (g_ratio < 0.5, see _coupled_steps): the search then runs
    exactly T steps per map.  device_coupled: the same batch coupling decided on the device (_native.forward_coupled, T
    is the cap), which returns T_batch and the goal clamp as device tensors (None otherwise)."""
    if device_coupled:
        hist, paths, t_solve, n_steps, T_batch, goal_clamp = _native.forward_coupled(
            cost_maps, start_maps, goal_maps, obstacles_maps, g_ratio, T, **_mech_kw(mechanism))
        return hist, paths, t_solve, n_steps, None, T_batch, goal_clamp
    no_early_exit = goal_clamped is not None
    hist, paths, t_solve, n_steps, trace = _native.forward(
        cost_maps, start_maps, goal_maps, obstacles_maps, g_ratio, T, want_trace, no_early_exit, **_mech_kw(mechanism))
    return hist, paths, t_solve, n_steps, trace, None, None


def _channel0_grad(grad_cost: torch.Tensor, cost: torch.Tensor) -> torch.Tensor:
    """dL/dcost for all of `cost`'s channels from the gradient of channel 0, the only one searched (:177)."""
    if grad_cost.shape != cost.shape:
        full = torch.zeros_like(cost)
        full[:, :1] = grad_cost
        grad_cost = full
    return grad_cost


class _AstarSearch(torch.autograd.Function):
    """forward: libnastar_b200 search; backward: closed-form dL/dcost kernel."""

    @staticmethod
    def forward(ctx, cost_maps, start_maps, goal_maps, obstacles_maps, g_ratio, T, want_trace, goal_clamped=None,
                mechanism="moore", device_coupled=False):
        # goal_clamped (host-coupled) and device_coupled: see _search.  The backward is told which goals were selected
        # more than once, and on the device route gets T_batch and the goal clamp as device tensors
        hist, paths, t_solve, n_steps, trace, T_batch, goal_clamp = _search(
            cost_maps, start_maps, goal_maps, obstacles_maps, g_ratio, T, want_trace, goal_clamped, mechanism,
            device_coupled)
        ctx.device_T_batch = T_batch
        ctx.g_ratio = g_ratio
        ctx.mechanism = mechanism
        ctx.T = T
        ctx.no_early_exit = no_early_exit = goal_clamped is not None
        if device_coupled:
            t_for_bwd = goal_clamp   # already the backward's encoding (include/nastar_b200.h, nastar_bwd_params)
        elif no_early_exit:
            # encoding understood by nastar_b200_backward: t_solve < T_batch-1  <=>  gradient blocked at the goal
            t_for_bwd = torch.where(goal_clamped, torch.zeros_like(t_solve), torch.full_like(t_solve, T))
        else:
            t_for_bwd = t_solve
        ctx.save_for_backward(cost_maps, start_maps, goal_maps, obstacles_maps, t_for_bwd, n_steps)
        ctx.mark_non_differentiable(paths, t_solve, n_steps)
        if trace is not None:
            ctx.mark_non_differentiable(trace)
        return hist, paths, t_solve, n_steps, trace

    @staticmethod
    def backward(ctx, grad_hist, *_unused):
        cost, start, goal, obst, t_solve, n_steps = ctx.saved_tensors
        grad_cost = None
        if ctx.needs_input_grad[0]:
            if ctx.device_T_batch is not None:
                T_batch = ctx.device_T_batch
            elif ctx.no_early_exit:   # the forward already ran exactly the reference's T_batch steps
                T_batch = torch.full((1,), ctx.T, dtype=torch.int32, device=cost.device)
            else:
                T_batch = _native.batch_steps(t_solve, n_steps, ctx.T)
            grad_cost = _native.backward(cost, start, goal, obst, grad_hist.contiguous(), T_batch, t_solve, ctx.g_ratio,
                                         **_mech_kw(ctx.mechanism))
            grad_cost = _channel0_grad(grad_cost, cost)
        return grad_cost, None, None, None, None, None, None, None, None, None


class _BlackboxSearch(torch.autograd.Function):
    """forward: _AstarSearch's search call, also keeping its histories; backward: the black-box gradient of Vlastelica
    et al. (ICLR 2020), (y(w + lam * dL/dhistories) - y(w)) / lam, from one more search on the perturbed costs
    (_native.backward_blackbox).  `T_cap` is the search's step bound; the forward's own T is T_batch on the host-coupled
    path.  `coupled`: the search on the perturbed costs is batch-coupled too, with its own T_batch decided on the
    device."""

    @staticmethod
    def forward(ctx, cost_maps, start_maps, goal_maps, obstacles_maps, g_ratio, T, want_trace, goal_clamped, mechanism,
                device_coupled, lam, T_cap, coupled):
        hist, paths, t_solve, n_steps, trace, _, _ = _search(
            cost_maps, start_maps, goal_maps, obstacles_maps, g_ratio, T, want_trace, goal_clamped, mechanism,
            device_coupled)
        ctx.lam, ctx.g_ratio, ctx.mechanism, ctx.T_cap, ctx.coupled = lam, g_ratio, mechanism, T_cap, coupled
        ctx.save_for_backward(cost_maps, start_maps, goal_maps, obstacles_maps, hist)
        ctx.mark_non_differentiable(paths, t_solve, n_steps)
        if trace is not None:
            ctx.mark_non_differentiable(trace)
        return hist, paths, t_solve, n_steps, trace

    @staticmethod
    def backward(ctx, grad_hist, *_unused):
        cost, start, goal, obst, hist = ctx.saved_tensors
        grad_cost = None
        if ctx.needs_input_grad[0]:
            grad_cost = _native.backward_blackbox(cost, start, goal, obst, hist, grad_hist.contiguous(), ctx.lam,
                                                  ctx.g_ratio, ctx.T_cap, coupled=ctx.coupled,
                                                  **_mech_kw(ctx.mechanism))
            grad_cost = _channel0_grad(grad_cost, cost)
        return (grad_cost,) + (None,) * 12


class DifferentiableAstar(nn.Module, metaclass=TakesMechanism):
    def __init__(self, g_ratio: float = 0.5, Tmax: float = 1.0):
        """
        Differentiable A* module (reference :129-148).

        Args:
            g_ratio: ratio between g(v) + h(v). Set 0 to perform as best-first search.
            Tmax: how much of the map the planner explores during training.
        Keyword-only (TakesMechanism):
            mechanism: "moore" (8-connected, Chebyshev heuristic, the reference's search) or "news" (4-connected,
                Manhattan heuristic: the planning-datasets generator's NorthEastWestSouth, for its *_news_* datasets).
                This keyword alone decides the search; `neighbor_filter` and `get_heuristic` are set to match it but
                are never read by the engine.
        """
        super().__init__()
        self.mechanism = "moore"
        # kept so that reference checkpoints load with "All keys matched" (state-dict key `astar.neighbor_filter`) and
        # a NEWS planner's state dict looks like a reference model given the generator's NEWS filter; the stencil
        # itself is compiled into the kernel and chosen by `mechanism`.
        self.neighbor_filter = nn.Parameter(neighbor_filter_of("moore"), requires_grad=False)
        self.get_heuristic = get_heuristic
        self.g_ratio = g_ratio
        assert (Tmax > 0) & (Tmax <= 1), "Tmax must be within (0, 1]"
        self.Tmax = Tmax

    def _select_mechanism(self, mechanism: str) -> None:
        self.mechanism = mechanism
        self.neighbor_filter.data = neighbor_filter_of(mechanism)
        self.get_heuristic = get_news_heuristic if mechanism == "news" else get_heuristic

    def num_steps(self, width: int) -> int:
        """Loop bound of the reference (:200-202): int(Tmax_eff * W * W), W = last dim."""
        Tmax = self.Tmax if self.training else 1.0
        return int(Tmax * width * width)

    def forward(
        self,
        cost_maps: torch.Tensor,
        start_maps: torch.Tensor,
        goal_maps: torch.Tensor,
        obstacles_maps: torch.Tensor,
        store_intermediate_results: bool = False,
    ) -> AstarOutput:
        assert cost_maps.ndim == 4
        assert start_maps.ndim == 4
        assert goal_maps.ndim == 4
        assert obstacles_maps.ndim == 4

        T = self.num_steps(cost_maps.shape[-1])
        if T < 1:
            raise ValueError("Tmax * W * W < 1: the reference loop would not execute (:203)")
        check_steps(T, f"the step bound int(Tmax * W * W) of a map of width W = {cost_maps.shape[-1]}")
        g_ratio = float(self.g_ratio)
        coupled = batch_coupled(g_ratio, cost_maps.shape[0])
        goal_clamped = None
        T_cap = T
        if coupled and cost_maps.is_cuda and torch.cuda.is_current_stream_capturing():
            # under CUDA-graph capture the host decision below cannot happen: decide T_batch on the device instead
            # (_native.forward_coupled, the same outputs and gradient); frames need the host procedure's trace
            if store_intermediate_results:
                raise ValueError("store_intermediate_results needs a host sync and cannot be captured")
            hist, paths, _, _, _ = self._apply_search(
                cost_maps, start_maps, goal_maps, obstacles_maps, g_ratio, T, False, None, True, T, coupled)
            return AstarOutput(hist, paths, [])
        if coupled:
            # For g_ratio < 0.5 a solved map does not necessarily keep re-selecting its goal (SURVEY App. A.4),
            # so the reference's batch-synchronous loop (:251-252) changes the outputs of already-solved maps.
            # Reproduce it: step every map without early exit, find the first step at which ALL maps select
            # their goal, and take the state after exactly that many steps.  (One host sync; the reference
            # synchronises every step.)
            T, goal_clamped = _coupled_steps(cost_maps, start_maps, goal_maps, obstacles_maps, g_ratio, T,
                                             self.mechanism)
        hist, paths, t_solve, n_steps, trace = self._apply_search(
            cost_maps, start_maps, goal_maps, obstacles_maps, g_ratio, T, bool(store_intermediate_results), goal_clamped,
            False, T_cap, coupled)

        intermediate_results: List[dict] = []
        if store_intermediate_results and _recording.get() is not None:
            intermediate_results = SearchRecord(hist, paths, goal_maps, t_solve, trace, T, T if coupled else None)
        elif store_intermediate_results:
            intermediate_results = _materialise_frames(hist, paths, goal_maps, t_solve, n_steps, trace, T,
                                                       T_batch=T if coupled else None)
        return AstarOutput(hist, paths, intermediate_results)


    def _apply_search(self, cost_maps, start_maps, goal_maps, obstacles_maps, g_ratio, T, want_trace, goal_clamped,
                      device_coupled, T_cap, coupled):
        """The autograd search of forward(): T is the step count the search runs (T_batch on the host-coupled path),
        T_cap the step bound int(Tmax * W * W), `coupled` whether the batch is searched batch-coupled."""
        if device_coupled:
            return _AstarSearch.apply(cost_maps, start_maps, goal_maps, obstacles_maps, g_ratio, T, want_trace,
                                      goal_clamped, self.mechanism, True)
        return _AstarSearch.apply(cost_maps, start_maps, goal_maps, obstacles_maps, g_ratio, T, want_trace, goal_clamped,
                                  self.mechanism)

    def search_from_taps(self, taps: torch.Tensor, bias: float, scale: float, start_maps: torch.Tensor,
                         goal_maps: torch.Tensor, obstacles_maps: torch.Tensor,
                         store_intermediate_results: bool = False) -> AstarOutput:
        """Inference-only entry of the fused encoder hand-off (SURVEY.md 8(f)-3): `taps` [B,H,W,9] are the
        partial products of the encoder's last 3x3 conv; the kernel prologue computes
        cost = sigmoid(bias + gather(taps)) * scale (encoder.py:32-34) and searches on it.  No autograd.
        A batch of more than one map with g_ratio < 0.5 is searched batch-coupled like `forward` (the reference's
        loop, :251-252), with T_batch decided on the device (_native.forward_coupled); it has no frames."""
        W = start_maps.shape[-1]
        T = self.num_steps(W)
        if batch_coupled(self.g_ratio, start_maps.shape[0]):
            if store_intermediate_results:
                raise ValueError("store_intermediate_results is not available for a batch-coupled search from taps "
                                 "(g_ratio < 0.5, more than one map): use forward() on the cost maps")
            hist, paths = _native.forward_coupled(
                taps, start_maps, goal_maps, obstacles_maps, float(self.g_ratio), T, cost_kind=_native.COST_TAPS,
                cost_scale=scale, cost_bias=bias, **_mech_kw(self.mechanism))[:2]
            return AstarOutput(hist, paths, [])
        hist, paths, t_solve, n_steps, trace = _native.forward(
            taps, start_maps, goal_maps, obstacles_maps, float(self.g_ratio), T, bool(store_intermediate_results),
            cost_kind=_native.COST_TAPS, cost_scale=scale, cost_bias=bias, **_mech_kw(self.mechanism))
        frames: List[dict] = []
        if store_intermediate_results and _recording.get() is not None:
            frames = SearchRecord(hist, paths, goal_maps, t_solve, trace, T, None)
        elif store_intermediate_results:
            frames = _materialise_frames(hist, paths, goal_maps, t_solve, n_steps, trace, T)
        return AstarOutput(hist, paths, frames)


class BlackboxAstar(DifferentiableAstar):
    """DifferentiableAstar whose gradient is the black-box one of BB-A* (_BlackboxSearch): the same forward, and in the
    backward one more search on the costs perturbed by `bbastar_lambda` times the incoming gradient.  Its state dict
    is DifferentiableAstar's; lambda is an attribute, not a buffer."""

    def __init__(self, g_ratio: float = 0.5, Tmax: float = 1.0, bbastar_lambda: float = 20.0):
        super().__init__(g_ratio=g_ratio, Tmax=Tmax)
        self.bbastar_lambda = _native.check_lambda(bbastar_lambda)

    def _apply_search(self, cost_maps, start_maps, goal_maps, obstacles_maps, g_ratio, T, want_trace, goal_clamped,
                      device_coupled, T_cap, coupled):
        return _BlackboxSearch.apply(cost_maps, start_maps, goal_maps, obstacles_maps, g_ratio, T, want_trace,
                                     goal_clamped, self.mechanism, device_coupled, self.bbastar_lambda, T_cap, coupled)


def _coupled_steps(cost_maps, start_maps, goal_maps, obstacles_maps, g_ratio: float, T: int, mechanism: str = "moore"):
    """(T_batch, goal_clamped[B]) for g_ratio < 0.5: the number of iterations the reference's loop executes when
    solved maps keep evolving, and per map whether its goal is selected more than once within them — then
    clamp(hist + sel) saw 2 at the goal and blocks its gradient (differentiable_astar.py:222-223)."""
    with torch.no_grad():
        _, _, _, _, trace = _native.forward(cost_maps, start_maps, goal_maps, obstacles_maps, g_ratio, T,
                                            want_trace=True, no_early_exit=True, **_mech_kw(mechanism))
        B = goal_maps.shape[0]
        goal_idx = goal_maps[:, 0].reshape(B, -1).argmax(-1).to(trace.dtype)
        at_goal = trace == goal_idx[:, None]
        all_at_goal = at_goal.all(0)
        first = torch.where(all_at_goal.any(), all_at_goal.float().argmax() + 1, torch.tensor(T, device=trace.device))
        T_batch = int(first.item())
        goal_clamped = at_goal[:, :T_batch].sum(1) >= 2
    return T_batch, goal_clamped


def _materialise_frames(hist, paths, goal_maps, t_solve, n_steps, trace, T, T_batch=None) -> List[dict]:
    """Rebuild the reference's per-step frames (:210-216, :257-263) from the selection trace.

    Frame t holds the closed set BEFORE step t and the node selected AT step t; the reference keeps
    stepping every map until the slowest one is solved, re-selecting the goal (App. A.4), so
    post-solve frames repeat the goal.  One host sync (T_batch) is inherent to returning a list.
    """
    B, _, H, W = hist.shape
    N = H * W
    if T_batch is None:
        T_batch = int(_native.batch_steps(t_solve, n_steps, T).item())
    goal_idx = goal_maps[:, 0].reshape(B, -1).argmax(-1)
    tr = trace[:, :T_batch].to(torch.int64)
    tr = torch.where(tr < 0, goal_idx[:, None].expand_as(tr), tr)
    sel = torch.zeros((T_batch, B, N), dtype=hist.dtype, device=hist.device)
    sel.scatter_(2, tr.t().unsqueeze(-1), 1.0)
    closed_before = (sel.cumsum(0) - sel).clamp_(0, 1)
    frames = [
        {"histories": closed_before[t].reshape(B, 1, H, W), "paths": sel[t].reshape(B, 1, H, W)}
        for t in range(T_batch)
    ]
    frames.append({"histories": hist.detach(), "paths": paths.detach()})
    return frames
