"""`pq_astar`: the search behind `use_differentiable_astar=False`, with the reference's signature
(/root/reference/src/neural_astar/planner/pq_astar.py:75-104).  CPU tensors in give CPU tensors out, CUDA in gives
CUDA out; the search itself always runs on the GPU (on the current CUDA device for CPU inputs).

Two semantics, chosen by the keyword-only `semantics` (the planners' `pq_semantics`):

* **"engine"** (default) — the dense GPU search of DifferentiableAstar with no step cap.  For uniform costs
  (VanillaAstar: cost == map design) its `histories` and `paths` equal the reference's heap A*, which is what the
  reference's own test pins (/root/reference/tests/astar_test.py:33-42, mirrored in tests/test_gpu_module_api.py).
  With learned costs it follows DifferentiableAstar's convention (cost of the SELECTED node, h + cost, ties by flat
  index, a passable cell is one != 0), so it expands different nodes than the reference's heap A*; a one-time warning
  is issued when a non-binary host cost map arrives.
* **"reference"** — the reference's `solve_single` exactly, on the GPU (csrc/nastar_pq.cuh, DESIGN.md §17): a heap A*
  charging the cost of the NEIGHBOUR entered, f_new = ((f_sel - (1-g) h(sel)) + g c[nb]) + (1-g) h(nb) in fp64 with
  h = max(dx, dy) + 0.001 * euclid (no cost term), a cell passable iff map == 1, ties decided by pqdict 1.2.0's heap
  moves, and all-zero `histories` and `paths` for a map whose goal is unreachable.  Two differences from the
  reference: the planes are read as fp32 (float64 costs are rounded to fp32 first), and g * c is always computed in
  fp64, as the reference's pinned NumPy 1 does (under NumPy >= 2 it would be fp32; the two agree whenever g * c is
  exact in fp32, which includes the default g_ratio 0.5).  `histories` take the goal maps' dtype and `paths` are
  int64, channel 0 of the goal maps' shape, as the reference returns.  A map whose start or goal plane does not have
  exactly one non-zero cell raises ValueError naming the maps (the reference's `.item()` raises there); to do so the
  call synchronises once.
"""
from __future__ import annotations

import warnings

import torch

from .. import _native
from .differentiable_astar import AstarOutput

PQ_SEMANTICS = ("engine", "reference")
_warned = False


def _check_semantics(semantics: str) -> None:
    if semantics not in PQ_SEMANTICS:
        raise ValueError(f"pq_astar semantics must be one of {list(PQ_SEMANTICS)} (got {semantics!r})")


def pq_astar(pred_costs, start_maps, goal_maps, map_designs, store_intermediate_results: bool = False,
             g_ratio: float = 0.5, *, semantics: str = "engine") -> AstarOutput:
    assert (
        store_intermediate_results == False  # noqa: E712
    ), "store_intermediate_results = True is currently supported only for differentiable A*"
    _check_semantics(semantics)
    if semantics == "reference":
        return _reference_pq_astar(pred_costs, start_maps, goal_maps, map_designs, g_ratio)
    return _engine_pq_astar(pred_costs, start_maps, goal_maps, map_designs, g_ratio)


def _reference_pq_astar(pred_costs, start_maps, goal_maps, map_designs, g_ratio: float) -> AstarOutput:
    src = pred_costs.device
    dev = src if src.type == "cuda" else torch.device("cuda", torch.cuda.current_device())
    args = [t.detach().to(dev, torch.float32) for t in (pred_costs, start_maps, goal_maps, map_designs)]
    hist, paths, status, _ = _native.pq_astar(*args, g_ratio)
    bad = torch.nonzero(status == _native.PQ_BAD_ENDS).flatten().tolist()
    if bad:
        raise ValueError(f"pq_astar: the start or goal map of map(s) {bad} does not have exactly one non-zero cell")
    shape = goal_maps.shape
    if shape[1] != 1:   # the reference fills channel 0 of arrays shaped like the goal maps
        hist = torch.cat((hist, hist.new_zeros((shape[0], shape[1] - 1) + tuple(shape[2:]))), 1)
        paths = torch.cat((paths, paths.new_zeros((shape[0], shape[1] - 1) + tuple(shape[2:]))), 1)
    return AstarOutput(hist.to(src, goal_maps.dtype), paths.to(src))


def _engine_pq_astar(pred_costs, start_maps, goal_maps, map_designs, g_ratio: float) -> AstarOutput:
    global _warned
    src = pred_costs.device
    dev = src if src.type == "cuda" else torch.device("cuda", torch.cuda.current_device())
    W = pred_costs.shape[-1]
    if not _warned and map_designs is not pred_costs and src.type == "cpu":
        # cheap only for host tensors; device inputs are not inspected (no sync on the hot path)
        c = pred_costs.detach()
        if bool(((c != 0) & (c != 1)).any()):
            _warned = True
            warnings.warn("pq_astar on the H100 engine follows DifferentiableAstar's cost convention (cost of the "
                          "selected node, h + cost); with non-uniform costs it differs from the reference's heap A* "
                          "— pass semantics=\"reference\" (pq_semantics= on the planners) for the reference's "
                          "results; see neural_astar/planner/pq_astar.py", stacklevel=3)
    args = [t.detach().to(dev, torch.float32) for t in (pred_costs, start_maps, goal_maps, map_designs)]
    if map_designs is pred_costs:
        args[3] = args[0]
    H = pred_costs.shape[-2]
    hist, paths, _, _, _ = _native.forward(*args, g_ratio, H * W, False)  # heap A* has no step cap
    return AstarOutput(hist.to(src), paths.to(src))
