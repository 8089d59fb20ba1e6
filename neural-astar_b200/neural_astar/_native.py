"""ctypes binding of libnastar_b200.so (C ABI declared in include/nastar_b200.h).

PyTorch is used here only for device memory and the current CUDA stream; the library itself
has no torch dependency.  Loading fails loudly when the library is missing: the product has no
CPU or eager-PyTorch fallback for the search.
"""
from __future__ import annotations

import contextlib
import ctypes
import math
import os
from typing import Optional, Tuple

import numpy as np
import torch

_PKG_ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))  # neural-astar_b200/
LIB_PATH = os.environ.get("NASTAR_B200_LIB", os.path.join(_PKG_ROOT, "lib", "libnastar_b200.so"))

ABI_VERSION = 4
NASTAR_OK = 0
TS_CAPPED = -1
TS_EXHAUSTED = -2


class FwdParams(ctypes.Structure):
    """struct nastar_fwd_params (include/nastar_b200.h)"""

    _fields_ = [
        ("cost", ctypes.c_void_p), ("cost_stride", ctypes.c_int64),
        ("start", ctypes.c_void_p), ("start_stride", ctypes.c_int64),
        ("goal", ctypes.c_void_p), ("goal_stride", ctypes.c_int64),
        ("obst", ctypes.c_void_p), ("obst_stride", ctypes.c_int64),
        ("B", ctypes.c_int32), ("H", ctypes.c_int32), ("W", ctypes.c_int32),
        ("g_ratio", ctypes.c_float), ("one_minus_g_ratio", ctypes.c_float),
        ("T", ctypes.c_int32), ("flags", ctypes.c_int32),
        ("cost_kind", ctypes.c_int32), ("cost_scale", ctypes.c_float), ("cost_bias", ctypes.c_float),
        ("histories", ctypes.c_void_p), ("paths", ctypes.c_void_p),
        ("t_solve", ctypes.c_void_p), ("n_steps", ctypes.c_void_p), ("trace", ctypes.c_void_p),
        ("n_closed", ctypes.c_void_p), ("path_len", ctypes.c_void_p),
        ("workspace", ctypes.c_void_p), ("workspace_bytes", ctypes.c_size_t),
    ]


class BwdParams(ctypes.Structure):
    """struct nastar_bwd_params (include/nastar_b200.h)"""

    _fields_ = [
        ("cost", ctypes.c_void_p), ("cost_stride", ctypes.c_int64),
        ("start", ctypes.c_void_p), ("start_stride", ctypes.c_int64),
        ("goal", ctypes.c_void_p), ("goal_stride", ctypes.c_int64),
        ("obst", ctypes.c_void_p), ("obst_stride", ctypes.c_int64),
        ("B", ctypes.c_int32), ("H", ctypes.c_int32), ("W", ctypes.c_int32),
        ("g_ratio", ctypes.c_float), ("one_minus_g_ratio", ctypes.c_float), ("sqrt_w", ctypes.c_float),
        ("T_batch", ctypes.c_void_p), ("t_solve", ctypes.c_void_p),
        ("grad_histories", ctypes.c_void_p), ("grad_stride", ctypes.c_int64),
        ("grad_cost", ctypes.c_void_p),
        ("workspace", ctypes.c_void_p), ("workspace_bytes", ctypes.c_size_t),
    ]


class GifParams(ctypes.Structure):
    """struct nastar_gif_params (include/nastar_b200.h)"""

    _fields_ = [
        ("maps", ctypes.c_void_p), ("histories", ctypes.c_void_p), ("paths", ctypes.c_void_p),
        ("goal_maps", ctypes.c_void_p), ("trace", ctypes.c_void_p), ("t_solve", ctypes.c_void_p),
        ("B", ctypes.c_int32), ("H", ctypes.c_int32), ("W", ctypes.c_int32), ("T", ctypes.c_int32),
        ("layout", ctypes.c_int32), ("steps_mode", ctypes.c_int32),
        ("screen_w", ctypes.c_int32), ("screen_h", ctypes.c_int32), ("delay_cs", ctypes.c_int32),
        ("tables", ctypes.c_void_p),
    ]


_p, _i32, _i64, _int = ctypes.c_void_p, ctypes.c_int32, ctypes.c_int64, ctypes.c_int

# every entry point of include/nastar_b200.h: symbol -> (restype, argtypes)
_SIGNATURES = {
    "nastar_b200_abi_version": (_int, []),
    "nastar_b200_forward_workspace_bytes": (ctypes.c_size_t, [_i32] * 3),
    "nastar_b200_backward_workspace_bytes": (ctypes.c_size_t, [_i32] * 3),
    "nastar_b200_forward": (_int, [ctypes.POINTER(FwdParams), _p]),
    "nastar_b200_forward_coupled_workspace_bytes": (ctypes.c_size_t, [_i32] * 4),
    "nastar_b200_forward_coupled": (_int, [ctypes.POINTER(FwdParams), _p, _p, _p]),
    "nastar_b200_backward": (_int, [ctypes.POINTER(BwdParams), _p]),
    "nastar_b200_backward_mech": (_int, [ctypes.POINTER(BwdParams), _i32, _p]),
    "nastar_b200_backward_blackbox": (_int, [ctypes.POINTER(FwdParams), _p, _p, _i64, ctypes.c_float, _p, _p, _p, _p]),
    "nastar_b200_batch_steps": (_int, [_p, _p, _i32, _i32, _p, _p]),
    "nastar_b200_engine_for": (_int, [_i32, _i32]),
    "nastar_b200_bin16_supported": (_int, [_i32, _i32]),
    "nastar_b200_pack_inputs": (_int, [_p, _i32, _i32, _i32, _p, _i64, _p, _i64, _i32, _i32, _i32, _p, _p]),
    "nastar_b200_cost_from_taps": (_int, [_p, _i32, _i32, _i32, ctypes.c_float, ctypes.c_float, _p, _p]),
    "nastar_b200_head_taps": (_int, [_p, _i64, _i32, _p, _p, _p]),
    "nastar_b200_conv1_marks": (_int, [_p, _p, _i64, _p, _i64, _i32, _i32, _i32, _p, _p, _p, _p]),
    "nastar_b200_conv3x3_head_taps": (_int, [_p] + [_i32] * 5 + [_p] * 5),
    "nastar_b200_upsample_concat": (_int, [_p] + [_i32] * 4 + [_p, _i32, _p, _p]),
    "nastar_b200_selftest_sqrt": (_int, [_i32, _p, _p]),
    "nastar_b200_opt_labels": (_int, [_p, _i64, _p, _i32, _i32, _i32, _p, _p, _p, _p]),
    "nastar_b200_opt_labels_mech": (_int, [_p, _i64, _p, _i32, _i32, _i32, _i32, _p, _p, _p, _p]),
    "nastar_b200_weighted_labels": (_int, [_p, _i64, _p, _i64] + [_p] * 2 + [_i32] * 3 + [_p] * 8),
    "nastar_b200_weighted_labels_mech": (_int, [_p, _i64, _p, _i64] + [_p] * 2 + [_i32] * 4 + [_p] * 8),
    "nastar_b200_sampler_prepare": (_int, [_p] * 3 + [_i32] * 3 + [ctypes.c_double] * 4 + [_p] * 7),
    "nastar_b200_sampler_sample": (_int, [_p] * 2 + [_i32] * 3 + [_p] * 6 + [_i32] * 2 + [_p] * 5),
    "nastar_b200_sample_goals": (_int, [_p, _i64] + [_i32] * 4 + [_p] * 5),
    "nastar_b200_maps_from_images": (_int, [_p, _i64] + [_i32] * 5 + [_p] * 5),
    "nastar_b200_draw_policies": (_int, [_p, _p, _i32, _i32, _p, _p]),
    "nastar_b200_decode_png": (_int, [_p, _i64, _p, _p, _i32, _p, _i64, _p, _p, ctypes.c_size_t, _p]),
    "nastar_b200_decode_png_workspace_bytes": (ctypes.c_size_t, [_p, _i32]),
    "nastar_b200_pq_astar": (_int, [_p, _i64] * 4 + [_i32] * 3 + [ctypes.c_double] + [_p] * 5
                             + [ctypes.c_size_t, _p]),
    "nastar_b200_pq_astar_workspace_bytes": (ctypes.c_size_t, [_i32] * 3),
    "nastar_b200_deflate": (_int, [_p, _p, _i32, _p, _i64, _p, _p, _p, _p, ctypes.c_size_t, _p]),
    "nastar_b200_deflate_bound": (_i64, [_p, _i32]),
    "nastar_b200_deflate_workspace_bytes": (ctypes.c_size_t, [_p, _i32]),
    "nastar_b200_png_filter": (_int, [_p, _p, _i32, _p, _i64, _p, _p]),
    "nastar_b200_png_finish": (_int, [_p, _p, _i32, _p, _p, _p, _p, _i64, _p]),
    "nastar_b200_png_gap": (_i64, [_i32]),
    "nastar_b200_png_encode_bound": (_i64, [_p, _i32]),
    "nastar_b200_crop_resize_rgb": (_int, [_p, _p, _i32, _p, _p] + [_i32] * 3 + [_p, _p]),
    "nastar_b200_inflate": (_int, [_p, _i64, _p, _p, _i32, _p, _i64, _p, _p, _p, ctypes.c_size_t, _p]),
    "nastar_b200_chamfer": (_int, [_p] + [_i32] * 3 + [_p, _p, ctypes.c_size_t, _p]),
    "nastar_b200_chamfer_workspace_bytes": (ctypes.c_size_t, [_i32] * 3),
    "nastar_b200_gif_tables_bytes": (_i64, [ctypes.POINTER(GifParams)]),
    "nastar_b200_gif_plan": (_int, [ctypes.POINTER(GifParams), _p, _p, _p, ctypes.c_size_t, _p]),
    "nastar_b200_gif_record_bytes": (_i64, [_i64]),
    "nastar_b200_gif_encode": (_int, [ctypes.POINTER(GifParams), _p, _p, _p, _p, _i64, _p, _i64, _p, ctypes.c_size_t,
                                      _p]),
    "nastar_b200_gif_workspace_bytes": (ctypes.c_size_t, [ctypes.POINTER(GifParams)]),
    "nastar_b200_launch_count": (ctypes.c_uint64, []),
    "nastar_b200_status_string": (ctypes.c_char_p, [_int]),
    "nastar_b200_last_cuda_error": (ctypes.c_char_p, []),
}
EXPORTS = tuple(_SIGNATURES)

_lib = None
_ws_cache = {}
_coupled_ws_cache = {}


class NativeLibraryMissing(ImportError):
    pass


def lib():
    """Load the engine. Raises NativeLibraryMissing (never falls back) if it is not built."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise NativeLibraryMissing(
            f"{LIB_PATH} not found: build the sm_90a engine first "
            "(python -c 'import __graft_entry__ as g; g.build()' or make -C neural-astar_b200). "
            "neural_astar (H100) has no CPU fallback."
        )
    L = ctypes.CDLL(LIB_PATH)
    for name, (restype, argtypes) in _SIGNATURES.items():
        fn = getattr(L, name)
        fn.restype, fn.argtypes = restype, argtypes
    if L.nastar_b200_abi_version() != ABI_VERSION:
        raise ImportError(f"{LIB_PATH}: ABI {L.nastar_b200_abi_version()} != expected {ABI_VERSION}")
    _lib = L
    return L


def _check(status: int, what: str) -> None:
    if status != NASTAR_OK:
        L = lib()
        msg = L.nastar_b200_status_string(status).decode()
        if status == 3:
            msg += ": " + L.nastar_b200_last_cuda_error().decode()
        raise RuntimeError(f"{what} failed: {msg}")


def host_scalars(g_ratio: float, W: int) -> Tuple[float, float, float]:
    """The Python-double scalar arithmetic of differentiable_astar.py:206-207; ctypes then rounds
    each to fp32 exactly as ATen rounds a Python scalar operand."""
    return float(g_ratio), float(1 - g_ratio), math.sqrt(W)


def _plane(x: torch.Tensor) -> Tuple[torch.Tensor, int, int]:
    """Return (tensor kept alive, device pointer of channel 0, map stride in elements)."""
    if x.dtype != torch.float32:
        raise TypeError(f"planes must be float32 (got {x.dtype}); the reference path is fp32-only")
    H, W = x.shape[-2], x.shape[-1]
    if x.stride(-1) != 1 or x.stride(-2) != W:
        x = x.contiguous()
    return x, x.data_ptr(), x.stride(0)


def _set_planes(p: ctypes.Structure, planes) -> list:
    """Write the channel-0 pointer and map stride of each (name, plane) into p.<name> / p.<name>_stride (FwdParams,
    BwdParams).  Returns the tensors that must stay alive until the call has been issued."""
    keep = []
    for name, t_ in planes:
        k, ptr, stride = _plane(t_.detach())
        keep.append(k)
        setattr(p, name, ptr)
        setattr(p, name + "_stride", stride)
    return keep


def _maps(x: torch.Tensor, cuda_msg: str, shape_msg: str) -> Tuple[torch.Tensor, int, int]:
    """_plane of fp32 CUDA maps given as [B,H,W] or [B,1,H,W]; the tensor kept alive is [B,H,W]."""
    if not x.is_cuda or x.dtype != torch.float32:
        raise RuntimeError(cuda_msg)
    if x.ndim == 4 and x.shape[1] == 1:
        x = x[:, 0]
    if x.ndim != 3:
        raise ValueError(shape_msg)
    return _plane(x.detach())


@contextlib.contextmanager
def _on_device(dev: torch.device):
    """Make `dev` the current device (entering the guard only when it is not already) and yield its current stream
    as the `void* stream` argument of the C ABI."""
    with contextlib.nullcontext() if dev.index == torch.cuda.current_device() else torch.cuda.device(dev):
        yield ctypes.c_void_p(torch.cuda.current_stream(dev).cuda_stream)


def launch_count() -> int:
    return int(lib().nastar_b200_launch_count())


FWD_NO_EARLY_EXIT = 1
FWD_PAIR = 2
FWD_NEWS = 4
COST_PLANE, COST_LOGIT, COST_TAPS = 0, 1, 2
TAPS_MAX_SIDE = 64     # largest H and W whose search reads COST_LOGIT / COST_TAPS (engines 1 and 4)


# NASTAR_MECH_*: the planning-datasets generator's --mechanism values
MECHANISMS = {"moore": 0, "news": 1}


def mechanism_code(mechanism: str) -> int:
    """NASTAR_MECH_* of a mechanism name; anything but "moore" and "news" is a ValueError."""
    if mechanism not in MECHANISMS:
        raise ValueError(f"mechanism must be one of {sorted(MECHANISMS)} (got {mechanism!r})")
    return MECHANISMS[mechanism]


# the loop bound reaches the library as int32_t (nastar_fwd_params.T, the T of nastar_b200_batch_steps, *T_batch)
MAX_STEPS = 2**31 - 1
MAX_EVAL_WIDTH = math.isqrt(MAX_STEPS)   # 46 340: the widest map whose evaluation bound W*W fits


def check_steps(T: int, what: str = "the step bound T") -> int:
    """int(T), or a ValueError when T does not fit the library's int32 loop bound (a silent ctypes truncation would
    search with a wrong bound)."""
    T = int(T)
    if T > MAX_STEPS:
        raise ValueError(f"{what} = {T} exceeds 2**31 - 1, the largest loop bound the search takes: the evaluation "
                         f"bound W*W fits for W <= {MAX_EVAL_WIDTH} only")
    return T


class SearchCounts(tuple):
    """(n_closed [B'] i32, path_len [B'] i32): histories.sum() / paths.sum() per map, written by the kernel."""


def _search_params(cost: torch.Tensor, start: torch.Tensor, goal: torch.Tensor, obst: torch.Tensor, g_ratio: float,
                   T: int, flags: int, cost_kind: int, cost_scale: float, cost_bias: float, mechanism: str):
    """Check the inputs of `forward` / `forward_coupled` and fill their FwdParams up to the outputs.  `flags` gets
    NASTAR_FWD_NEWS added for `mechanism` "news".  Returns (p, planes to keep alive, B, H, W, device)."""
    news = mechanism_code(mechanism) == MECHANISMS["news"]
    T = check_steps(T)
    lib()
    if not cost.is_cuda:
        raise RuntimeError("neural_astar (H100): the search runs on CUDA tensors only (no CPU fallback); "
                           "move the planner inputs to the GPU")
    dev = cost.device
    for t_ in (start, goal, obst):
        if t_.device != dev:
            raise RuntimeError("all planes must live on the same CUDA device")
    if start.ndim != 4:
        raise ValueError("planes are [B,C,H,W]")
    B, _, H, W = start.shape
    planes = [("start", start), ("goal", goal), ("obst", obst)]
    p = FwdParams()
    if cost_kind == COST_TAPS:
        if cost.dtype != torch.float32 or tuple(cost.shape) != (B, H, W, 9) or not cost.is_contiguous():
            raise ValueError("COST_TAPS expects a contiguous fp32 [B,H,W,9] tensor")
        p.cost, p.cost_stride = cost.data_ptr(), 9 * H * W
    else:
        planes.insert(0, ("cost", cost))
    for _, t_ in planes:
        if t_.shape[0] != B or t_.shape[-2:] != (H, W):
            raise ValueError("plane shapes differ")
    keep = _set_planes(p, planes)
    gr, omg, _ = host_scalars(g_ratio, W)
    p.B, p.H, p.W = B, H, W
    p.g_ratio, p.one_minus_g_ratio = gr, omg
    p.T = int(T)
    p.flags = flags | (FWD_NEWS if news else 0)
    p.cost_kind, p.cost_scale, p.cost_bias = int(cost_kind), float(cost_scale), float(cost_bias)
    return p, keep, B, H, W, dev


def forward(cost: torch.Tensor, start: torch.Tensor, goal: torch.Tensor, obst: torch.Tensor,
            g_ratio: float, T: int, want_trace: bool = False, no_early_exit: bool = False, *,
            pair: bool = False, cost_kind: int = COST_PLANE, cost_scale: float = 1.0, cost_bias: float = 0.0,
            want_counts: bool = False, mechanism: str = "moore"):
    """Run the search for a batch of [B,C,H,W] fp32 CUDA planes (channel 0 is used).

    Returns (histories [B',1,H,W] f32, paths [B',1,H,W] i64, t_solve [B'] i32, n_steps [B'] i32,
    trace [B',T] i32 or None), all on the inputs' device, asynchronously on the current stream; with
    `want_counts` a sixth element (n_closed [B'], path_len [B']) is appended.  B' = 2B with `pair`
    (NASTAR_FWD_PAIR: second half = the same problems with cost = obstacles), else B.
    `cost_kind` = COST_LOGIT / COST_TAPS: `cost` holds the encoder's raw output [B,1,H,W] / the 9-tap partial
    products [B,H,W,9] and the kernel prologue finishes encoder.py:32-34 itself (H, W <= 64 only).
    `mechanism` = "moore" (8-connected, Chebyshev heuristic) or "news" (NASTAR_FWD_NEWS: 4-connected, Manhattan
    heuristic; both halves of a `pair`).
    """
    flags = (FWD_NO_EARLY_EXIT if no_early_exit else 0) | (FWD_PAIR if pair else 0)
    p, keep, B, H, W, dev = _search_params(cost, start, goal, obst, g_ratio, T, flags, cost_kind, cost_scale,
                                           cost_bias, mechanism)
    L = lib()
    Bo = 2 * B if pair else B
    ws_bytes = _ws_cache.get((B, H, W))
    if ws_bytes is None:
        ws_bytes = _ws_cache[(B, H, W)] = int(L.nastar_b200_forward_workspace_bytes(B, H, W))
    with _on_device(dev) as stream:
        hist = torch.empty((Bo, 1, H, W), dtype=torch.float32, device=dev)
        paths = torch.empty((Bo, 1, H, W), dtype=torch.int64, device=dev)
        counters = torch.empty((4 if want_counts else 2, Bo), dtype=torch.int32, device=dev)   # [t_solve | n_steps | ...]
        t_solve, n_steps = counters[0], counters[1]
        trace = torch.empty((Bo, int(T)), dtype=torch.int32, device=dev) if want_trace else None
        ws = torch.empty((ws_bytes,), dtype=torch.uint8, device=dev) if ws_bytes else None
        p.histories, p.paths = hist.data_ptr(), paths.data_ptr()
        p.t_solve, p.n_steps = t_solve.data_ptr(), n_steps.data_ptr()
        if want_counts:
            p.n_closed, p.path_len = counters[2].data_ptr(), counters[3].data_ptr()
        p.trace = trace.data_ptr() if want_trace else None
        p.workspace = ws.data_ptr() if ws is not None else None
        p.workspace_bytes = ws_bytes
        _check(L.nastar_b200_forward(ctypes.byref(p), stream), "nastar_b200_forward")
    del keep
    if want_counts:
        return hist, paths, t_solve, n_steps, trace, SearchCounts((counters[2], counters[3]))
    return hist, paths, t_solve, n_steps, trace


def forward_coupled(cost: torch.Tensor, start: torch.Tensor, goal: torch.Tensor, obst: torch.Tensor,
                    g_ratio: float, T: int, *, cost_kind: int = COST_PLANE, cost_scale: float = 1.0,
                    cost_bias: float = 0.0, mechanism: str = "moore", want_counts: bool = False):
    """The reference's batch-synchronous search for g_ratio < 0.5 with T_batch decided on the device
    (include/nastar_b200.h, nastar_b200_forward_coupled): every map's outputs after exactly
    T_batch = 1 + min{k < T : every map selects its goal at step k} steps (T if there is none), in three launches on the
    current stream and without a host synchronisation, so the call can be captured in a CUDA graph.

    Inputs as in `forward` (no trace, no pair).  Returns (histories [B,1,H,W] f32, paths [B,1,H,W] i64, t_solve [B] i32,
    n_steps [B] i32, T_batch [1] i32, goal_clamp [B] i32), all on the inputs' device; with `want_counts` a seventh
    element (n_closed [B], path_len [B]) is appended.  The first five equal `forward(..., T=T_batch,
    no_early_exit=True)`; goal_clamp is 0 where the goal is selected at least twice within T_batch steps and T_batch
    elsewhere, the `t_solve` that `backward` takes for such a forward."""
    p, keep, B, H, W, dev = _search_params(cost, start, goal, obst, g_ratio, T, 0, cost_kind, cost_scale, cost_bias,
                                           mechanism)
    L = lib()
    key = (B, H, W, int(T))
    ws_bytes = _coupled_ws_cache.get(key)
    if ws_bytes is None:
        ws_bytes = _coupled_ws_cache[key] = int(L.nastar_b200_forward_coupled_workspace_bytes(B, H, W, int(T)))
    with _on_device(dev) as stream:
        hist = torch.empty((B, 1, H, W), dtype=torch.float32, device=dev)
        paths = torch.empty((B, 1, H, W), dtype=torch.int64, device=dev)
        counters = torch.empty((5 if want_counts else 3, B), dtype=torch.int32, device=dev)  # [t_solve | n_steps | clamp | ...]
        t_solve, n_steps, goal_clamp = counters[0], counters[1], counters[2]
        T_batch = torch.empty((1,), dtype=torch.int32, device=dev)
        ws = torch.empty((ws_bytes,), dtype=torch.uint8, device=dev)
        p.histories, p.paths = hist.data_ptr(), paths.data_ptr()
        p.t_solve, p.n_steps = t_solve.data_ptr(), n_steps.data_ptr()
        if want_counts:
            p.n_closed, p.path_len = counters[3].data_ptr(), counters[4].data_ptr()
        p.trace = None
        p.workspace, p.workspace_bytes = ws.data_ptr(), ws_bytes
        _check(L.nastar_b200_forward_coupled(ctypes.byref(p), T_batch.data_ptr(), goal_clamp.data_ptr(), stream),
               "nastar_b200_forward_coupled")
    del keep
    if want_counts:
        return hist, paths, t_solve, n_steps, T_batch, goal_clamp, SearchCounts((counters[3], counters[4]))
    return hist, paths, t_solve, n_steps, T_batch, goal_clamp


def pack_inputs(map_designs: torch.Tensor, start: torch.Tensor, goal: torch.Tensor) -> torch.Tensor:
    """Encoder input of NeuralAstar.encode (reference astar.py:172-177) in ONE kernel: channels-last
    [B, C+1, Hm, Wm] = cat(map_designs, nearest-upsampled(start + goal))."""
    L = lib()
    if not map_designs.is_cuda or map_designs.dtype != torch.float32:
        raise RuntimeError("pack_inputs: fp32 CUDA tensors only")
    B, C, Hm, Wm = map_designs.shape
    H, W = start.shape[-2], start.shape[-1]
    md = map_designs.detach().contiguous()
    ks, ps, ss = _plane(start.detach())
    kg, pg, sg = _plane(goal.detach())
    dev = map_designs.device
    with _on_device(dev) as stream:
        out = torch.empty((B, Hm, Wm, C + 1), dtype=torch.float32, device=dev)
        _check(L.nastar_b200_pack_inputs(md.data_ptr(), C, Hm, Wm, ps, ss, pg, sg, B, H, W, out.data_ptr(),
                                         stream), "nastar_b200_pack_inputs")
    del ks, kg
    return out.permute(0, 3, 1, 2)   # logical NCHW view with channels-last strides


HEAD_CHANNELS = (16, 32, 64, 128, 256)


def conv1_marks(map_designs: torch.Tensor, start: torch.Tensor, goal: torch.Tensor, w_host, bias_host) -> torch.Tensor:
    """relu(bias + conv3x3(cat(map_designs, start + goal))) as a channels-last [B,32,H,W] tensor in one kernel (the
    "m+" encoder's first layer fused with NeuralAstar.encode's input assembly).  w_host: C-contiguous float32 NumPy
    array [9,2,32] = [tap, cin, cout] (BatchNorm folded), bias_host: float32 NumPy [32]; both on the HOST (they travel
    as kernel parameters)."""
    L = lib()
    B, C, H, W = map_designs.shape
    if C != 1 or start.shape[-2:] != (H, W) or map_designs.dtype != torch.float32 or not map_designs.is_cuda:
        raise ValueError("conv1_marks: one-channel fp32 CUDA maps with start/goal maps of the same size")
    if (w_host.dtype.name != "float32" or w_host.shape != (9, 2, 32) or not w_host.flags["C_CONTIGUOUS"]
            or bias_host.dtype.name != "float32" or bias_host.shape != (32,) or not bias_host.flags["C_CONTIGUOUS"]):
        raise ValueError("conv1_marks: w_host must be a C-contiguous float32 [9,2,32] array, bias_host float32 [32]")
    md = map_designs.detach().contiguous()
    ks, ps, ss = _plane(start.detach())
    kg, pg, sg = _plane(goal.detach())
    dev = map_designs.device
    with _on_device(dev) as stream:
        out = torch.empty((B, H, W, 32), dtype=torch.float32, device=dev)
        _check(L.nastar_b200_conv1_marks(md.data_ptr(), ps, ss, pg, sg, B, H, W, w_host.ctypes.data,
                                         bias_host.ctypes.data, out.data_ptr(), stream),
               "nastar_b200_conv1_marks")
    del ks, kg
    return out.permute(0, 3, 1, 2)


def head_taps(x: torch.Tensor, w_host, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """taps [B,H,W,9] = per-pixel products of a channels-last activation x [B,C,H,W] with the head conv's folded
    weights `w_host` (a contiguous float32 NumPy array [C,9] on the HOST: it travels as a kernel parameter)."""
    L = lib()
    B, C, H, W = x.shape
    if C not in HEAD_CHANNELS or x.dtype != torch.float32 or not x.is_contiguous(memory_format=torch.channels_last):
        raise ValueError("head_taps expects a channels-last fp32 activation with 16/32/64/128/256 channels")
    if w_host.dtype.name != "float32" or w_host.shape != (C, 9) or not w_host.flags["C_CONTIGUOUS"]:
        raise ValueError("w_host must be a C-contiguous float32 [C,9] array")
    dev = x.device
    with _on_device(dev) as stream:
        if out is None:
            out = torch.empty((B, H, W, 9), dtype=torch.float32, device=dev)
        _check(L.nastar_b200_head_taps(x.data_ptr(), B * H * W, C, w_host.ctypes.data, out.data_ptr(),
                                       stream), "nastar_b200_head_taps")
    return out


def upsample_concat(dec: torch.Tensor, skip: Optional[torch.Tensor]) -> torch.Tensor:
    """torch.cat((F.interpolate(dec, scale_factor=2, mode="nearest"), skip), 1) in one kernel, bit for bit: the input of
    a U-Net decoder block.  dec: channels-last fp32 CUDA [B,Cd,h,w]; skip: channels-last fp32 [B,Cs,2h,2w] on the same
    device, or None for the last block.  Channel counts must be multiples of 4.  Returns a channels-last
    [B,Cd+Cs,2h,2w] tensor."""
    L = lib()
    B, Cd, h, w = dec.shape
    Cs = 0 if skip is None else skip.shape[1]
    if (not dec.is_cuda or dec.dtype != torch.float32 or not dec.is_contiguous(memory_format=torch.channels_last)
            or Cd % 4 or Cs % 4):
        raise ValueError("upsample_concat expects channels-last fp32 CUDA tensors with channel counts divisible by 4")
    if skip is not None and (tuple(skip.shape) != (B, Cs, 2 * h, 2 * w) or skip.dtype != torch.float32
                             or skip.device != dec.device
                             or not skip.is_contiguous(memory_format=torch.channels_last)):
        raise ValueError("upsample_concat expects a channels-last fp32 skip [B,Cs,2h,2w] on dec's device")
    dev = dec.device
    with _on_device(dev) as stream:
        out = torch.empty((B, 2 * h, 2 * w, Cd + Cs), dtype=torch.float32, device=dev)
        _check(L.nastar_b200_upsample_concat(dec.data_ptr(), B, h, w, Cd, skip.data_ptr() if Cs else None, Cs,
                                             out.data_ptr(), stream), "nastar_b200_upsample_concat")
    return out.permute(0, 3, 1, 2)


CONVHEAD_CHANNELS = (128, 256)    # (C_in, C_out) of the fused last-conv + head kernel
CONVHEAD_MAX_SIDE = 64


def conv3x3_head_taps(x: torch.Tensor, w: torch.Tensor, b: torch.Tensor, head_w_host,
                      out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """taps [B,H,W,9] = head products of relu(conv3x3(x, w, pad 1) + b) in one kernel, without writing the activation
    (include/nastar_b200.h, nastar_b200_conv3x3_head_taps).  x: channels-last fp32 CUDA [B,128,H,W], H, W <= 64;
    w: folded conv weights [256,128,3,3] stored channels-last; b: [256]; head_w_host: C-contiguous float32 NumPy [256,9]
    on the HOST.  The convolution runs on TF32 tensor cores with fp32 accumulation; the head products are fp32."""
    L = lib()
    B, C, H, W = x.shape
    if (not x.is_cuda or x.dtype != torch.float32 or not x.is_contiguous(memory_format=torch.channels_last)
            or (C, w.shape[0]) != CONVHEAD_CHANNELS or H > CONVHEAD_MAX_SIDE or W > CONVHEAD_MAX_SIDE):
        raise ValueError("conv3x3_head_taps expects a channels-last fp32 CUDA activation [B,128,H,W], H, W <= 64")
    if (tuple(w.shape) != (256, 128, 3, 3) or w.dtype != torch.float32 or w.device != x.device
            or not w.is_contiguous(memory_format=torch.channels_last)):
        raise ValueError("conv3x3_head_taps expects fp32 weights [256,128,3,3] stored channels-last on x's device")
    if tuple(b.shape) != (256,) or b.dtype != torch.float32 or b.device != x.device or not b.is_contiguous():
        raise ValueError("conv3x3_head_taps expects a contiguous fp32 bias [256] on x's device")
    if head_w_host.dtype.name != "float32" or head_w_host.shape != (256, 9) or not head_w_host.flags["C_CONTIGUOUS"]:
        raise ValueError("head_w_host must be a C-contiguous float32 [256,9] array")
    dev = x.device
    with _on_device(dev) as stream:
        if out is None:
            out = torch.empty((B, H, W, 9), dtype=torch.float32, device=dev)
        elif tuple(out.shape) != (B, H, W, 9) or out.dtype != torch.float32 or not out.is_contiguous():
            raise ValueError("out must be a contiguous fp32 [B,H,W,9] tensor")
        _check(L.nastar_b200_conv3x3_head_taps(x.data_ptr(), B, H, W, C, 256, w.data_ptr(), b.data_ptr(),
                                               head_w_host.ctypes.data, out.data_ptr(), stream),
               "nastar_b200_conv3x3_head_taps")
    return out


def cost_from_taps(taps: torch.Tensor, bias: float, scale: float) -> torch.Tensor:
    """cost maps [B,1,H,W] = sigmoid(bias + 9-tap gather(taps)) * scale; taps is fp32 [B,H,W,9] (the same
    arithmetic as the search kernel's COST_TAPS prologue)."""
    L = lib()
    B, H, W, nine = taps.shape
    if nine != 9 or taps.dtype != torch.float32 or not taps.is_contiguous() or not taps.is_cuda:
        raise ValueError("cost_from_taps expects a contiguous fp32 CUDA [B,H,W,9] tensor")
    dev = taps.device
    with _on_device(dev) as stream:
        cost = torch.empty((B, 1, H, W), dtype=torch.float32, device=dev)
        _check(L.nastar_b200_cost_from_taps(taps.data_ptr(), B, H, W, float(bias), float(scale), cost.data_ptr(),
                                            stream), "nastar_b200_cost_from_taps")
    return cost


def batch_steps(t_solve: torch.Tensor, n_steps: torch.Tensor, T: int) -> torch.Tensor:
    """Device-side T_batch (int32[1]); replaces the per-step host sync of differentiable_astar.py:251."""
    T = check_steps(T)
    L = lib()
    dev = t_solve.device
    with _on_device(dev) as stream:
        out = torch.empty((1,), dtype=torch.int32, device=dev)
        _check(L.nastar_b200_batch_steps(t_solve.data_ptr(), n_steps.data_ptr(), t_solve.numel(), int(T),
                                         out.data_ptr(), stream), "nastar_b200_batch_steps")
    return out


LABELS_MAX_SIDE = 512


def opt_labels(maps: torch.Tensor, goal_idx: torch.Tensor, mechanism: str = "moore"):
    """Shortest-path labels of B maps in one kernel (include/nastar_b200.h, nastar_b200_opt_labels_mech).

    maps: fp32 CUDA [B,H,W] or [B,1,H,W] (a cell is passable iff != 0); goal_idx: int32 CUDA [B], flat goal index;
    mechanism: "moore" (8 actions) or "news" (4 actions, act_mask bits 0..3 only).
    Returns (dists fp32 [B,1,H,W], act_mask uint8 [B,1,H,W], action int8 [B,1,H,W]) on the current stream."""
    if mechanism not in MECHANISMS:
        raise ValueError(f"opt_labels: mechanism must be one of {sorted(MECHANISMS)} (got {mechanism!r})")
    L = lib()
    m, ptr, stride = _maps(maps, "opt_labels: fp32 CUDA maps only (there is no CPU fallback)",
                           "opt_labels: maps are [B,H,W] or [B,1,H,W]")
    B, H, W = m.shape
    dev = m.device
    if goal_idx.dtype != torch.int32 or goal_idx.device != dev or tuple(goal_idx.shape) != (B,):
        raise ValueError("opt_labels: goal_idx must be an int32 [B] tensor on the maps' device")
    if H > LABELS_MAX_SIDE or W > LABELS_MAX_SIDE:
        raise ValueError(f"opt_labels: maps up to {LABELS_MAX_SIDE}x{LABELS_MAX_SIDE} (got {H}x{W})")
    gi = goal_idx.contiguous()
    with _on_device(dev) as stream:
        dists = torch.empty((B, 1, H, W), dtype=torch.float32, device=dev)
        mask = torch.empty((B, 1, H, W), dtype=torch.uint8, device=dev)
        action = torch.empty((B, 1, H, W), dtype=torch.int8, device=dev)
        _check(L.nastar_b200_opt_labels_mech(ptr, stride, gi.data_ptr(), B, H, W, MECHANISMS[mechanism],
                                             dists.data_ptr(), mask.data_ptr(), action.data_ptr(), stream),
               "nastar_b200_opt_labels_mech")
    del m, gi
    return dists, mask, action


WLABELS_MAX_SIDE = 128


class WeightedLabels(tuple):
    """Output of weighted_labels: (dists f32 [B,1,H,W], hops i32 [B,1,H,W], act_mask u8 [B,1,H,W], action i8
    [B,1,H,W], path_maps f32 [B,1,H,W] or None, path_costs f32 [B] or None, status i32 [B])."""


def weighted_labels(cost: torch.Tensor, goal_idx: torch.Tensor, passable: Optional[torch.Tensor] = None,
                    start_idx: Optional[torch.Tensor] = None, mechanism: str = "moore") -> WeightedLabels:
    """Exact vertex-weighted shortest paths of B cost maps in one kernel (include/nastar_b200.h,
    nastar_b200_weighted_labels_mech).

    cost: fp32 CUDA [B,H,W] or [B,1,H,W]; passable: the same shape (a cell is passable iff != 0) or None (every cell);
    goal_idx / start_idx: int32 CUDA [B] flat indices (start_idx None: no paths); mechanism: "moore" (8 moves) or
    "news" (4 moves N, E, W, S; act_mask bits 0..3 only).  H, W <= 128.  Asynchronous on the current stream; the
    per-map status is not read back here."""
    if mechanism not in MECHANISMS:
        raise ValueError(f"weighted_labels: mechanism must be one of {sorted(MECHANISMS)} (got {mechanism!r})")
    L = lib()

    def plane(x, name):
        return _maps(x, f"weighted_labels: {name} must be fp32 CUDA maps (there is no CPU fallback)",
                     f"weighted_labels: {name} are [B,H,W] or [B,1,H,W]")

    c, cptr, cstride = plane(cost, "cost maps")
    B, H, W = c.shape
    dev = c.device
    p, pptr, pstride = (None, None, 0) if passable is None else plane(passable, "passable maps")
    if p is not None and (p.shape != c.shape or p.device != dev):
        raise ValueError("weighted_labels: passable maps must match the cost maps' shape and device")
    for name, ix in (("goal_idx", goal_idx), ("start_idx", start_idx)):
        if ix is not None and (ix.dtype != torch.int32 or ix.device != dev or tuple(ix.shape) != (B,)):
            raise ValueError(f"weighted_labels: {name} must be an int32 [B] tensor on the cost maps' device")
    if H > WLABELS_MAX_SIDE or W > WLABELS_MAX_SIDE:
        raise ValueError(f"weighted_labels: maps up to {WLABELS_MAX_SIDE}x{WLABELS_MAX_SIDE} (got {H}x{W})")
    gi = goal_idx.contiguous()
    si = None if start_idx is None else start_idx.contiguous()
    with _on_device(dev) as stream:
        dists = torch.empty((B, 1, H, W), dtype=torch.float32, device=dev)
        hops = torch.empty((B, 1, H, W), dtype=torch.int32, device=dev)
        mask = torch.empty((B, 1, H, W), dtype=torch.uint8, device=dev)
        action = torch.empty((B, 1, H, W), dtype=torch.int8, device=dev)
        paths = None if si is None else torch.empty((B, 1, H, W), dtype=torch.float32, device=dev)
        pcost = None if si is None else torch.empty((B,), dtype=torch.float32, device=dev)
        status = torch.empty((B,), dtype=torch.int32, device=dev)
        _check(L.nastar_b200_weighted_labels_mech(cptr, cstride, pptr, pstride, gi.data_ptr(),
                                                  None if si is None else si.data_ptr(), B, H, W,
                                                  MECHANISMS[mechanism], dists.data_ptr(), hops.data_ptr(),
                                                  mask.data_ptr(), action.data_ptr(),
                                                  None if paths is None else paths.data_ptr(),
                                                  None if pcost is None else pcost.data_ptr(), status.data_ptr(),
                                                  stream), "nastar_b200_weighted_labels_mech")
    del c, p, gi, si
    return WeightedLabels((dists, hops, mask, action, paths, pcost, status))


SAMPLER_MAX_SIDE = 512


class SamplerTables(tuple):
    """Per-map output of sampler_prepare: (band_bits i32 [B,3,ceil(N/32)], counts i32 [B,3], goal_idx i32 [B],
    actions i32 [B,ceil(N/8)], thresholds f64 [B,4], status i32 [B]), N = H*W (u32 words carried as int32)."""


def sampler_prepare(dists: torch.Tensor, policies: torch.Tensor, goal_maps: torch.Tensor, quantiles) -> SamplerTables:
    """MazeDataset._prepared for B maps in one kernel (include/nastar_b200.h, nastar_b200_sampler_prepare).

    dists [B,1,H,W], policies [B,8,1,H,W], goal_maps [B,1,H,W]: fp32 CUDA tensors; quantiles: the four fp64 fractions
    np.percentile evaluates.  Asynchronous on the current stream."""
    L = lib()
    B, _, H, W = dists.shape
    for name, t_, shape in (("dists", dists, (B, 1, H, W)), ("policies", policies, (B, 8, 1, H, W)),
                            ("goal_maps", goal_maps, (B, 1, H, W))):
        if not t_.is_cuda or t_.dtype != torch.float32 or tuple(t_.shape) != shape or t_.device != dists.device:
            raise ValueError(f"sampler_prepare: {name} must be an fp32 CUDA tensor {list(shape)} on the dists' device")
    if H > SAMPLER_MAX_SIDE or W > SAMPLER_MAX_SIDE:
        raise ValueError(f"sampler_prepare: maps up to {SAMPLER_MAX_SIDE}x{SAMPLER_MAX_SIDE} (got {H}x{W})")
    d, p, g = (t_.detach().contiguous() for t_ in (dists, policies, goal_maps))
    N = H * W
    dev = dists.device
    with _on_device(dev) as stream:
        i32 = dict(dtype=torch.int32, device=dev)
        out = SamplerTables((torch.empty((B, 3, (N + 31) // 32), **i32), torch.empty((B, 3), **i32),
                             torch.empty((B,), **i32), torch.empty((B, (N + 7) // 8), **i32),
                             torch.empty((B, 4), dtype=torch.float64, device=dev), torch.empty((B,), **i32)))
        q = [float(v) for v in quantiles]
        _check(L.nastar_b200_sampler_prepare(d.data_ptr(), p.data_ptr(), g.data_ptr(), B, H, W, *q,
                                             *(t_.data_ptr() for t_ in out), stream),
               "nastar_b200_sampler_prepare")
    del d, p, g
    return out


def sampler_sample(maps: torch.Tensor, goal_maps: torch.Tensor, tables: SamplerTables, indices: torch.Tensor,
                   draws: torch.Tensor):
    """One training batch in one kernel (nastar_b200_sampler_sample): maps / goal_maps fp32 CUDA [n,1,H,W] (contiguous),
    tables from sampler_prepare for the same n maps, indices int64 CUDA [B], draws int32 CUDA [B,S,2].
    Returns (map_designs [B,1,H,W], start_maps [B,S,H,W], goal_maps [B,1,H,W], opt_trajs [B,S,H,W]), fp32."""
    L = lib()
    n, _, H, W = maps.shape
    if (maps.dtype != torch.float32 or not maps.is_cuda or not maps.is_contiguous() or goal_maps.shape != maps.shape
            or goal_maps.dtype != torch.float32 or not goal_maps.is_contiguous() or goal_maps.device != maps.device):
        raise ValueError("sampler_sample: maps and goal_maps must be contiguous fp32 CUDA tensors [n,1,H,W]")
    B, S, two = draws.shape
    if two != 2 or draws.dtype != torch.int32 or not draws.is_contiguous() or draws.device != maps.device:
        raise ValueError("sampler_sample: draws must be a contiguous int32 [B,S,2] tensor on the maps' device")
    if (indices.dtype != torch.int64 or tuple(indices.shape) != (B,) or not indices.is_contiguous()
            or indices.device != maps.device):
        raise ValueError("sampler_sample: indices must be a contiguous int64 [B] tensor on the maps' device")
    bits, counts, goal_idx, actions = tables[:4]
    dev = maps.device
    with _on_device(dev) as stream:
        f32 = dict(dtype=torch.float32, device=dev)
        out = (torch.empty((B, 1, H, W), **f32), torch.empty((B, S, H, W), **f32), torch.empty((B, 1, H, W), **f32),
               torch.empty((B, S, H, W), **f32))
        _check(L.nastar_b200_sampler_sample(maps.data_ptr(), goal_maps.data_ptr(), n, H, W, bits.data_ptr(),
                                            counts.data_ptr(), goal_idx.data_ptr(), actions.data_ptr(),
                                            indices.data_ptr(), draws.data_ptr(), B, S,
                                            *(t_.data_ptr() for t_ in out), stream),
               "nastar_b200_sampler_sample")
    return out


GOALS_MAX_SIDE = 512


def sample_goals(maps: torch.Tensor, draws: torch.Tensor, edge_size: int = 0):
    """Goals of B maps in one kernel (include/nastar_b200.h, nastar_b200_sample_goals): a cell of the largest
    4-connected passable region, in its edge_size corner squares when it reaches one, chosen by the map's u32 draw.

    maps: fp32 CUDA [B,H,W] or [B,1,H,W] (a cell is passable iff != 0); draws: int32 [B] on the maps' device.
    Returns (goal_idx int32 [B], goal_maps fp32 [B,1,H,W], status int32 [B]) on the current stream; status 1 marks a map
    without a passable cell (goal_idx -1, all-zero plane) and is not read back here."""
    L = lib()
    B = maps.shape[0] if maps.ndim in (3, 4) else None
    if not isinstance(draws, torch.Tensor) or draws.dtype != torch.int32 or tuple(draws.shape) != (B,):
        raise ValueError(f"sample_goals: draws must be an int32 [B] tensor, B = {B} maps")
    m, ptr, stride = _maps(maps, "sample_goals: fp32 CUDA maps only (there is no CPU fallback)",
                           "sample_goals: maps are [B,H,W] or [B,1,H,W]")
    _, H, W = m.shape
    dev = m.device
    if draws.device != dev:
        raise ValueError("sample_goals: draws must be on the maps' device")
    if H > GOALS_MAX_SIDE or W > GOALS_MAX_SIDE:
        raise ValueError(f"sample_goals: maps up to {GOALS_MAX_SIDE}x{GOALS_MAX_SIDE} (got {H}x{W})")
    if int(edge_size) < 0:
        raise ValueError(f"sample_goals: edge_size must be >= 0 (got {edge_size})")
    d = draws.contiguous()
    with _on_device(dev) as stream:
        goal_idx = torch.empty((B,), dtype=torch.int32, device=dev)
        goal_maps = torch.empty((B, 1, H, W), dtype=torch.float32, device=dev)
        status = torch.empty((B,), dtype=torch.int32, device=dev)
        _check(L.nastar_b200_sample_goals(ptr, stride, B, H, W, int(edge_size), d.data_ptr(), goal_idx.data_ptr(),
                                          goal_maps.data_ptr(), status.data_ptr(), stream), "nastar_b200_sample_goals")
    del m, d
    return goal_idx, goal_maps, status


MAPS_MAX_SIDE = 512
MAPS_MAX_SOURCE_SIDE = 2048


def maps_from_images(images: torch.Tensor, H: int, W: int, want_resized: bool = False):
    """Planning maps of B decoded L images in one kernel (include/nastar_b200.h, nastar_b200_maps_from_images): Pillow's
    bicubic resize to H x W, skimage's Otsu threshold, level > threshold.

    images: uint8 CUDA [B,H0,W0].  Returns (maps fp32 [B,1,H,W], resized uint8 [B,H,W] or None, thresholds fp32 [B],
    status int32 [B]) on the current stream; status 1 marks a uniform resized image (all-zero map) and is not read back
    here."""
    L = lib()
    if not isinstance(images, torch.Tensor) or not images.is_cuda or images.dtype != torch.uint8:
        raise RuntimeError("maps_from_images: uint8 CUDA images only (there is no CPU fallback)")
    if images.ndim != 3 or min(images.shape) < 1:
        raise ValueError(f"maps_from_images: images are [B,H0,W0] with B, H0, W0 >= 1 (got {tuple(images.shape)})")
    B, H0, W0 = images.shape
    H, W = int(H), int(W)
    if not (1 <= H <= MAPS_MAX_SIDE and 1 <= W <= MAPS_MAX_SIDE):
        raise ValueError(f"maps_from_images: maps from 1x1 up to {MAPS_MAX_SIDE}x{MAPS_MAX_SIDE} (got {H}x{W})")
    if H0 > MAPS_MAX_SOURCE_SIDE or W0 > MAPS_MAX_SOURCE_SIDE:
        raise ValueError(f"maps_from_images: images up to {MAPS_MAX_SOURCE_SIDE}x{MAPS_MAX_SOURCE_SIDE} "
                         f"(got {H0}x{W0})")
    x = images.contiguous()
    dev = x.device
    with _on_device(dev) as stream:
        maps = torch.empty((B, 1, H, W), dtype=torch.float32, device=dev)
        resized = torch.empty((B, H, W), dtype=torch.uint8, device=dev) if want_resized else None
        thresholds = torch.empty((B,), dtype=torch.float32, device=dev)
        status = torch.empty((B,), dtype=torch.int32, device=dev)
        _check(L.nastar_b200_maps_from_images(x.data_ptr(), H0 * W0, B, H0, W0, H, W, maps.data_ptr(),
                                              resized.data_ptr() if want_resized else None, thresholds.data_ptr(),
                                              status.data_ptr(), stream), "nastar_b200_maps_from_images")
    del x
    return maps, resized, thresholds, status


def draw_policies(act_mask: torch.Tensor, draws: torch.Tensor) -> torch.Tensor:
    """One-hot policies drawn from maximal action sets in one kernel (include/nastar_b200.h, nastar_b200_draw_policies).

    act_mask: uint8 CUDA [B,1,H,W] or [B,H,W] (bit a = action a is maximal); draws: int32 tensor of the same number of
    cells on the mask's device.  Returns policies fp32 [B,8,1,H,W] on the current stream: cell c takes set bit
    (d * popc) >> 32 of its mask in action order, an empty mask gives an all-zero column."""
    L = lib()
    if not isinstance(act_mask, torch.Tensor) or not act_mask.is_cuda or act_mask.dtype != torch.uint8:
        raise RuntimeError("draw_policies: uint8 CUDA action masks only (there is no CPU fallback)")
    if act_mask.ndim == 4 and act_mask.shape[1] == 1:
        act_mask = act_mask[:, 0]
    if act_mask.ndim != 3 or act_mask.numel() == 0:
        raise ValueError("draw_policies: act_mask is [B,H,W] or [B,1,H,W]")
    B, H, W = act_mask.shape
    dev = act_mask.device
    if (not isinstance(draws, torch.Tensor) or draws.dtype != torch.int32 or draws.device != dev
            or draws.numel() != B * H * W):
        raise ValueError(f"draw_policies: draws must be an int32 tensor of B*H*W = {B * H * W} cells on the mask's "
                         "device")
    m, d = act_mask.contiguous(), draws.contiguous()
    with _on_device(dev) as stream:
        policies = torch.empty((B, 8, 1, H, W), dtype=torch.float32, device=dev)
        _check(L.nastar_b200_draw_policies(m.data_ptr(), d.data_ptr(), B, H * W, policies.data_ptr(), stream),
               "nastar_b200_draw_policies")
    del m, d
    return policies


# struct nastar_png_desc (include/nastar_b200.h) as a NumPy record, so a batch of descriptors is one host array
PNG_DESC_DTYPE = np.dtype([("in_off", "<i8"), ("in_len", "<i8"), ("plte_off", "<i8"), ("plte_len", "<i8"),
                           ("out_off", "<i8"), ("W0", "<i4"), ("H0", "<i4"), ("bit_depth", "<i4"),
                           ("color_type", "<i4"), ("interlace", "<i4"), ("reserved", "<i4")])
PNG_MAX_SIDE = 2048
# status bits of nastar_b200_decode_png
PNG_STATUS = {1: "bad zlib header", 2: "bad block type or Huffman code", 4: "distance past the start of the output",
              8: "stream ends early or inflates to the wrong length", 16: "Adler-32 mismatch", 32: "filter byte above 4"}


def decode_png_workspace_bytes(desc) -> int:
    """nastar_b200_decode_png_workspace_bytes of a NumPy array of PNG_DESC_DTYPE descriptors (0 when they are
    rejected)."""
    d = np.ascontiguousarray(desc, dtype=PNG_DESC_DTYPE)
    return int(lib().nastar_b200_decode_png_workspace_bytes(d.ctypes.data, len(d)))


def decode_png(data: torch.Tensor, desc, desc_dev: torch.Tensor, out_bytes: int):
    """PNG images to L planes in one kernel (include/nastar_b200.h, nastar_b200_decode_png).

    data: uint8 CUDA tensor holding every zlib stream and palette the descriptors point into; desc: a NumPy array of
    PNG_DESC_DTYPE (the host copy, checked before the launch); desc_dev: the same descriptors' bytes in device memory
    (a uint8 CUDA tensor, for example a slice of `data`).  Returns (out uint8 [out_bytes], status int32 [B]) on the
    current stream; status is not read back here."""
    L = lib()
    d = np.ascontiguousarray(desc, dtype=PNG_DESC_DTYPE)
    if not data.is_cuda or data.dtype != torch.uint8 or data.ndim != 1:
        raise RuntimeError("decode_png: data must be a 1-D uint8 CUDA tensor (there is no CPU fallback)")
    if (desc_dev.device != data.device or desc_dev.dtype != torch.uint8 or not desc_dev.is_contiguous()
            or desc_dev.numel() != d.nbytes):
        raise ValueError(f"decode_png: desc_dev must be {d.nbytes} contiguous uint8 bytes on the data's device")
    dev = data.device
    ws_bytes = int(L.nastar_b200_decode_png_workspace_bytes(d.ctypes.data, len(d)))
    with _on_device(dev) as stream:
        out = torch.empty((int(out_bytes),), dtype=torch.uint8, device=dev)
        status = torch.empty((len(d),), dtype=torch.int32, device=dev)
        ws = torch.empty((max(ws_bytes, 1),), dtype=torch.uint8, device=dev)
        _check(L.nastar_b200_decode_png(data.data_ptr(), data.numel(), d.ctypes.data, desc_dev.data_ptr(), len(d),
                                        out.data_ptr(), int(out_bytes), status.data_ptr(), ws.data_ptr(), ws_bytes,
                                        stream), "nastar_b200_decode_png")
    return out, status


# status of nastar_b200_pq_astar
PQ_SOLVED, PQ_NOT_FOUND, PQ_BAD_ENDS = 0, 1, 2
PQ_MAX_CELLS = 1 << 20


def pq_astar(cost: torch.Tensor, start: torch.Tensor, goal: torch.Tensor, map_design: torch.Tensor, g_ratio: float):
    """The reference's heap A* (include/nastar_b200.h, nastar_b200_pq_astar) on channel 0 of fp32 CUDA planes
    [B,C,H,W], one launch on the current stream.  Returns histories f32 [B,1,H,W], paths i64 [B,1,H,W], status i32 [B]
    (PQ_*) and expansions i32 [B]; nothing is read back."""
    L = lib()
    planes = (cost, start, goal, map_design)
    if any(not t.is_cuda or t.dtype != torch.float32 or t.ndim != 4 for t in planes):
        raise RuntimeError("pq_astar: planes must be fp32 CUDA tensors [B,C,H,W] (there is no CPU fallback)")
    B, _, H, W = cost.shape
    if any(t.shape[0] != B or t.shape[-2:] != (H, W) or t.device != cost.device for t in planes):
        raise ValueError("pq_astar: cost, start, goal and map must share B, H, W and the device")
    if H * W > PQ_MAX_CELLS:
        raise ValueError(f"pq_astar: H*W = {H * W} is above {PQ_MAX_CELLS} cells")
    dev = cost.device
    keep = [_plane(t.detach()) for t in planes]
    ws_bytes = int(L.nastar_b200_pq_astar_workspace_bytes(B, H, W))
    with _on_device(dev) as stream:
        hist = torch.empty((B, 1, H, W), dtype=torch.float32, device=dev)
        paths = torch.empty((B, 1, H, W), dtype=torch.int64, device=dev)
        status = torch.empty((B,), dtype=torch.int32, device=dev)
        expansions = torch.empty((B,), dtype=torch.int32, device=dev)
        ws = torch.empty((ws_bytes,), dtype=torch.uint8, device=dev)
        args = [a for _, ptr, stride in keep for a in (ptr, stride)]
        _check(L.nastar_b200_pq_astar(*args, B, H, W, float(g_ratio), hist.data_ptr(), paths.data_ptr(),
                                      status.data_ptr(), expansions.data_ptr(), ws.data_ptr(), ws_bytes, stream),
               "nastar_b200_pq_astar")
    del keep
    return hist, paths, status, expansions


def backward(cost, start, goal, obst, grad_hist: torch.Tensor, T_batch, t_solve: torch.Tensor,
             g_ratio: float, mechanism: str = "moore") -> torch.Tensor:
    """dL/dcost [B,1,H,W] from dL/dhistories (closed form of the reference's autograd, SURVEY App. B), for a forward
    that ran with the same `mechanism`.  `T_batch` is the replayed step count: an int32 [1] device tensor
    (batch_steps, forward_coupled) or a Python int, which must fit int32 like the forward's bound."""
    mech = mechanism_code(mechanism)
    dev = cost.device
    if not isinstance(T_batch, torch.Tensor):
        T_batch = torch.full((1,), check_steps(T_batch, "T_batch"), dtype=torch.int32, device=dev)
    L = lib()
    B, _, H, W = cost.shape
    p = BwdParams()
    keep = _set_planes(p, (("cost", cost), ("start", start), ("goal", goal), ("obst", obst)))
    gh, p.grad_histories, p.grad_stride = _plane(grad_hist.detach().to(torch.float32))
    gr, omg, sq = host_scalars(g_ratio, W)
    p.B, p.H, p.W = B, H, W
    p.g_ratio, p.one_minus_g_ratio, p.sqrt_w = gr, omg, sq
    p.T_batch = T_batch.data_ptr()
    p.t_solve = t_solve.data_ptr()
    with _on_device(dev) as stream:
        grad_cost = torch.empty((B, 1, H, W), dtype=torch.float32, device=dev)
        ws_bytes = L.nastar_b200_backward_workspace_bytes(B, H, W)
        ws = torch.empty((ws_bytes,), dtype=torch.uint8, device=dev) if ws_bytes else None
        p.grad_cost = grad_cost.data_ptr()
        p.workspace = ws.data_ptr() if ws is not None else None
        p.workspace_bytes = ws_bytes
        _check(L.nastar_b200_backward_mech(ctypes.byref(p), mech, stream), "nastar_b200_backward_mech")
    del keep
    return grad_cost


def check_lambda(lam: float) -> float:
    """The black-box backward's lambda as the fp32 value the library receives, or a ValueError when that value is not
    finite or not > 0."""
    with np.errstate(over="ignore"):
        lam32 = float(np.float32(lam))
    if not (math.isfinite(lam32) and lam32 > 0.0):
        raise ValueError(f"the black-box lambda must be a finite float32 > 0 (got {lam!r})")
    return lam32


def backward_blackbox(cost: torch.Tensor, start: torch.Tensor, goal: torch.Tensor, obst: torch.Tensor,
                      hist: torch.Tensor, grad_hist: torch.Tensor, lam: float, g_ratio: float, T: int, *,
                      mechanism: str = "moore", coupled: bool = False) -> torch.Tensor:
    """dL/dcost [B,1,H,W] of the black-box backward (BB-A*, include/nastar_b200.h, nastar_b200_backward_blackbox):
    (y(w') - hist) / lam with w' = fl(cost + fl(lam * grad_hist)) and y the histories of the same search on w'.
    `hist` [B,1,H,W] are the forward's histories for `cost`; the planes are those of `forward` (channel 0 of `cost` is
    searched).  `coupled` = False: each map of the search on w' stops at its solve step, one launch (the forward without
    flags, exact for g_ratio >= 0.5 or one map).  `coupled` = True: the batch-coupled search of `forward_coupled` with
    cap `T`, its T_batch decided on the device, three launches.  Asynchronous on the current stream, no host
    synchronisation."""
    lam = check_lambda(lam)
    p, keep, B, H, W, dev = _search_params(cost, start, goal, obst, g_ratio, T, 0, COST_PLANE, 1.0, 0.0, mechanism)
    for name, t_ in (("hist", hist), ("grad_hist", grad_hist)):
        if t_.device != dev:
            raise RuntimeError("all planes must live on the same CUDA device")
        if t_.shape[0] != B or t_.shape[-2:] != (H, W):
            raise ValueError(f"{name} must be [B,1,H,W] like the search planes")
    if hist.dtype != torch.float32:
        raise TypeError("hist must be the forward's float32 histories")
    hk = hist.detach().reshape(B, H * W).contiguous()
    gk, g_ptr, g_stride = _plane(grad_hist.detach().to(torch.float32))
    L = lib()
    if coupled:
        key = (B, H, W, int(T))
        ws_bytes = _coupled_ws_cache.get(key)
        if ws_bytes is None:
            ws_bytes = _coupled_ws_cache[key] = int(L.nastar_b200_forward_coupled_workspace_bytes(B, H, W, int(T)))
    else:
        ws_bytes = _ws_cache.get((B, H, W))
        if ws_bytes is None:
            ws_bytes = _ws_cache[(B, H, W)] = int(L.nastar_b200_forward_workspace_bytes(B, H, W))
    with _on_device(dev) as stream:
        grad_cost = torch.empty((B, 1, H, W), dtype=torch.float32, device=dev)
        # coupled: the search on w' gets its own T_batch [1] and goal clamp [B] (the second is not needed here)
        rec = torch.empty((B + 1,), dtype=torch.int32, device=dev) if coupled else None
        ws = torch.empty((ws_bytes,), dtype=torch.uint8, device=dev) if ws_bytes else None
        p.workspace = ws.data_ptr() if ws is not None else None
        p.workspace_bytes = ws_bytes
        _check(L.nastar_b200_backward_blackbox(ctypes.byref(p), hk.data_ptr(), g_ptr, g_stride, lam,
                                               grad_cost.data_ptr(), rec[:1].data_ptr() if coupled else None,
                                               rec[1:].data_ptr() if coupled else None, stream),
               "nastar_b200_backward_blackbox")
    del keep, hk, gk
    return grad_cost


# struct nastar_deflate_desc (include/nastar_b200.h) as a NumPy record
DEFLATE_DESC_DTYPE = np.dtype([("head", "<u8"), ("head_len", "<i8"), ("data", "<u8"), ("data_len", "<i8"),
                               ("gap", "<i8"), ("chunk0", "<i8")])
DEFLATE_CHUNK = 256 * 1024   # nastar_deflate.cuh kDeflateChunk


def deflate_chunk_counts(data_len) -> np.ndarray:
    """Chunks of each member: its head, then ceil(data_len / DEFLATE_CHUNK)."""
    n = np.asarray(data_len, dtype=np.int64)
    return 1 + (n + DEFLATE_CHUNK - 1) // DEFLATE_CHUNK


def deflate(desc, desc_dev: torch.Tensor, tail: int = 0):
    """Raw deflate streams of the members in one kernel (include/nastar_b200.h, nastar_b200_deflate).

    desc: a NumPy array of DEFLATE_DESC_DTYPE (the host copy, checked before the launch; head / data are device
    addresses); desc_dev: the same descriptors' bytes in device memory (a uint8 CUDA tensor).  Returns (out uint8
    [bound + tail], out_off int64 [M], out_len int64 [M], crc int32 [M] (the CRC-32's bits)) on the current stream;
    nothing is read back.  `tail` bytes after the bound are left for the caller (a PNG's last trailer)."""
    L = lib()
    d = np.ascontiguousarray(desc, dtype=DEFLATE_DESC_DTYPE)
    if not isinstance(desc_dev, torch.Tensor) or not desc_dev.is_cuda:
        raise RuntimeError("deflate: desc_dev must be a CUDA tensor (there is no CPU fallback)")
    if desc_dev.dtype != torch.uint8 or not desc_dev.is_contiguous() or desc_dev.numel() != d.nbytes:
        raise ValueError(f"deflate: desc_dev must be {d.nbytes} contiguous uint8 bytes")
    bound = int(L.nastar_b200_deflate_bound(d.ctypes.data, len(d)))
    if bound < 0:
        raise ValueError("deflate: invalid descriptors")
    dev = desc_dev.device
    ws_bytes = int(L.nastar_b200_deflate_workspace_bytes(d.ctypes.data, len(d)))
    with _on_device(dev) as stream:
        out = torch.empty((max(bound + int(tail), 1),), dtype=torch.uint8, device=dev)
        ws = torch.empty((ws_bytes,), dtype=torch.uint8, device=dev)
        out_off = torch.empty((len(d),), dtype=torch.int64, device=dev)
        out_len = torch.empty((len(d),), dtype=torch.int64, device=dev)
        crc = torch.empty((len(d),), dtype=torch.int32, device=dev)
        _check(L.nastar_b200_deflate(d.ctypes.data, desc_dev.data_ptr(), len(d), out.data_ptr(), bound + int(tail),
                                     out_off.data_ptr(), out_len.data_ptr(), crc.data_ptr(), ws.data_ptr(), ws_bytes,
                                     stream), "nastar_b200_deflate")
    return out, out_off, out_len, crc


# struct nastar_png_enc_desc (include/nastar_b200.h) as a NumPy record
PNG_ENC_DESC_DTYPE = np.dtype([("pixels", "<u8"), ("filt_off", "<i8"), ("W", "<i4"), ("H", "<i4")])
PNG_ENC_HEAD, PNG_ENC_TAIL = 43, 20   # the bytes of a file before and after its deflate stream


def png_gaps(B: int) -> np.ndarray:
    """nastar_b200_png_gap of images 0 .. B-1: the deflate gap before each image's stream."""
    return np.where(np.arange(B) > 0, PNG_ENC_HEAD + PNG_ENC_TAIL, PNG_ENC_HEAD).astype(np.int64)


def png_encode_bound(desc) -> int:
    """nastar_b200_png_encode_bound of a NumPy array of PNG_ENC_DESC_DTYPE descriptors (-1 when they are rejected)."""
    d = np.ascontiguousarray(desc, dtype=PNG_ENC_DESC_DTYPE)
    return int(lib().nastar_b200_png_encode_bound(d.ctypes.data, len(d)))


def png_filter(desc, desc_dev: torch.Tensor, filt: torch.Tensor) -> torch.Tensor:
    """The first PNG encode launch (include/nastar_b200.h, nastar_b200_png_filter): every image's filtered scanlines
    into `filt` (a uint8 CUDA tensor) at its filt_off.  desc: a NumPy array of PNG_ENC_DESC_DTYPE (the host copy,
    checked before the launch); desc_dev: the same descriptors' bytes in device memory.  Returns the Adler-32s, int32
    [B] (their bits), on the current stream."""
    L = lib()
    d = np.ascontiguousarray(desc, dtype=PNG_ENC_DESC_DTYPE)
    if not filt.is_cuda or filt.dtype != torch.uint8 or not desc_dev.is_cuda:
        raise RuntimeError("png_filter: filt and desc_dev must be CUDA tensors (there is no CPU fallback)")
    if desc_dev.dtype != torch.uint8 or not desc_dev.is_contiguous() or desc_dev.numel() != d.nbytes:
        raise ValueError(f"png_filter: desc_dev must be {d.nbytes} contiguous uint8 bytes")
    with _on_device(filt.device) as stream:
        adler = torch.empty((len(d),), dtype=torch.int32, device=filt.device)
        _check(L.nastar_b200_png_filter(d.ctypes.data, desc_dev.data_ptr(), len(d), filt.data_ptr(), filt.numel(),
                                        adler.data_ptr(), stream), "nastar_b200_png_filter")
    return adler


def png_finish(desc, desc_dev: torch.Tensor, out_off: torch.Tensor, out_len: torch.Tensor, adler: torch.Tensor,
               out: torch.Tensor) -> None:
    """The third PNG encode launch (nastar_b200_png_finish): each file's head and tail around its deflate stream in
    `out`, on the current stream."""
    L = lib()
    d = np.ascontiguousarray(desc, dtype=PNG_ENC_DESC_DTYPE)
    with _on_device(out.device) as stream:
        _check(L.nastar_b200_png_finish(d.ctypes.data, desc_dev.data_ptr(), len(d), out_off.data_ptr(),
                                        out_len.data_ptr(), adler.data_ptr(), out.data_ptr(), out.numel(), stream),
               "nastar_b200_png_finish")


# struct nastar_rgb_image / nastar_rgb_crop (include/nastar_b200.h) as NumPy records
RGB_IMAGE_DTYPE = np.dtype([("pixels", "<u8"), ("pitch", "<i8"), ("W", "<i4"), ("H", "<i4")])
RGB_CROP_DTYPE = np.dtype([("src", "<i4"), ("out", "<i4"), ("x0", "<i4"), ("y0", "<i4"), ("x1", "<i4"),
                           ("y1", "<i4")])
CROP_MAX_SIDE = 4096   # source and box sides
CROP_MAX_OUT = 1024    # Ho, Wo


def crop_resize_rgb(images, src, boxes, Ho: int, Wo: int) -> torch.Tensor:
    """RGB crops resized to Wo x Ho in one kernel (include/nastar_b200.h, nastar_b200_crop_resize_rgb), bit-equal to
    Pillow's image.crop(box).resize((Wo, Ho)).

    images: S uint8 CUDA tensors [H,W,3] on one device (rows may be strided; pixels within a row contiguous); src:
    int [N] source indices; boxes: int [N,4] (x0, y0, x1, y1), past any edge allowed.  Returns uint8 [N,Ho,Wo,3] on
    the current stream.  The CTAs take the crops in descending box area, so the largest start first."""
    L = lib()
    images = list(images)
    if not images or any(not isinstance(t, torch.Tensor) or not t.is_cuda or t.dtype != torch.uint8 for t in images):
        raise RuntimeError("crop_resize_rgb: uint8 CUDA images only (there is no CPU fallback)")
    dev = images[0].device
    keep = []
    img = np.zeros(len(images), RGB_IMAGE_DTYPE)
    for i, t in enumerate(images):
        if t.ndim != 3 or t.shape[2] != 3 or t.device != dev:
            raise ValueError(f"crop_resize_rgb: images are [H,W,3] on one device (image {i}: {tuple(t.shape)})")
        if t.stride(2) != 1 or t.stride(1) != 3:
            t = t.contiguous()
        keep.append(t)
        img[i] = (t.data_ptr(), t.stride(0), t.shape[1], t.shape[0])
    src = np.asarray(src, np.int64).reshape(-1)
    boxes = np.asarray(boxes, np.int64).reshape(-1, 4)
    N = len(src)
    if len(boxes) != N or N == 0:
        raise ValueError(f"crop_resize_rgb: one box per source index, at least one (got {len(boxes)} and {N})")
    if boxes.min() < -2 ** 31 or boxes.max() >= 2 ** 31:
        raise ValueError("crop_resize_rgb: box coordinates must fit int32")
    area = (boxes[:, 2] - boxes[:, 0]) * (boxes[:, 3] - boxes[:, 1])
    order = np.argsort(-area, kind="stable")
    crops = np.zeros(N, RGB_CROP_DTYPE)
    crops["src"], crops["out"] = src[order], order
    crops["x0"], crops["y0"], crops["x1"], crops["y1"] = boxes[order].T
    ctl = torch.empty((img.nbytes + crops.nbytes,), dtype=torch.uint8, pin_memory=True)
    c = ctl.numpy()
    c[:img.nbytes] = img.view(np.uint8)
    c[img.nbytes:] = crops.view(np.uint8)
    with _on_device(dev) as stream:
        ctl_dev = torch.empty((ctl.numel(),), dtype=torch.uint8, device=dev)
        ctl_dev.copy_(ctl, non_blocking=True)
        out = torch.empty((N, int(Ho), int(Wo), 3), dtype=torch.uint8, device=dev)
        _check(L.nastar_b200_crop_resize_rgb(img.ctypes.data, ctl_dev.data_ptr(), len(img), crops.ctypes.data,
                                             ctl_dev.data_ptr() + img.nbytes, N, int(Ho), int(Wo), out.data_ptr(),
                                             stream), "nastar_b200_crop_resize_rgb")
    del keep
    return out


# NASTAR_GIF_* (include/nastar_b200.h)
GIF_EACH, GIF_GRID = 0, 1
GIF_STEPS_MAP, GIF_STEPS_BATCH, GIF_STEPS_ALL = 0, 1, 2


def gif_params(maps, hist, paths, goal, trace, t_solve, layout: int, steps_mode: int, screen_w: int, screen_h: int,
               delay_cs: int):
    """GifParams of a search's planes ([B,1,H,W] CUDA tensors: fp32 maps, histories and goals, int64 paths; trace
    [B,T] and t_solve [B] int32), without the tables.  Returns (params, tensors to keep alive)."""
    planes = [t.detach().contiguous() for t in (maps, hist, paths, goal, trace, t_solve)]
    if any(not t.is_cuda or t.device != planes[0].device for t in planes):
        raise RuntimeError("gif: every tensor must be on one CUDA device (there is no CPU fallback)")
    dtypes = (torch.float32, torch.float32, torch.int64, torch.float32, torch.int32, torch.int32)
    if any(t.dtype != d for t, d in zip(planes, dtypes)):
        raise TypeError("gif: maps, histories, goals fp32; paths int64; trace and t_solve int32")
    B, _, H, W = planes[0].shape
    p = GifParams()
    p.maps, p.histories, p.paths, p.goal_maps, p.trace, p.t_solve = (t.data_ptr() for t in planes)
    p.B, p.H, p.W, p.T = B, H, W, planes[4].shape[1]
    p.layout, p.steps_mode = layout, steps_mode
    p.screen_w, p.screen_h, p.delay_cs = screen_w, screen_h, delay_cs
    return p, planes


def gif_tables_bytes(p: GifParams) -> int:
    return int(lib().nastar_b200_gif_tables_bytes(ctypes.byref(p)))


def gif_record_bytes(lzw_bytes) -> np.ndarray:
    """nastar_b200_gif_record_bytes, vectorised: each frame's record around an LZW stream of lzw_bytes."""
    n = np.asarray(lzw_bytes, dtype=np.int64)
    return 19 + n + (n + 254) // 255 + 1


def gif_plan(p: GifParams, dev: torch.device):
    """The first GIF launch (nastar_b200_gif_plan).  p.tables must point at the device tables.  Returns (steps int32
    [G], nbytes int32 [G*(T+1)], workspace) on the current stream; nothing is read back."""
    L = lib()
    G = 1 if p.layout == GIF_GRID else p.B
    ws_bytes = int(L.nastar_b200_gif_workspace_bytes(ctypes.byref(p)))
    with _on_device(dev) as stream:
        steps = torch.empty((G,), dtype=torch.int32, device=dev)
        nbytes = torch.empty((G * (p.T + 1),), dtype=torch.int32, device=dev)
        ws = torch.empty((max(ws_bytes, 1),), dtype=torch.uint8, device=dev)
        _check(L.nastar_b200_gif_plan(ctypes.byref(p), steps.data_ptr(), nbytes.data_ptr(), ws.data_ptr(), ws_bytes,
                                      stream), "nastar_b200_gif_plan")
    return steps, nbytes, ws


def gif_encode(p: GifParams, nbytes: torch.Tensor, nbytes_host: np.ndarray, offset_host: np.ndarray,
               offset_dev: torch.Tensor, ws: torch.Tensor) -> torch.Tensor:
    """The second GIF launch (nastar_b200_gif_encode): every frame's record, frame f at offset_host[f].  Returns out
    uint8 [offset_host[-1]] on the current stream."""
    L = lib()
    nb = np.ascontiguousarray(nbytes_host, dtype=np.int32)
    off = np.ascontiguousarray(offset_host, dtype=np.int64)
    if len(off) != len(nb) + 1 or offset_dev.dtype != torch.int64 or offset_dev.numel() != len(off):
        raise ValueError("gif_encode: offsets are one more than the frames, int64")
    dev = nbytes.device
    with _on_device(dev) as stream:
        out = torch.empty((max(int(off[-1]), 1),), dtype=torch.uint8, device=dev)
        _check(L.nastar_b200_gif_encode(ctypes.byref(p), nbytes.data_ptr(), nb.ctypes.data, off.ctypes.data,
                                        offset_dev.data_ptr(), len(nb), out.data_ptr(), int(off[-1]), ws.data_ptr(),
                                        ws.numel(), stream), "nastar_b200_gif_encode")
    return out


# struct nastar_inflate_desc (include/nastar_b200.h) as a NumPy record
INFLATE_DESC_DTYPE = np.dtype([("in_off", "<i8"), ("in_len", "<i8"), ("out_off", "<i8"), ("out_len", "<i8"),
                               ("method", "<i4"), ("reserved", "<i4")])
INFLATE_WORKSPACE_BYTES = 256
# status bits of nastar_b200_inflate
INFLATE_STATUS = {2: "bad block type or Huffman code", 4: "distance past the start of the output",
                  8: "stream ends early or inflates to the wrong size"}


def inflate(data: torch.Tensor, desc, desc_dev: torch.Tensor, out: torch.Tensor):
    """Zip members to their bytes in one kernel (include/nastar_b200.h, nastar_b200_inflate): member i of `desc` (a
    NumPy array of INFLATE_DESC_DTYPE, the host copy checked before the launch) from `data` into `out` (1-D uint8 CUDA
    tensors); desc_dev: the same descriptors' bytes in device memory.  Returns (status int32 [M], crc int32 [M] (the
    CRC-32's bits)) on the current stream; nothing is read back."""
    L = lib()
    d = np.ascontiguousarray(desc, dtype=INFLATE_DESC_DTYPE)
    if any(not t.is_cuda or t.dtype != torch.uint8 or t.ndim != 1 for t in (data, out, desc_dev)):
        raise RuntimeError("inflate: data, out and desc_dev must be 1-D uint8 CUDA tensors (there is no CPU fallback)")
    if not desc_dev.is_contiguous() or desc_dev.numel() != d.nbytes or desc_dev.device != data.device:
        raise ValueError(f"inflate: desc_dev must be {d.nbytes} contiguous uint8 bytes on the data's device")
    dev = data.device
    with _on_device(dev) as stream:
        status = torch.empty((len(d),), dtype=torch.int32, device=dev)
        crc = torch.empty((len(d),), dtype=torch.int32, device=dev)
        ws = torch.empty((INFLATE_WORKSPACE_BYTES,), dtype=torch.uint8, device=dev)
        _check(L.nastar_b200_inflate(data.data_ptr(), data.numel(), d.ctypes.data, desc_dev.data_ptr(), len(d),
                                     out.data_ptr(), out.numel(), status.data_ptr(), crc.data_ptr(), ws.data_ptr(),
                                     INFLATE_WORKSPACE_BYTES, stream), "nastar_b200_inflate")
    return status, crc


CHAMFER_MAX_SIDE = 1024


def chamfer(masks: torch.Tensor) -> torch.Tensor:
    """Directed Chamfer distances in one kernel (include/nastar_b200.h, nastar_b200_chamfer): masks is a uint8 CUDA
    tensor [B,H,W] with bit 0 = set A and bit 1 = set B.  Returns fp64 [B,2] (d(A -> B), d(B -> A)) on the current
    stream."""
    L = lib()
    if not masks.is_cuda or masks.dtype != torch.uint8 or masks.ndim != 3:
        raise RuntimeError("chamfer: masks must be a uint8 CUDA tensor [B,H,W] (there is no CPU fallback)")
    masks = masks.contiguous()
    B, H, W = masks.shape
    dev = masks.device
    ws_bytes = int(L.nastar_b200_chamfer_workspace_bytes(B, H, W))
    with _on_device(dev) as stream:
        out = torch.empty((B, 2), dtype=torch.float64, device=dev)
        ws = torch.empty((ws_bytes,), dtype=torch.uint8, device=dev) if ws_bytes else None
        _check(L.nastar_b200_chamfer(masks.data_ptr(), B, H, W, out.data_ptr(), ws.data_ptr() if ws is not None else None,
                                     ws_bytes, stream), "nastar_b200_chamfer")
    return out
