"""ctypes front-end of the CPU oracle (oracle/astar_oracle.c).

TEST INFRASTRUCTURE ONLY: imported by tests/, __graft_entry__.smoke() and bench.py's
cpu_baseline / --impl reference legs.  The product package never imports this module.

Restates /root/reference/src/neural_astar/planner/differentiable_astar.py:150-267
(see the C file's header for the per-function map).
"""
from __future__ import annotations

import ctypes
import math
import os
import subprocess
from typing import NamedTuple, Optional

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB_PATH = os.path.join(_HERE, "libastar_oracle.so")
_lib = None
MECHANISMS = {"moore": 0, "news": 1}   # NASTAR_MECH_MOORE / NASTAR_MECH_NEWS (include/nastar_b200.h)


def mechanism_code(mechanism: str) -> int:
    """The NASTAR_MECH_* value of "moore" or "news"; anything else is a ValueError."""
    if mechanism not in MECHANISMS:
        raise ValueError(f"mechanism must be one of {sorted(MECHANISMS)} (got {mechanism!r})")
    return MECHANISMS[mechanism]


def build(force: bool = False) -> str:
    """Compile the oracle with gcc (a few hundred ms)."""
    src = os.path.join(_HERE, "astar_oracle.c")
    if force or not os.path.exists(_LIB_PATH) or os.path.getmtime(_LIB_PATH) < os.path.getmtime(src):
        subprocess.check_call(["make", "-s", "-C", _HERE, "-B", "libastar_oracle.so"])
    return _LIB_PATH


def _load():
    global _lib
    if _lib is None:
        build()
        lib = ctypes.CDLL(_LIB_PATH)
        fp = ctypes.POINTER(ctypes.c_float)
        ip = ctypes.POINTER(ctypes.c_int32)
        lp = ctypes.POINTER(ctypes.c_int64)
        lib.nastar_oracle_forward_literal.argtypes = [fp, fp, fp, fp, ctypes.c_int, ctypes.c_int, ctypes.c_int,
                                                      ctypes.c_float, ctypes.c_float, ctypes.c_float, ctypes.c_int,
                                                      fp, lp, ip, ip, ip, ctypes.c_int]
        lib.nastar_oracle_forward_literal.restype = ctypes.c_int
        lib.nastar_oracle_forward_spec.argtypes = [fp, fp, fp, fp, ctypes.c_int, ctypes.c_int, ctypes.c_int,
                                                   ctypes.c_float, ctypes.c_float, ctypes.c_int, ctypes.c_int,
                                                   fp, lp, ip, ip, ip, ctypes.c_int]
        lib.nastar_oracle_forward_spec.restype = ctypes.c_int
        lib.nastar_oracle_backward.argtypes = [fp, fp, fp, fp, fp, ctypes.c_int, ctypes.c_int, ctypes.c_int,
                                               ctypes.c_float, ctypes.c_float, ctypes.c_float, ctypes.c_int,
                                               ctypes.POINTER(ctypes.c_double), ctypes.c_int]
        lib.nastar_oracle_backward.restype = ctypes.c_int
        lib.nastar_oracle_backward_bound.argtypes = [fp, fp, fp, fp, fp, ctypes.c_int, ctypes.c_int, ctypes.c_int,
                                                     ctypes.c_float, ctypes.c_float, ctypes.c_float, ctypes.c_int,
                                                     ctypes.c_int, ctypes.POINTER(ctypes.c_double),
                                                     ctypes.POINTER(ctypes.c_double), ctypes.c_int]
        lib.nastar_oracle_backward_bound.restype = ctypes.c_int
        lib.nastar_oracle_num_threads.restype = ctypes.c_int
        lib.nastar_oracle_set_threads.argtypes = [ctypes.c_int]
        _lib = lib
    return _lib


class OracleOutput(NamedTuple):
    histories: np.ndarray  # [B,1,H,W] float32
    paths: np.ndarray  # [B,1,H,W] int64
    t_solve: np.ndarray  # [B] int32
    n_steps: np.ndarray  # [B] int32 (spec) / T_batch broadcast (literal)
    T_batch: int
    trace: Optional[np.ndarray]  # [B,T] int32 or None


def _planes(x) -> np.ndarray:
    a = np.asarray(x, dtype=np.float32)
    assert a.ndim == 4, "planes are [B,1,H,W] (differentiable_astar.py:172-175)"
    return np.ascontiguousarray(a[:, 0])


def _p(a, ty):
    return a.ctypes.data_as(ctypes.POINTER(ty))


def scalars(g_ratio: float, W: int):
    """Host-side scalar preparation exactly as the reference does it in Python doubles
    (differentiable_astar.py:206-207) before ATen casts them to fp32."""
    return np.float32(g_ratio), np.float32(1 - g_ratio), np.float32(math.sqrt(W))


def num_steps(Tmax: float, training: bool, W: int) -> int:
    """differentiable_astar.py:200-202"""
    return int((Tmax if training else 1.0) * W * W)


MAX_STEPS = 2**31 - 1   # the C oracle takes the loop bound as a C int


def check_steps(T: int) -> int:
    """int(T), refused with a ValueError above 2**31 - 1 rather than truncated by ctypes into a wrong bound."""
    T = int(T)
    if T > MAX_STEPS:
        raise ValueError(f"step bound {T} exceeds 2**31 - 1, the largest the oracle takes (W*W fits for W <= 46340)")
    return T


def forward(cost, start, goal, obst, g_ratio=0.5, Tmax=1.0, training=False, mode="spec",
            want_trace=False, T=None, no_early_exit=False, mechanism="moore") -> OracleOutput:
    """The search of DifferentiableAstar(mechanism=mechanism): "moore" (8 neighbours, Chebyshev heuristic) or "news"
    (N, E, W, S, Manhattan heuristic), in the LITERAL or SPEC form of astar_oracle.c."""
    mech = mechanism_code(mechanism)
    lib = _load()
    c, s, g, o = _planes(cost), _planes(start), _planes(goal), _planes(obst)
    B, H, W = c.shape
    T = check_steps(T if T is not None else num_steps(Tmax, training, W))
    gr, omg, sq = scalars(g_ratio, W)
    hist = np.zeros((B, H, W), np.float32)
    paths = np.zeros((B, H, W), np.int64)
    ts = np.zeros(B, np.int32)
    ns = np.zeros(B, np.int32)
    trace = np.full((B, T), -1, np.int32) if want_trace else None
    tp = _p(trace, ctypes.c_int32) if want_trace else None
    if mode == "literal":
        tb = ctypes.c_int32(0)
        rc = lib.nastar_oracle_forward_literal(_p(c, ctypes.c_float), _p(s, ctypes.c_float), _p(g, ctypes.c_float),
                                               _p(o, ctypes.c_float), B, H, W, gr, omg, sq, T,
                                               _p(hist, ctypes.c_float), _p(paths, ctypes.c_int64),
                                               _p(ts, ctypes.c_int32), tp, ctypes.byref(tb), mech)
        T_batch = int(tb.value)
        ns[:] = T_batch
    elif mode == "spec":
        rc = lib.nastar_oracle_forward_spec(_p(c, ctypes.c_float), _p(s, ctypes.c_float), _p(g, ctypes.c_float),
                                            _p(o, ctypes.c_float), B, H, W, gr, omg, T, int(bool(no_early_exit)),
                                            _p(hist, ctypes.c_float), _p(paths, ctypes.c_int64),
                                            _p(ts, ctypes.c_int32), _p(ns, ctypes.c_int32), tp, mech)
        T_batch = int(ns.max())
    else:
        raise ValueError(mode)
    if rc != 0:
        raise RuntimeError(f"oracle returned {rc}")
    return OracleOutput(hist[:, None], paths[:, None], ts, ns, T_batch, trace)


def backward(cost, start, goal, obst, grad_hist, T_batch: int, g_ratio=0.5, dtype=np.float32,
             mechanism="moore") -> np.ndarray:
    """Closed-form dL/dcost [B,1,H,W] for dL/dhistories = grad_hist.  The sums run in double; dtype=np.float64 returns
    them unrounded, np.float32 rounds each once."""
    mech = mechanism_code(mechanism)
    lib = _load()
    c, s, g, o, gh = _planes(cost), _planes(start), _planes(goal), _planes(obst), _planes(grad_hist)
    B, H, W = c.shape
    gr, omg, sq = scalars(g_ratio, W)
    T_batch = check_steps(T_batch)
    out = np.zeros((B, H, W), np.float64)
    rc = lib.nastar_oracle_backward(_p(c, ctypes.c_float), _p(s, ctypes.c_float), _p(g, ctypes.c_float),
                                    _p(o, ctypes.c_float), _p(gh, ctypes.c_float), B, H, W, gr, omg, sq,
                                    T_batch, _p(out, ctypes.c_double), mech)
    if rc != 0:
        raise RuntimeError(f"oracle returned {rc}")
    return out[:, None].astype(dtype)


def backward_with_bound(cost, start, goal, obst, grad_hist, T_batch: int, g_ratio=0.5, mechanism="moore",
                        model=False):
    """(want, M), both [B,1,H,W] float64: the closed-form dL/dcost of `backward`, unrounded, and per cell the bound M
    on |engine - want| from the fp32 rounding of the softmax numerators (derivation in astar_oracle.c,
    nastar_oracle_backward_bound).  model=True returns in place of `want` the closed form with the numerators rounded
    as the engines round them, expf(fl32(-f / sqrt(W))) in fp32; M is the same."""
    mech = mechanism_code(mechanism)
    lib = _load()
    c, s, g, o, gh = _planes(cost), _planes(start), _planes(goal), _planes(obst), _planes(grad_hist)
    B, H, W = c.shape
    gr, omg, sq = scalars(g_ratio, W)
    T_batch = check_steps(T_batch)
    out = np.zeros((B, H, W), np.float64)
    bound = np.zeros((B, H, W), np.float64)
    rc = lib.nastar_oracle_backward_bound(_p(c, ctypes.c_float), _p(s, ctypes.c_float), _p(g, ctypes.c_float),
                                          _p(o, ctypes.c_float), _p(gh, ctypes.c_float), B, H, W, gr, omg, sq,
                                          T_batch, int(bool(model)), _p(out, ctypes.c_double),
                                          _p(bound, ctypes.c_double), mech)
    if rc != 0:
        raise RuntimeError(f"oracle returned {rc}")
    return out[:, None], bound[:, None]


def set_threads(n: int) -> None:
    _load().nastar_oracle_set_threads(int(n))


def max_threads() -> int:
    return int(_load().nastar_oracle_num_threads())
