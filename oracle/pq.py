"""ctypes front-end of the CPU oracle of the reference's heap A* (oracle/pq_oracle.c).

TEST / BASELINE INFRASTRUCTURE ONLY: imported by tests/ and tools/; the product package never imports this module.
"""
from __future__ import annotations

import ctypes
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_SRC = os.path.join(_HERE, "pq_oracle.c")
_LIB_PATH = os.path.join(_HERE, "libpq_oracle.so")
# the flags of oracle/labels.py: no FMA contraction, so every fp64 product and sum is rounded once
_CC = ["/usr/bin/gcc", "-O2", "-fPIC", "-fopenmp", "-ffp-contract=off", "-fno-fast-math", "-Wall", "-Wextra", "-std=c11"]
_lib = None


def build(force: bool = False) -> str:
    """Compile the oracle with gcc (well under a second)."""
    if force or not os.path.exists(_LIB_PATH) or os.path.getmtime(_LIB_PATH) < os.path.getmtime(_SRC):
        subprocess.check_call(_CC + ["-shared", "-o", _LIB_PATH, _SRC, "-lm"])
    return _LIB_PATH


def _load():
    global _lib
    if _lib is None:
        build()
        lib = ctypes.CDLL(_LIB_PATH)
        lib.nastar_oracle_pq_astar.argtypes = ([ctypes.c_void_p] * 4 + [ctypes.c_int] * 3 + [ctypes.c_double]
                                               + [ctypes.c_void_p] * 4)
        lib.nastar_oracle_pq_astar.restype = ctypes.c_int
        _lib = lib
    return _lib


def _maps(x):
    a = np.asarray(x, dtype=np.float32)
    if a.ndim == 4:
        a = a[:, 0]
    return np.ascontiguousarray(a)


def pq_astar(cost, start, goal, map_design, g_ratio: float = 0.5):
    """The reference's heap A* on maps [B,H,W] or [B,1,H,W] (cast to fp32).  Returns histories f32 [B,1,H,W], paths
    i64 [B,1,H,W], status i32 [B] (0 solved, 1 goal not found, 2 start or goal not one cell), expansions i32 [B]."""
    lib = _load()
    c, s, g, m = (_maps(x) for x in (cost, start, goal, map_design))
    B, H, W = c.shape
    if not (s.shape == g.shape == m.shape == c.shape):
        raise ValueError("cost, start, goal and map must have one shape")
    hist = np.empty((B, 1, H, W), np.float32)
    paths = np.empty((B, 1, H, W), np.int64)
    status = np.empty(B, np.int32)
    exp = np.empty(B, np.int32)
    rc = lib.nastar_oracle_pq_astar(c.ctypes.data, s.ctypes.data, g.ctypes.data, m.ctypes.data, B, H, W,
                                    float(g_ratio), hist.ctypes.data, paths.ctypes.data, status.ctypes.data,
                                    exp.ctypes.data)
    if rc != 0:
        raise RuntimeError(f"pq oracle returned {rc}")
    return hist, paths, status, exp
