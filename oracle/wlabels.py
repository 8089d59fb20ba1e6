"""ctypes front-end of the CPU oracle of the vertex-weighted shortest-path labels (oracle/wlabels_oracle.c).

TEST / BASELINE INFRASTRUCTURE ONLY: imported by tests/ and tools/; the product package never imports this module.
"""
from __future__ import annotations

import ctypes
import os
import subprocess

import numpy as np

from .oracle import mechanism_code

_HERE = os.path.dirname(os.path.abspath(__file__))
_SRC = os.path.join(_HERE, "wlabels_oracle.c")
_LIB_PATH = os.path.join(_HERE, "libwlabels_oracle.so")
# the flags of oracle/labels.py: no FMA contraction, so every float add of the fold is rounded once
_CC = ["/usr/bin/gcc", "-O2", "-fPIC", "-fopenmp", "-ffp-contract=off", "-fno-fast-math", "-Wall", "-Wextra", "-std=c11",
       "-I" + os.path.join(os.path.dirname(_HERE), "include")]
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
        lib.nastar_oracle_weighted_labels.argtypes = [ctypes.c_void_p] * 4 + [ctypes.c_int] * 3 + [ctypes.c_void_p] * 7 + [
            ctypes.c_int]
        lib.nastar_oracle_weighted_labels.restype = ctypes.c_int
        _lib = lib
    return _lib


def _maps(x):
    a = np.asarray(x, dtype=np.float32)
    if a.ndim == 4:
        a = a[:, 0]
    return np.ascontiguousarray(a)


def weighted_labels(cost, goal_idx, passable=None, start_idx=None, mechanism="moore"):
    """Labels of cost maps [B,H,W] or [B,1,H,W] with flat goal (and optional start) indices [B], passable iff != 0
    (None: every cell), with the 8 moves of "moore" or the 4 moves N, E, W, S of "news".  Returns a dict of dists f32,
    hops i32, act_mask u8, action i8 (each [B,1,H,W]) and status i32 [B]; with starts also path_maps f32 [B,1,H,W]
    and path_costs f32 [B].  See wlabels_oracle.c."""
    mech = mechanism_code(mechanism)
    lib = _load()
    c = _maps(cost)
    B, H, W = c.shape
    p = None if passable is None else _maps(passable)
    if p is not None and p.shape != c.shape:
        raise ValueError("passable must have the cost maps' shape")
    g = np.ascontiguousarray(np.asarray(goal_idx, dtype=np.int32).reshape(B))
    s = None if start_idx is None else np.ascontiguousarray(np.asarray(start_idx, dtype=np.int32).reshape(B))
    out = dict(dists=np.empty((B, 1, H, W), np.float32), hops=np.empty((B, 1, H, W), np.int32),
               act_mask=np.empty((B, 1, H, W), np.uint8), action=np.empty((B, 1, H, W), np.int8),
               status=np.empty(B, np.int32))
    if s is not None:
        out["path_maps"] = np.empty((B, 1, H, W), np.float32)
        out["path_costs"] = np.empty(B, np.float32)

    def ptr(a):
        return None if a is None else a.ctypes.data

    rc = lib.nastar_oracle_weighted_labels(ptr(c), ptr(p), ptr(g), ptr(s), B, H, W, ptr(out["dists"]),
                                           ptr(out["hops"]), ptr(out["act_mask"]), ptr(out["action"]),
                                           ptr(out.get("path_maps")), ptr(out.get("path_costs")), ptr(out["status"]), mech)
    if rc != 0:
        raise RuntimeError(f"weighted labels oracle returned {rc}")
    return out
