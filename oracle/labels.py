"""ctypes front-end of the CPU label oracle (oracle/labels_oracle.c), and the staging of the planning-datasets
generator's own dijkstra_dist for the CPU timing arm of tools/labels_bench.py.

TEST / BASELINE INFRASTRUCTURE ONLY: imported by tests/, tests/golden/make_golden_labels.py and tools/; the product
package never imports this module.
"""
from __future__ import annotations

import ctypes
import filecmp
import os
import shutil
import subprocess

import numpy as np

from .oracle import mechanism_code

_HERE = os.path.dirname(os.path.abspath(__file__))
_SRC = os.path.join(_HERE, "labels_oracle.c")
_LIB_PATH = os.path.join(_HERE, "liblabels_oracle.so")
# same compiler and flags as oracle/Makefile (the image's default CC lacks libgomp.spec)
_CC = ["/usr/bin/gcc", "-O2", "-fPIC", "-fopenmp", "-ffp-contract=off", "-fno-fast-math", "-Wall", "-Wextra", "-std=c11",
       "-I" + os.path.join(os.path.dirname(_HERE), "include")]
_lib = None

# build output, git-ignored like the rest of oracle/_ref: the generator's modules, byte for byte, imported as the
# top-level modules `dijkstra` and `mechanism` (their package __init__ pulls in data.py, which needs natsort, skimage,
# PIL and tqdm)
REF_UTILS = "/root/reference/planning-datasets/planning_datasets_utils"
REF_STAGE = os.path.join(_HERE, "_ref", "planning_datasets")
REF_FILES = ("dijkstra.py", "mechanism.py")


def build(force: bool = False) -> str:
    """Compile the oracle with gcc (well under a second)."""
    if force or not os.path.exists(_LIB_PATH) or os.path.getmtime(_LIB_PATH) < os.path.getmtime(_SRC):
        subprocess.check_call(_CC + ["-shared", "-o", _LIB_PATH, _SRC])
    return _LIB_PATH


def stage_reference() -> bool:
    """Copy the generator's dijkstra.py / mechanism.py into oracle/_ref/planning_datasets where a reference checkout
    exists; elsewhere report whether a staged copy is present."""
    if not os.path.isdir(REF_UTILS):
        return os.path.isdir(REF_STAGE)
    os.makedirs(REF_STAGE, exist_ok=True)
    for f in REF_FILES:
        a, b = os.path.join(REF_UTILS, f), os.path.join(REF_STAGE, f)
        if not os.path.exists(b) or not filecmp.cmp(a, b, shallow=False):
            shutil.copyfile(a, b)
    return True


def _load():
    global _lib
    if _lib is None:
        build()
        lib = ctypes.CDLL(_LIB_PATH)
        lib.nastar_oracle_opt_labels.argtypes = [ctypes.POINTER(ctypes.c_float), ctypes.POINTER(ctypes.c_int32),
                                                 ctypes.c_int, ctypes.c_int, ctypes.c_int,
                                                 ctypes.POINTER(ctypes.c_float), ctypes.POINTER(ctypes.c_uint8),
                                                 ctypes.POINTER(ctypes.c_int8), ctypes.c_int]
        lib.nastar_oracle_opt_labels.restype = ctypes.c_int
        _lib = lib
    return _lib


def _p(a, ty):
    return a.ctypes.data_as(ctypes.POINTER(ty))


def opt_labels(maps, goal_idx, mechanism="moore"):
    """Labels of the planning-datasets generator for maps [B,H,W] or [B,1,H,W] (passable iff != 0) and flat goal
    indices [B]: (dists float32 [B,1,H,W], act_mask uint8 [B,1,H,W], action int8 [B,1,H,W]), see labels_oracle.c.
    mechanism "moore" has 8 actions, "news" the 4 actions N, E, W, S."""
    mech = mechanism_code(mechanism)
    lib = _load()
    m = np.asarray(maps, dtype=np.float32)
    if m.ndim == 4:
        m = m[:, 0]
    m = np.ascontiguousarray(m)
    B, H, W = m.shape
    g = np.ascontiguousarray(np.asarray(goal_idx, dtype=np.int32).reshape(B))
    dists = np.empty((B, 1, H, W), np.float32)
    mask = np.empty((B, 1, H, W), np.uint8)
    action = np.empty((B, 1, H, W), np.int8)
    rc = lib.nastar_oracle_opt_labels(_p(m, ctypes.c_float), _p(g, ctypes.c_int32), B, H, W, _p(dists, ctypes.c_float),
                                      _p(mask, ctypes.c_uint8), _p(action, ctypes.c_int8), mech)
    if rc != 0:
        raise RuntimeError(f"labels oracle returned {rc}")
    return dists, mask, action
