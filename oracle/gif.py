"""ctypes front-end of the CPU oracle of the search GIFs (oracle/gif_oracle.c).

TEST / BASELINE INFRASTRUCTURE ONLY: imported by tests/ and tools/; the product package never imports this module.
"""
from __future__ import annotations

import ctypes
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_SRC = os.path.join(_HERE, "gif_oracle.c")
_LIB_PATH = os.path.join(_HERE, "libgif_oracle.so")
_CC = ["/usr/bin/gcc", "-O2", "-fPIC", "-Wall", "-Wextra", "-std=c11"]
_lib = None


def build(force: bool = False) -> str:
    """Compile the oracle with gcc (well under a second)."""
    if force or not os.path.exists(_LIB_PATH) or os.path.getmtime(_LIB_PATH) < os.path.getmtime(_SRC):
        subprocess.check_call(_CC + ["-shared", "-o", _LIB_PATH, _SRC])
    return _LIB_PATH


def _load():
    global _lib
    if _lib is None:
        build()
        lib = ctypes.CDLL(_LIB_PATH)
        p = ctypes.c_void_p
        lib.nastar_oracle_gif.argtypes = [p] * 5 + [ctypes.c_int] * 8 + [p, p] + [ctypes.c_int] * 3 + [p,
                                                                                                     ctypes.c_int64]
        lib.nastar_oracle_gif.restype = ctypes.c_int64
        _lib = lib
    return _lib


def index_map(n_in: int, n_out: int) -> np.ndarray:
    """Source index of each of n_out samples of Pillow's NEAREST resize from n_in, read from Pillow."""
    if n_in == n_out:
        return np.arange(n_in, dtype=np.int32)
    from PIL import Image

    row = Image.fromarray(np.arange(n_in, dtype=np.int32)[None, :])
    return np.asarray(row.resize((n_out, 1), resample=Image.NEAREST), dtype=np.int32)[0]


def gif(maps, histories, paths, trace, goal_idx, steps: int, grid: bool = False, scale: int = 4, fps: float = 30,
        hold: int = 15, loop: int = 0) -> bytes:
    """One GIF of a search record: maps / histories / paths [n,1,H,W] (or [n,H,W]), trace [n,T] int, goal_idx [n];
    `steps` frames from the trace, then the final frame, then `hold` copies.  With grid (and n > 1) the maps are tiled
    like make_grid.  Screen: the image enlarged to (rows * scale, cols * scale) as Pillow's (width, height)."""
    maps = np.asarray(maps, np.float32)
    n, H, W = maps.shape[0], maps.shape[-2], maps.shape[-1]
    grey = (maps.reshape(n, H * W) * np.float32(255)).astype(np.uint8)
    hist = (np.asarray(histories).reshape(n, H * W) == 1).astype(np.uint8)
    path = (np.asarray(paths).reshape(n, H * W) == 1).astype(np.uint8)
    tr = np.ascontiguousarray(np.asarray(trace).reshape(n, -1), np.int32)
    goal = np.ascontiguousarray(np.asarray(goal_idx).reshape(n), np.int32)
    if grid and n > 1:
        xm = min(8, n)
        Hi, Wi = (H + 2) * (-(-n // xm)) + 2, (W + 2) * xm + 2
    else:
        Hi, Wi = H, W
    SW, SH = (Hi * scale, Wi * scale) if scale > 1 else (Wi, Hi)
    xmap, ymap = index_map(Wi, SW), index_map(Hi, SH)
    args = [grey, hist, path, tr, goal]
    lib = _load()
    call = lambda out, cap: lib.nastar_oracle_gif(  # noqa: E731
        *[a.ctypes.data for a in args], n, H, W, tr.shape[1], int(steps), int(bool(grid)), SW, SH, xmap.ctypes.data,
        ymap.ctypes.data, round(100 / fps), int(hold), int(loop), out, cap)
    size = call(None, 0)
    if size < 0:
        raise ValueError("more than 256 palette entries")
    out = np.zeros(size, np.uint8)
    call(out.ctypes.data, size)
    return out.tobytes()
