"""NumPy + scipy.ndimage restatement of the GPU goal rule (csrc/nastar_goals.cuh, DESIGN.md §12), replaying the draws.

Per map: the largest 4-connected region of cells != 0 (ties to the region labelled first, i.e. whose first cell comes
first in raster order), its cells with (y < e or y >= H - e) and (x < e or x >= W - e) when there is one (else the
whole region), then candidate (d * count) >> 32 in raster order for the map's u32 draw d."""
import numpy as np
from scipy import ndimage

NO_PASSABLE = 1


def corner_mask(H, W, e):
    y, x = np.mgrid[0:H, 0:W]
    return ((y < e) | (y >= H - e)) & ((x < e) | (x >= W - e))


def candidates(m, e):
    """flat indices of the cells the goal is drawn from, in raster order (empty without a passable cell)"""
    lab, _ = ndimage.label(np.asarray(m) != 0)
    counts = np.bincount(lab.ravel())
    counts[0] = 0
    if counts.max() == 0:
        return np.zeros(0, np.int64)
    region = lab == np.argmax(counts)
    corner = region & corner_mask(*region.shape, e)
    return np.flatnonzero(corner if corner.any() else region)


def pick(n, d):
    return (int(d) & 0xFFFFFFFF) * n >> 32


def draw_for(k, n):
    """the smallest u32 draw that picks candidate k of n"""
    return -(-(k << 32) // n)


def sample(maps, e, draws):
    """(goal_idx int32 [B], goal_maps float32 [B,1,H,W], status int32 [B]) for maps [B,H,W] or [B,1,H,W]"""
    maps = np.asarray(maps)
    if maps.ndim == 4:
        maps = maps[:, 0]
    B, H, W = maps.shape
    goal_idx = np.full(B, -1, np.int32)
    goals = np.zeros((B, 1, H, W), np.float32)
    status = np.zeros(B, np.int32)
    for i in range(B):
        c = candidates(maps[i], e)
        if len(c) == 0:
            status[i] = NO_PASSABLE
            continue
        goal_idx[i] = c[pick(len(c), draws[i])]
        goals[i, 0].reshape(-1)[goal_idx[i]] = 1.0
    return goal_idx, goals, status
