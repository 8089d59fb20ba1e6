"""NumPy restatement of the GPU batch sampler (csrc/nastar_sampler.cuh, utils.data.DeviceMazeDataset): thresholds,
bands, the preparation status, the draw mapping and the trajectory walk.  Test infrastructure only."""
from __future__ import annotations

import math

import numpy as np

MOVES = ((-1, 0), (0, 1), (0, -1), (1, 0), (-1, 1), (-1, -1), (1, 1), (1, -1))   # MazeDataset's _ACTION_TO_MOVE
PCTS = (0.55, 0.70, 0.85)


def fractions(pcts=PCTS) -> np.ndarray:
    return np.true_divide(100.0 * (1 - np.array([*pcts, 1.0])), np.float32(100))


def thresholds(od: np.ndarray, q: np.ndarray) -> np.ndarray:
    """np.percentile's linear method over od[od > od.min()], written out the way the kernel computes it."""
    od = od.ravel().astype(np.float32)
    vals = np.sort(od[od > od.min()])
    n = len(vals)
    vi_max = float(n - 1)
    out = []
    for qj in q:
        vi = vi_max * float(qj)
        if vi >= vi_max:
            prev, lo, hi = -1.0, vals[n - 1], vals[n - 1]
        else:
            prev = float(math.floor(vi))
            lo, hi = vals[int(prev)], vals[int(prev) + 1]
        g = vi - prev
        d = float(np.float32(hi) - np.float32(lo))
        t = float(lo) + d * g
        if g >= 0.5:
            t = float(hi) - d * (1.0 - g)
        out.append(t)
    return np.array(out, np.float64)


def band_masks(od: np.ndarray, th: np.ndarray) -> np.ndarray:
    """bool [3, N]: band r = cells above od.min() with th[r+1] <= od <= th[r]."""
    od = od.ravel().astype(np.float32)
    cand = od > od.min()
    return np.stack([cand & (th[r + 1] <= od) & (od <= th[r]) for r in range(3)])


def first_max_actions(policy: np.ndarray) -> np.ndarray:
    return policy.reshape(8, -1).argmax(0)


def status(od: np.ndarray, act: np.ndarray, goal: int, H: int, W: int, q: np.ndarray) -> int:
    """The kernel's per-map status bits (include/nastar_b200.h, nastar_b200_sampler_prepare)."""
    od = od.ravel().astype(np.float32)
    N = H * W
    if not (np.all(od >= -N) and np.all(od <= 0) and np.all(od == np.trunc(od))):
        return 1
    if not (od > od.min()).any():
        return 2
    st = 0
    if not band_masks(od, thresholds(od, q)).any(1).all():
        st |= 4
    c = np.flatnonzero((od > -N) & (np.arange(N) != goal))
    y, x = np.divmod(c, W)
    dy = np.array([m[0] for m in MOVES])[act[c]]
    dx = np.array([m[1] for m in MOVES])[act[c]]
    ty, tx = y + dy, x + dx
    on = (ty >= 0) & (ty < H) & (tx >= 0) & (tx < W)
    if not on.all() or not (od[(ty * W + tx)[on]] == od[c[on]] + 1).all():
        st |= 8
    if (od == 0).sum() != 1 or od[goal] != 0:
        st |= 16
    return st


def start_from_draws(masks: np.ndarray, d0: int, d1: int) -> int:
    r = (int(d0) * 3) >> 32
    cells = np.flatnonzero(masks[r])
    return int(cells[(int(d1) * len(cells)) >> 32])


def draws_for(r: int, k: int, count: int):
    """The smallest u32 draws (d0, d1) that select candidate k of band r (of `count` candidates)."""
    return -(-(r << 32) // 3), -(-(k << 32) // count)


def walk(start: int, goal: int, act: np.ndarray, W: int) -> np.ndarray:
    traj = np.zeros(act.shape[0], np.float32)
    off = np.array([m[0] * W + m[1] for m in MOVES])
    loc = start
    while loc != goal:
        traj[loc] = 1.0
        loc = int(loc + off[act[loc]])
    return traj


def sample(od, policy, goal_map, draws, q=None):
    """(starts [S, N], trajs [S, N]) of one map for u32 draws [S, 2]."""
    q = fractions() if q is None else q
    H, W = od.shape[-2:]
    masks = band_masks(od, thresholds(od, q))
    act = first_max_actions(policy)
    goal = int(np.argmax(goal_map.ravel()))
    S = len(draws)
    starts = np.zeros((S, H * W), np.float32)
    trajs = np.zeros((S, H * W), np.float32)
    for s, (d0, d1) in enumerate(np.asarray(draws, np.uint64).tolist()):
        st = start_from_draws(masks, d0, d1)
        starts[s, st] = 1.0
        trajs[s] = walk(st, goal, act, W)
    return starts, trajs
