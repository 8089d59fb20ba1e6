"""CPU oracle of the black-box backward (BB-A*, Vlastelica et al., ICLR 2020): the existing search oracles run on the
costs w and on the perturbed costs w' = fl(w + fl(lambda * g)), the latter formed in float32 NumPy with two rounded
operations, and dL/dw = (y(w') - y(w)) / lambda.

Both mechanisms' searches go through oracle/oracle.py.  Per-map early exit
(the spec oracles) or, for a batch-coupled search, the reference's batch-synchronous loop (the literal oracles) with the
step bound T as its cap; each search gets its own T_batch."""
from __future__ import annotations

from typing import NamedTuple

import numpy as np

from oracle import oracle

F32 = np.float32


class BlackboxOutput(NamedTuple):
    grad: np.ndarray        # [B,1,H,W] float32: dL/dw, channel 0
    histories: np.ndarray   # [B,1,H,W] float32: y(w)
    perturbed: np.ndarray   # [B,1,H,W] float32: y(w')
    costs: np.ndarray       # [B,1,H,W] float32: w'


def perturbed_costs(cost, grad_hist, lam: float) -> np.ndarray:
    """w' = fl(w + fl(lambda * g)) of channel 0, [B,1,H,W] float32 (no FMA, no clamp)."""
    w = np.asarray(cost, F32)[:, :1]
    g = np.asarray(grad_hist, F32).reshape(w.shape)
    return np.add(w, np.multiply(F32(lam), g, dtype=F32), dtype=F32)


def search(cost, start, goal, obst, g_ratio: float, T: int, mechanism: str = "moore",
           coupled: bool = False) -> np.ndarray:
    """The histories y(cost) of the search that the planner runs: per-map early exit, or batch-coupled."""
    out = oracle.forward(cost, start, goal, obst, g_ratio, T=T, mode="literal" if coupled else "spec",
                         mechanism=mechanism)
    return np.asarray(out.histories, F32)


def blackbox_backward(cost, start, goal, obst, grad_hist, lam: float, g_ratio: float, T: int,
                      mechanism: str = "moore", coupled: bool = False) -> BlackboxOutput:
    """dL/dw of BB-A* for the search of (cost, start, goal, obst) and the incoming gradient grad_hist [B,1,H,W]."""
    y = search(cost, start, goal, obst, g_ratio, T, mechanism, coupled)
    w2 = perturbed_costs(cost, grad_hist, lam)
    y2 = search(w2, start, goal, obst, g_ratio, T, mechanism, coupled)
    return BlackboxOutput(np.subtract(y2, y, dtype=F32) / F32(lam), y, y2, w2)
