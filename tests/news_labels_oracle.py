"""NumPy restatement of the planning-datasets generator's NEWS labels (NorthEastWestSouth, mechanism.py:52-131, with
dijkstra_dist, dijkstra.py:120-157, and the max set of extract_policy, data.py:40-58), which checks
nastar_b200_opt_labels_mech with NASTAR_MECH_NEWS (csrc/nastar_labels.cuh, DESIGN.md §9).

Per map: a cell is passable iff its value != 0.0; actions 0..3 = N, E, W, S, and a move off the grid or onto a
non-passable cell stays put.  Every step costs 1, so dijkstra_dist's distances are breadth-first distances from the
goal: a cell first reached in wavefront k (a passable 4-neighbour of a cell of wavefront k-1) gets -k, the goal 0
(it is the source even when it is not passable), every other cell -(H*W), the generator's never-relaxed initial value.
The mask holds the actions whose target has the maximal value, the action its lowest member."""
import numpy as np

MOVES = ((-1, 0), (0, 1), (0, -1), (1, 0))      # N, E, W, S as (dy, dx), mechanism.py:58


def opt_labels(maps, goal_idx):
    """(dists float32 [B,1,H,W], act_mask uint8 [B,1,H,W], action int8 [B,1,H,W]) for maps [B,H,W] or [B,1,H,W] and
    flat goal indices [B] (an index outside [0, H*W) means no goal: every cell -(H*W))."""
    m = np.asarray(maps, dtype=np.float32)
    if m.ndim == 4:
        m = m[:, 0]
    B, H, W = m.shape
    N = H * W
    g = np.asarray(goal_idx, dtype=np.int64).reshape(B)
    passable = m != 0.0
    dist = np.full((B, H, W), N, np.int64)
    front = np.zeros((B, H, W), bool)
    has = (g >= 0) & (g < N)
    front.reshape(B, N)[np.flatnonzero(has), g[has]] = True
    dist[front] = 0
    seen = front.copy()
    k = 0
    while front.any():
        k += 1
        grow = np.zeros_like(front)
        grow[:, 1:, :] |= front[:, :-1, :]
        grow[:, :-1, :] |= front[:, 1:, :]
        grow[:, :, 1:] |= front[:, :, :-1]
        grow[:, :, :-1] |= front[:, :, 1:]
        front = grow & passable & ~seen
        seen |= front
        dist[front] = k
    value = -dist
    y, x = np.mgrid[0:H, 0:W]
    vals = []
    for dy, dx in MOVES:
        ty, tx = y + dy, x + dx
        on = (ty >= 0) & (ty < H) & (tx >= 0) & (tx < W)
        ty, tx = np.where(on, ty, y), np.where(on, tx, x)
        ok = on & passable[:, ty, tx]                     # [B,H,W]: the move leaves the cell
        vals.append(np.where(ok, value[:, ty, tx], value))
    vals = np.stack(vals)                                 # [4,B,H,W]
    best = vals.max(0)
    mask = np.zeros((B, H, W), np.uint8)
    for a in range(len(MOVES)):
        mask |= (vals[a] == best).astype(np.uint8) << a
    action = np.argmax(vals == best, axis=0).astype(np.int8)      # the lowest maximal action
    return value.astype(np.float32)[:, None], mask[:, None], action[:, None]
