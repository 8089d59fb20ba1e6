"""NumPy restatement of the vertex-weighted shortest-path labels (DESIGN.md §11) for the NEWS mechanism, which checks
nastar_b200_weighted_labels_mech with NASTAR_MECH_NEWS (csrc/nastar_wlabels.cuh, kNews).

Written from the semantics, with the move set as a parameter: actions 0..3 = N, E, W, S for "news", the 8 actions
N, E, W, S, NE, NW, SE, SW for "moore".  With the Moore moves it equals oracle/wlabels_oracle.c bit for bit
(tests/test_wlabels_news_cpu.py), which pins every rule below except the move set.  Per map:
  moves    from a passable cell other than the goal into an in-grid cell that is passable or is the goal; a move
           charges the cost of the cell it enters.
  D        D[goal] = +0, D[v] = min over moves v->t of fl(D[t] + c[t]) (one float32 add, rounded once), +inf where
           the goal is unreachable.  Computed by Jacobi rounds over the whole batch until nothing changes: for c >= 0
           the fold is monotone, so the fixpoint is the least fold over all paths, whatever the evaluation order.
  hop      breadth-first wavefronts from the goal over optimal moves (fl(D[t] + c[t]) == D[v]); -1 unreachable.
  policy   act_mask: the optimal moves into cells with hop one lower (0 at the goal and unreachable cells);
           action: its lowest bit, -1 where it is 0.
  path     the roll-out of `action` from the start (start and goal included); path_cost = fl(c[start] + D[start]).
  status   1 the goal or a passable cell has a negative, NaN or infinite cost (every plane filled as unreachable);
           2 no goal (index outside [0, H*W)); 4 a start was given and cannot reach the goal."""
import numpy as np

MOVES = {"moore": ((-1, 0), (0, 1), (0, -1), (1, 0), (-1, 1), (-1, -1), (1, 1), (1, -1)),
         "news": ((-1, 0), (0, 1), (0, -1), (1, 0))}


def _at(x, dy, dx, fill):
    """y[b, r, q] = x[b, r + dy, q + dx] where that is on the grid, `fill` elsewhere"""
    H, W = x.shape[1:]
    y = np.full_like(x, fill)
    y[:, max(0, -dy):H - max(0, dy), max(0, -dx):W - max(0, dx)] = \
        x[:, max(0, dy):H + min(0, dy), max(0, dx):W + min(0, dx)]
    return y


def _maps(x):
    a = np.asarray(x, dtype=np.float32)
    return np.ascontiguousarray(a[:, 0] if a.ndim == 4 else a)


def weighted_labels(cost, goal_idx, passable=None, start_idx=None, mechanism="news"):
    """Labels of cost maps [B,H,W] or [B,1,H,W] with flat goal (and optional start) indices [B], passable iff != 0
    (None: every cell).  Returns a dict of dists f32, hops i32, act_mask u8, action i8 (each [B,1,H,W]) and status
    i32 [B]; with starts also path_maps f32 [B,1,H,W] and path_costs f32 [B] -- the outputs of
    nastar_b200_weighted_labels_mech."""
    if mechanism not in MOVES:
        raise ValueError(f"mechanism must be one of {sorted(MOVES)} (got {mechanism!r})")
    c = _maps(cost)
    B, H, W = c.shape
    N = H * W
    pas = np.ones((B, H, W), bool) if passable is None else _maps(passable) != 0.0
    if pas.shape != c.shape:
        raise ValueError("passable must have the cost maps' shape")
    g = np.asarray(goal_idx, dtype=np.int64).reshape(B)
    has = (g >= 0) & (g < N)
    is_goal = np.zeros((B, H, W), bool)
    is_goal.reshape(B, N)[np.flatnonzero(has), g[has]] = True
    enter = pas | is_goal
    with np.errstate(invalid="ignore"):
        bad = (enter & ~(np.isfinite(c) & (c >= 0.0))).any((1, 2))
        return _labels(c, pas, g, is_goal, enter, bad, has, start_idx, MOVES[mechanism])


def _labels(c, pas, g, is_goal, enter, bad, has, start_idx, moves):
    B, H, W = c.shape
    N = H * W
    status = np.where(bad, 1, 0).astype(np.int32) | np.where(has, 0, 2).astype(np.int32)
    ok = (status == 0)[:, None, None]
    src = pas & ~is_goal & ok                              # cells whose D is a minimum over their moves
    inf = np.float32(np.inf)
    cm = np.where(enter, c, np.float32(0.0))               # costs that can be charged (finite on valid maps)
    tgt = [(_at(enter, dy, dx, False), _at(cm, dy, dx, np.float32(0.0))) for dy, dx in moves]

    D = np.full((B, H, W), inf, np.float32)
    D[is_goal & ok] = 0.0
    for _ in range(N + 1):
        best = D.copy()
        for (dy, dx), (t_ok, t_c) in zip(moves, tgt):
            via = np.where(t_ok, _at(D, dy, dx, inf) + t_c, inf)
            np.minimum(best, via, out=best)
        new = np.where(src, best, D)
        if np.array_equal(new, D):
            break
        D = new

    reach = np.isfinite(D)
    optimal = [t_ok & src & reach & (_at(D, dy, dx, inf) + t_c == D) for (dy, dx), (t_ok, t_c) in zip(moves, tgt)]
    hop = np.full((B, H, W), -1, np.int32)
    hop[is_goal & ok] = 0
    for k in range(1, N + 2):
        hit = np.zeros((B, H, W), bool)
        for (dy, dx), opt in zip(moves, optimal):
            hit |= opt & (_at(hop, dy, dx, -1) == k - 1)
        hit &= hop == -1
        if not hit.any():
            break
        hop[hit] = k

    mask = np.zeros((B, H, W), np.uint8)
    for a, ((dy, dx), opt) in enumerate(zip(moves, optimal)):
        mask |= ((opt & (hop > 0) & (_at(hop, dy, dx, -1) == hop - 1)).astype(np.uint8) << a)
    low = np.argmax((mask[None] >> np.arange(len(moves), dtype=np.uint8)[:, None, None, None]) & 1, axis=0)
    action = np.where(mask != 0, low, -1).astype(np.int8)
    out = dict(dists=(np.float32(0.0) - D)[:, None], hops=hop[:, None], act_mask=mask[:, None],
               action=action[:, None], status=status)
    if start_idx is None:
        return out

    s_idx = np.asarray(start_idx, dtype=np.int64).reshape(B)
    paths = np.zeros((B, N), np.float32)
    pcost = np.full(B, inf, np.float32)
    Df, cf, af = D.reshape(B, N), c.reshape(B, N), action.reshape(B, N)
    for b in range(B):
        s = int(s_idx[b])
        if status[b] != 0 or not 0 <= s < N or not np.isfinite(Df[b, s]):
            status[b] |= 4
            continue
        v = s
        paths[b, v] = 1.0
        for _ in range(N):
            if v == g[b] or af[b, v] < 0:
                break
            dy, dx = moves[af[b, v]]
            v += dy * W + dx
            paths[b, v] = 1.0
        if v != g[b]:                       # cannot happen: every policy move lowers hop by one
            paths[b] = 0.0
            status[b] |= 4
            continue
        pcost[b] = cf[b, s] + Df[b, s]
    out["path_maps"] = paths.reshape(B, 1, H, W)
    out["path_costs"] = pcost
    return out
