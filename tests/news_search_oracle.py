"""NumPy restatement of the differentiable A* search with the planning-datasets generator's NorthEastWestSouth
mechanism, which checks the engines' NASTAR_FWD_NEWS / NASTAR_MECH_NEWS instantiations (DESIGN.md §14).

The search is DifferentiableAstar's loop (differentiable_astar.py:187-255) with the two pieces a user of the reference
gives it for NEWS datasets (mechanism.py:113-131): the neighbour filter N, E, W, S (a selected cell never opens or
relaxes a diagonal neighbour) and h = manhattan + 0.001 * euclid.  Every fp32 operation is one IEEE rounding (NumPy
float32 arithmetic; the LITERAL form takes exp from ATen, the op the reference evaluates).  Three forms, as for the
Moore oracle in oracle/astar_oracle.c:
  literal   dense planes, exp / softmax / first argmax selection, batch-coupled stop, exactly as the loop is written;
  spec      the per-map state machine the engines implement: arg-min of (f, flat index) over the open set, per-map
            early exit (or exactly T steps with no_early_exit);
  backward  the closed-form gradient of the straight-through softmax (SURVEY.md App. B) in fp64, replaying spec for
            T_batch steps.
Planes are [B,1,H,W] float32; outputs have the layout of oracle.oracle.forward / backward."""
from typing import NamedTuple, Optional

import math

import numpy as np
import torch

F32 = np.float32
MOVES = ((-1, 0), (0, -1), (0, 1), (1, 0))      # the non-zero entries of the NEWS filter, in raster order


class Output(NamedTuple):
    histories: np.ndarray   # [B,1,H,W] float32
    paths: np.ndarray       # [B,1,H,W] int64
    t_solve: np.ndarray     # [B] int32: solve step, -1 step cap, -2 open set exhausted
    n_steps: np.ndarray     # [B] int32 (spec) / T_batch broadcast (literal)
    T_batch: int
    trace: Optional[np.ndarray]   # [B,T] int32, -1 beyond the executed steps


def _planes(x):
    a = np.asarray(x, dtype=F32)
    assert a.ndim == 4
    return np.ascontiguousarray(a[:, 0].reshape(a.shape[0], -1)), a.shape[-2], a.shape[-1]


def _scalars(g_ratio, W):
    return F32(g_ratio), F32(1 - g_ratio), F32(math.sqrt(W))


def heuristic(H, W, goal):
    """NorthEastWestSouth.get_heuristic for one goal, flat [H*W] float32, for any H x W."""
    ys, xs = np.divmod(np.arange(H * W), W)
    gy, gx = divmod(int(goal), W)
    dy = np.abs(ys - gy).astype(F32)
    dx = np.abs(xs - gx).astype(F32)
    return (dy + dx) + F32(0.001) * np.sqrt(dy * dy + dx * dx)


def _neighbours(ind, H, W):
    r, c = divmod(int(ind), W)
    for dr, dc in MOVES:
        y, x = r + dr, c + dc
        if 0 <= y < H and 0 <= x < W:
            yield y * W + x


class _Spec:
    """One map's state machine (arg-min selection)."""

    def __init__(self, cost, obst, H, W, si, gi):
        self.cost, self.obst, self.H, self.W, self.gi = cost, obst, H, W, gi
        self.h = heuristic(H, W, gi) + cost
        self.g = np.zeros(H * W, F32)
        self.open = np.zeros(H * W, bool)
        self.closed = np.zeros(H * W, bool)
        self.parent = np.full(H * W, gi, np.int64)
        self.open[si] = True

    def f(self, gr, omg):
        return gr * self.g + omg * self.h

    def select(self, gr, omg):
        if not self.open.any():
            return -1
        return int(np.argmin(np.where(self.open, self.f(gr, omg), F32(np.inf))))   # first minimum: lowest index

    def close_and_expand(self, ind):
        self.closed[ind] = True
        if ind != self.gi:
            self.open[ind] = False         # the goal, once selected, stays open
        g2 = self.g[ind] + self.cost[ind]
        for n in _neighbours(ind, self.H, self.W):
            if self.obst[n] == 0:
                continue
            if (not self.open[n] and not self.closed[n]) or (self.open[n] and self.g[n] > g2):
                self.g[n] = g2
                self.open[n] = True
                self.parent[n] = ind


def forward(cost, start, goal, obst, g_ratio=0.5, Tmax=1.0, training=False, mode="spec", want_trace=False, T=None,
            no_early_exit=False) -> Output:
    c, H, W = _planes(cost)
    s, g, o = _planes(start)[0], _planes(goal)[0], _planes(obst)[0]
    B, N = c.shape
    T = int(T) if T is not None else int((Tmax if training else 1.0) * W * W)
    si, gi = s.argmax(1), g.argmax(1)
    if mode == "literal":
        return _literal(c, g, o, si, gi, B, H, W, g_ratio, T, want_trace)
    if mode != "spec":
        raise ValueError(mode)
    gr, omg, _ = _scalars(g_ratio, W)
    hist = np.zeros((B, N), F32)
    paths = np.zeros((B, N), np.int64)
    ts = np.full(B, -1, np.int32)
    ns = np.zeros(B, np.int32)
    trace = np.full((B, T), -1, np.int32) if want_trace else None
    for b in range(B):
        m = _Spec(c[b], o[b], H, W, si[b], gi[b])
        for t in range(T):
            ind = m.select(gr, omg)
            if ind < 0:
                ts[b] = -2
                break
            if want_trace:
                trace[b, t] = ind
            ns[b] = t + 1
            m.close_and_expand(ind)
            if ind == gi[b] and ts[b] < 0:
                ts[b] = t
            if ind == gi[b] and not no_early_exit:
                break
        hist[b] = m.closed
        # backtrack (SURVEY App. A.3): solved -> walk to the start; otherwise at most T-1 hops
        paths[b, gi[b]] = 1
        loc = m.parent[gi[b]]
        for _ in range(N if ts[b] >= 0 else T - 1):
            paths[b, loc] = 1
            if ts[b] >= 0 and loc == si[b]:
                break
            loc = m.parent[loc]
    return Output(hist.reshape(B, 1, H, W), paths.reshape(B, 1, H, W), ts, ns, int(ns.max()), trace)


def _literal(c, goalmap, o, si, gi, B, H, W, g_ratio, T, want_trace) -> Output:
    """The batch loop as written: all maps step together until one step in which every map selects its goal."""
    N = H * W
    gr, omg, sqw = _scalars(g_ratio, W)
    rows = np.arange(B)
    h = np.stack([heuristic(H, W, gi[b]) for b in range(B)]) + c
    g = np.zeros((B, N), F32)
    open_ = np.zeros((B, N), F32)
    open_[rows, si] = 1
    hist = np.zeros((B, N), F32)
    parents = np.repeat(gi[:, None].astype(F32), N, 1)
    ts = np.full(B, -1, np.int32)
    trace = np.full((B, T), -1, np.int32) if want_trace else None
    one, zero = F32(1), F32(0)
    tb = 0
    for t in range(T):
        f = gr * g + omg * h
        e = torch.exp(torch.from_numpy((F32(-1) * f) / sqw)).numpy()
        v = e * open_
        y = v / v.sum(1, keepdims=True)
        ind = y.argmax(1)                                  # first maximum
        if want_trace:
            trace[:, t] = ind
        unsolved = (goalmap[rows, ind] < F32(1e-8)).astype(F32)
        ts[(unsolved == 0) & (ts < 0)] = t
        hist[rows, ind] = np.clip(hist[rows, ind] + one, zero, one)
        open_[rows, ind] = np.clip(open_[rows, ind] - unsolved, zero, one)
        r, cc = np.divmod(ind, W)
        g2 = g[rows, ind] + c[rows, ind]
        indf = ind.astype(F32)
        for dr, dc in MOVES:
            yy, xx = r + dr, cc + dc
            ok = (yy >= 0) & (yy < H) & (xx >= 0) & (xx < W)
            rr = rows[ok]
            n = (yy * W + xx)[ok]
            gt = (g[rr, n] > g2[ok]).astype(F32)
            idx = ((one - open_[rr, n]) * (one - hist[rr, n]) + open_[rr, n] * gt) * o[rr, n]
            g[rr, n] = g2[ok] * idx + g[rr, n] * (one - idx)
            open_[rr, n] = np.clip(open_[rr, n] + idx, zero, one)
            parents[rr, n] = indf[ok] * idx + parents[rr, n] * (one - idx)
        tb = t + 1
        if not unsolved.any():
            break
    paths = np.zeros((B, N), np.int64)
    for b in range(B):
        paths[b, gi[b]] = 1
        loc = int(parents[b, gi[b]])
        for _ in range(tb - 1):
            paths[b, loc] = 1
            loc = int(parents[b, loc])
    return Output(hist.reshape(B, 1, H, W), paths.reshape(B, 1, H, W), ts, np.full(B, tb, np.int32), tb, trace)


def backward(cost, start, goal, obst, grad_hist, T_batch: int, g_ratio=0.5, dtype=F32) -> np.ndarray:
    """dL/dcost [B,1,H,W] (float32, or `dtype`: float64 keeps the fp64 sums unrounded) for dL/dhistories = grad_hist,
    replaying spec for T_batch steps per map:
    sum_t -(1-g_ratio)/sqrt(W) * y_t * (G - <G, y_t>), y_t the softmax of -f/sqrt(W) over the open set, with G zeroed at
    the goal when the goal is selected twice (clamp(hist + sel) blocks it there)."""
    c, H, W = _planes(cost)
    s, g, o, G = _planes(start)[0], _planes(goal)[0], _planes(obst)[0], _planes(grad_hist)[0].astype(np.float64)
    B, N = c.shape
    gr, omg, sqw = _scalars(g_ratio, W)
    out = np.zeros((B, N), dtype)
    for b in range(B):
        gi = int(g[b].argmax())
        m = _Spec(c[b], o[b], H, W, int(s[b].argmax()), gi)
        acc_y, acc_yd, acc_yg = np.zeros(N), np.zeros(N), np.zeros(N)
        not_goal = np.arange(N) != gi
        blocked = False
        for _ in range(int(T_batch)):
            ind = m.select(gr, omg)
            if ind < 0:
                break
            y = np.where(m.open, np.exp(-m.f(gr, omg).astype(np.float64) / float(sqw)), 0.0)
            y /= y.sum()
            acc_y += y
            acc_yd += y * float(np.dot(G[b] * not_goal, y))
            acc_yg += y * y[gi]
            blocked |= bool(m.closed[ind])
            m.close_and_expand(ind)
        Gg = 0.0 if blocked else G[b, gi]
        Gi = np.where(not_goal, G[b], Gg)
        out[b] = (-float(omg) / float(sqw)) * (acc_y * Gi - acc_yd - acc_yg * Gg)
    return out.reshape(B, 1, H, W)
