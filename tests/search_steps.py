"""A NumPy step machine of the SPEC search for either mechanism, for tests that read the f values of the open set to
check their own preconditions (exp(-f / sqrt(W)) far from underflow, exp-collisions, near ties).  Expected outputs
come from the C oracle (oracle/astar_oracle.c), never from here."""
import numpy as np

MOVES = {"moore": ((-1, -1), (-1, 0), (-1, 1), (0, -1), (0, 1), (1, -1), (1, 0), (1, 1)),
         "news": ((-1, 0), (0, -1), (0, 1), (1, 0))}


def heuristic(H, W, goal, mechanism):
    """get_heuristic (Chebyshev) or get_news_heuristic (Manhattan) + 0.001 * Euclid for one goal, flat [H*W] float32."""
    ys, xs = np.divmod(np.arange(H * W), W)
    gy, gx = divmod(int(goal), W)
    dy, dx = np.abs(ys - gy).astype(np.float32), np.abs(xs - gx).astype(np.float32)
    dist = (dy + dx) - np.minimum(dy, dx) if mechanism == "moore" else dy + dx
    return dist + np.float32(0.001) * np.sqrt(dy * dy + dx * dx)


class SpecMachine:
    """One map's SPEC state machine in float32 NumPy, stepped by the caller."""

    def __init__(self, cost, obst, si, gi, mechanism):
        H, W = cost.shape
        self.cost, self.obst, self.H, self.W, self.gi, self.moves = cost.ravel(), obst.ravel(), H, W, gi, MOVES[mechanism]
        self.h = heuristic(H, W, gi, mechanism) + self.cost
        self.g = np.zeros(H * W, np.float32)
        self.open = np.zeros(H * W, bool)
        self.closed = np.zeros(H * W, bool)
        self.open[si] = True

    def f(self, gr, omg):
        return gr * self.g + omg * self.h

    def select(self, gr, omg):
        """arg-min of (f, index) over the open set, -1 when it is empty"""
        if not self.open.any():
            return -1
        return int(np.argmin(np.where(self.open, self.f(gr, omg), np.float32(np.inf))))

    def close_and_expand(self, ind):
        self.closed[ind] = True
        if ind != self.gi:
            self.open[ind] = False         # the goal, once selected, stays open
        g2 = self.g[ind] + self.cost[ind]
        r, c = divmod(int(ind), self.W)
        for dy, dx in self.moves:
            y, x = r + dy, c + dx
            n = y * self.W + x
            if not (0 <= y < self.H and 0 <= x < self.W) or self.obst[n] == 0:
                continue
            if (not self.open[n] and not self.closed[n]) or (self.open[n] and self.g[n] > g2):
                self.g[n], self.open[n] = g2, True


def machines(cost, start, goal, obst, mechanism):
    """A SpecMachine per map of [B,C,H,W] planes (channel 0 of the cost is searched)."""
    return [SpecMachine(cost[b, 0], obst[b, 0], int(start[b].argmax()), int(goal[b].argmax()), mechanism)
            for b in range(cost.shape[0])]
