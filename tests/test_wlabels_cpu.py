"""CPU tests of the vertex-weighted shortest-path labels: the oracle against scipy's Dijkstra and against the unit-cost
label oracle, its roll-outs (absorbed and zero costs included), and argument checks at the C ABI (no GPU needed)."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import labels_golden

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

_MOVES = ((-1, 0), (0, 1), (0, -1), (1, 0), (-1, 1), (-1, -1), (1, 1), (1, -1))


@pytest.fixture(scope="module")
def built_lib():
    subprocess.check_call(["make", "-C", os.path.join(ROOT, "neural-astar_b200"), "-s", "all"])
    from neural_astar import _native

    return _native


def _oracle(*args, **kw):
    from oracle import wlabels

    return wlabels.weighted_labels(*args, **kw)


def _random_costs(B, H, W, seed, zero_frac=0.0, block_frac=0.2):
    rs = np.random.RandomState(seed)
    cost = rs.uniform(0.05, 10.0, size=(B, H, W)).astype(np.float32)
    if zero_frac:
        cost[rs.rand(B, H, W) < zero_frac] = 0.0
    passable = (rs.rand(B, H, W) >= block_frac).astype(np.float32)
    goal = rs.randint(0, H * W, size=B).astype(np.int32)
    passable.reshape(B, -1)[np.arange(B), goal] = 1.0
    return cost, passable, goal


def _scipy_dists(cost, passable, goal):
    """float64 Dijkstra of scipy on the reversed move graph: an edge t -> v of weight c[t] for every move v -> t."""
    from scipy.sparse import csr_matrix
    from scipy.sparse.csgraph import dijkstra

    H, W = cost.shape
    rows, cols, w = [], [], []
    ys, xs = np.mgrid[0:H, 0:W]
    src_ok = (passable != 0).ravel()
    src_ok[goal] = False
    enter_ok = (passable != 0).ravel()
    enter_ok[goal] = True
    for dy, dx in _MOVES:
        ty, tx = ys + dy, xs + dx
        inside = (ty >= 0) & (ty < H) & (tx >= 0) & (tx < W)
        v = (ys * W + xs)[inside]
        t = (ty * W + tx)[inside]
        keep = src_ok[v] & enter_ok[t]
        rows.append(t[keep])
        cols.append(v[keep])
        w.append(cost.ravel()[t[keep]].astype(np.float64))
    g = csr_matrix((np.concatenate(w), (np.concatenate(rows), np.concatenate(cols))), shape=(H * W, H * W))
    return dijkstra(g, directed=True, indices=goal)


@pytest.mark.parametrize("H,W", [(5, 40), (12, 12), (33, 31), (64, 64), (100, 72), (128, 128)])
def test_oracle_matches_scipy_dijkstra(H, W):
    """Positive costs (csgraph drops explicit zero weights): the fp32 fold is within H*W * 2^-24 (relative) of the
    float64 optimum, and both agree on which cells reach the goal."""
    B = 4
    cost, passable, goal = _random_costs(B, H, W, seed=H * 1000 + W)
    o = _oracle(cost, goal, passable)
    assert (o["status"] == 0).all()
    for b in range(B):
        ref = _scipy_dists(cost[b], passable[b], int(goal[b]))
        d = -o["dists"][b, 0].ravel().astype(np.float64)
        assert np.array_equal(np.isinf(d), np.isinf(ref))
        fin = np.isfinite(ref)
        assert np.all(np.abs(d[fin] - ref[fin]) <= H * W * 2.0 ** -24 * ref[fin])


def _D(o, b):
    """the cost-to-go plane of map b (dists = 0 - D, so 0 - dists gives D back bit for bit, +0 included)"""
    return np.float32(0.0) - o["dists"][b, 0].ravel()


def _fold(cost, cells):
    """fp32 left fold from the goal over a path's cells, the first (start) excluded"""
    x = np.float32(0.0)
    for c in reversed(cells[1:]):
        x = np.float32(x + cost[c])
    return x


def _check_rollouts(cost, goal, o, b, starts=None):
    """Every roll-out of `action` from a reachable cell reaches the goal after exactly hop moves, lowers hop by one
    per move, and its fold equals D (= -dists) bit for bit."""
    H, W = cost.shape[-2:]
    c = cost[b].ravel()
    D = _D(o, b)
    hop = o["hops"][b, 0].ravel()
    act = o["action"][b, 0].ravel()
    cells = np.flatnonzero(np.isfinite(D)) if starts is None else starts
    for s in cells:
        path = [int(s)]
        v = int(s)
        while v != goal[b]:
            assert len(path) <= hop[s], "a roll-out takes more than hop moves"
            dy, dx = _MOVES[act[v]]
            y, x = divmod(v, W)
            assert 0 <= y + dy < H and 0 <= x + dx < W
            t = (y + dy) * W + x + dx
            assert hop[t] == hop[v] - 1
            v = t
            path.append(v)
        assert len(path) == hop[s] + 1
        assert _fold(c, path).tobytes() == np.float32(D[s]).tobytes(), "the fold along the roll-out is not D"


@pytest.mark.parametrize("H,W", [(12, 12), (5, 40), (33, 31)])
def test_oracle_rollouts_with_zero_costs(H, W):
    B = 6
    cost, passable, goal = _random_costs(B, H, W, seed=7 + H, zero_frac=0.3)
    o = _oracle(cost, goal, passable)
    for b in range(B):
        _check_rollouts(cost, goal, o, b)


def test_oracle_rollouts_on_absorbed_costs():
    """Costs of 1e-9 beside distances near 1e4 are absorbed (fl(D + c) == D), so every move between such cells is
    optimal and the optimal moves form cycles; the hop rule still sends every roll-out to the goal."""
    H, W = 12, 12
    cost = np.full((2, H, W), 1e-9, np.float32)
    cost[0, 0, 0] = 1e4                       # the goal of map 0: every other cell has D == 1e4
    rs = np.random.RandomState(3)
    cost[1] = np.where(rs.rand(H, W) < 0.5, 1e-9, 1e4).astype(np.float32)
    goal = np.array([0, H * W - 1], np.int32)
    o = _oracle(cost, goal)
    D0 = _D(o, 0)
    assert (D0[1:] == np.float32(1e4)).all()
    ys, xs = np.divmod(np.arange(H * W), W)
    assert np.array_equal(o["hops"][0, 0].ravel(), np.maximum(ys, xs))    # Chebyshev distance to the corner goal
    for b in range(2):
        _check_rollouts(cost, goal, o, b)
    # the same with starts: masks with hop + 1 cells, path cost = fl(c[start] + D[start])
    starts = np.array([H * W - 1, 0], np.int32)
    o = _oracle(cost, goal, start_idx=starts)
    for b in range(2):
        s = starts[b]
        assert o["path_maps"][b].sum() == o["hops"][b, 0].ravel()[s] + 1
        assert o["path_costs"][b] == np.float32(cost[b].ravel()[s] + _D(o, b)[s])


def test_oracle_reduces_to_unit_labels_on_fixtures():
    """cost = (map != 0), passable = map, a passable goal: -D equals labels_oracle's dists on every reachable cell,
    hop equals D, and the policy equals the unit labels' on every reachable non-goal cell."""
    from oracle import labels as label_oracle

    n = 0
    for name in labels_golden.NAMES:
        maps, goal_idx, _, _ = labels_golden.load(name)
        B = maps.shape[0]
        keep = maps.reshape(B, -1)[np.arange(B), goal_idx] != 0
        maps, goal_idx = maps[keep], goal_idx[keep]
        B, H, W = maps.shape
        ud, um, ua = label_oracle.opt_labels(maps, goal_idx)
        o = _oracle((maps != 0).astype(np.float32), goal_idx, maps)
        assert (o["status"] == 0).all()
        reach = np.isfinite(o["dists"])
        assert np.array_equal(reach, ud > -H * W)
        assert np.array_equal(o["dists"][reach], ud[reach])
        assert np.array_equal(o["hops"][reach], -ud[reach].astype(np.int32))
        nongoal = reach.copy()
        nongoal.reshape(B, -1)[np.arange(B), goal_idx] = False
        assert np.array_equal(o["act_mask"][nongoal], um[nongoal])
        assert np.array_equal(o["action"][nongoal], ua[nongoal])
        n += B
    assert n > 100


def test_oracle_status_and_edge_cases():
    H, W = 6, 7
    cost = np.ones((5, H, W), np.float32)
    passable = np.ones_like(cost)
    goal = np.array([10, 10, 99, 10, 10], np.int32)         # map 2: no goal
    starts = np.array([0, 0, 0, 0, 10], np.int32)           # map 4: start == goal
    cost[0, 3, 3] = -1.0                                    # a negative cost on a passable cell
    cost[1, 3, 3] = np.nan
    passable[1, 3, 3] = 0.0                                 # ... on an obstacle it is never charged
    passable[3, :, 2] = 0.0                                 # map 3: a wall between the start and the goal
    o = _oracle(cost, goal, passable, starts)
    assert o["status"].tolist() == [1 | 4, 0, 2 | 4, 4, 0]
    assert np.isneginf(o["dists"][0]).all() and (o["hops"][0] == -1).all() and (o["action"][0] == -1).all()
    assert o["path_costs"][4] == cost[4, 1, 3] and o["path_maps"][4].sum() == 1
    assert np.isinf(o["path_costs"][3]) and o["path_maps"][3].sum() == 0
    assert o["path_maps"][1].sum() == o["hops"][1, 0, 0, 0] + 1 == 4


def test_weighted_labels_rejects_bad_arguments_without_a_gpu(built_lib):
    L = built_lib.lib()
    f = L.nastar_b200_weighted_labels
    c, p, g, s = 0x10000, 0x20000, 0x30000, 0x40000
    d, h, m, a, pm, pc, st = 0x50000, 0x60000, 0x70000, 0x80000, 0x90000, 0xA0000, 0xB0000
    EINVAL, EUNSUPPORTED = 1, 2
    before = L.nastar_b200_launch_count()

    def call(**kw):
        args = dict(c=c, cs=144, p=p, ps=144, g=g, s=s, B=1, H=12, W=12, d=d, h=h, m=m, a=a, pm=pm, pc=pc, st=st)
        args.update(kw)
        return f(*args.values(), None)

    assert call(c=None) == EINVAL                   # null cost
    assert call(g=None) == EINVAL                   # null goals
    for k in ("d", "h", "m", "a", "st"):
        assert call(**{k: None}) == EINVAL          # null outputs
    assert call(B=0) == EINVAL and call(H=0) == EINVAL and call(W=-1) == EINVAL
    assert call(cs=143) == EINVAL                   # maps overlap
    assert call(ps=100) == EINVAL
    assert call(pm=None) == EINVAL and call(pc=None) == EINVAL      # a start without path outputs
    assert call(s=None) == EINVAL                   # path outputs without starts
    assert call(H=129, W=8, cs=129 * 8, ps=129 * 8) == EUNSUPPORTED
    assert call(H=8, W=200, cs=1600, ps=1600) == EUNSUPPORTED
    assert L.nastar_b200_launch_count() == before   # nothing above was launched
    # the binding refuses CPU tensors and maps above the limit before reaching the library
    with pytest.raises(RuntimeError):
        built_lib.weighted_labels(torch.ones(1, 12, 12), torch.zeros(1, dtype=torch.int32))
    from neural_astar.utils.data import compute_weighted_opt_labels

    with pytest.raises(RuntimeError):
        compute_weighted_opt_labels(torch.ones(1, 1, 12, 12), torch.zeros(1, 1, 12, 12))
