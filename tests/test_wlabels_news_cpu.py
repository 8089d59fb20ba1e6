"""CPU tests of the NEWS (4-connected) vertex-weighted shortest-path labels: the C oracle's NEWS mode
(oracle/wlabels_oracle.c) against scipy's Dijkstra on the 4-connected move graph and against the NEWS unit-cost labels;
its roll-outs (absorbed and zero costs included), status and edge cases; argument checks at the C ABI (no GPU
needed)."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import labels_golden
from oracle import labels as label_oracle
from oracle import wlabels

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

NEWS_MOVES = ((-1, 0), (0, 1), (0, -1), (1, 0))     # actions 0..3 = N, E, W, S


@pytest.fixture(scope="module")
def built_lib():
    subprocess.check_call(["make", "-C", os.path.join(ROOT, "neural-astar_b200"), "-s", "all"])
    from neural_astar import _native

    return _native


def _oracle(*args, **kw):
    return wlabels.weighted_labels(*args, mechanism="news", **kw)


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
    """float64 Dijkstra of scipy on the reversed 4-connected move graph: an edge t -> v of weight c[t] for every move
    v -> t between 4-neighbours"""
    from scipy.sparse import csr_matrix
    from scipy.sparse.csgraph import dijkstra

    H, W = cost.shape
    rows, cols, w = [], [], []
    ys, xs = np.mgrid[0:H, 0:W]
    src_ok = (passable != 0).ravel()
    src_ok[goal] = False
    enter_ok = (passable != 0).ravel()
    enter_ok[goal] = True
    for dy, dx in NEWS_MOVES:
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
def test_news_oracle_matches_scipy_dijkstra(H, W):
    """Positive costs: the fp32 fold is within H*W * 2^-24 (relative) of the float64 4-connected optimum, both agree
    on which cells reach the goal, and it is never below the Moore optimum of the same map."""
    B = 4
    cost, passable, goal = _random_costs(B, H, W, seed=H * 1000 + W + 1)
    o = _oracle(cost, goal, passable)
    moore = wlabels.weighted_labels(cost, goal, passable)
    assert (o["status"] == 0).all()
    assert o["act_mask"].max() < 16
    for b in range(B):
        ref = _scipy_dists(cost[b], passable[b], int(goal[b]))
        d = -o["dists"][b, 0].ravel().astype(np.float64)
        assert np.array_equal(np.isinf(d), np.isinf(ref))
        fin = np.isfinite(ref)
        assert np.all(np.abs(d[fin] - ref[fin]) <= H * W * 2.0 ** -24 * ref[fin])
        dm = -moore["dists"][b, 0].ravel()
        assert np.all(dm[fin] <= d[fin])


def _D(o, b):
    """the cost-to-go plane of map b (dists = 0 - D, so 0 - dists gives D back bit for bit, +0 included)"""
    return np.float32(0.0) - o["dists"][b, 0].ravel()


def _fold(cost, cells):
    """fp32 left fold from the goal over a path's cells, the first (start) excluded"""
    x = np.float32(0.0)
    for c in reversed(cells[1:]):
        x = np.float32(x + cost[c])
    return x


def _check_rollouts(cost, goal, o, b):
    """Every roll-out of `action` from a reachable cell moves between 4-neighbours only, reaches the goal after exactly
    hop moves, lowers hop by one per move, and its fold equals D (= -dists) bit for bit."""
    H, W = cost.shape[-2:]
    c = cost[b].ravel()
    D = _D(o, b)
    hop = o["hops"][b, 0].ravel()
    act = o["action"][b, 0].ravel()
    for s in np.flatnonzero(np.isfinite(D)):
        path = [int(s)]
        v = int(s)
        while v != goal[b]:
            assert len(path) <= hop[s], "a roll-out takes more than hop moves"
            assert 0 <= act[v] < 4, "a NEWS policy takes a diagonal move"
            dy, dx = NEWS_MOVES[act[v]]
            y, x = divmod(v, W)
            assert 0 <= y + dy < H and 0 <= x + dx < W
            t = (y + dy) * W + x + dx
            assert hop[t] == hop[v] - 1
            v = t
            path.append(v)
        assert len(path) == hop[s] + 1
        assert _fold(c, path).tobytes() == np.float32(D[s]).tobytes(), "the fold along the roll-out is not D"


@pytest.mark.parametrize("H,W", [(12, 12), (5, 40), (33, 31)])
def test_news_oracle_rollouts_with_zero_costs(H, W):
    B = 6
    cost, passable, goal = _random_costs(B, H, W, seed=17 + H, zero_frac=0.3)
    o = _oracle(cost, goal, passable)
    for b in range(B):
        _check_rollouts(cost, goal, o, b)


def test_news_oracle_rollouts_on_absorbed_costs():
    """Costs of 1e-9 beside distances near 1e4 are absorbed (fl(D + c) == D), so every move between such cells is
    optimal and the optimal moves form cycles; the hop rule still sends every roll-out to the goal, and hop is the
    Manhattan distance on the open map."""
    H, W = 12, 12
    cost = np.full((2, H, W), 1e-9, np.float32)
    cost[0, 0, 0] = 1e4                       # the goal of map 0: every other cell has D == 1e4
    rs = np.random.RandomState(13)
    cost[1] = np.where(rs.rand(H, W) < 0.5, 1e-9, 1e4).astype(np.float32)
    goal = np.array([0, H * W - 1], np.int32)
    o = _oracle(cost, goal)
    assert (_D(o, 0)[1:] == np.float32(1e4)).all()
    ys, xs = np.divmod(np.arange(H * W), W)
    assert np.array_equal(o["hops"][0, 0].ravel(), ys + xs)          # Manhattan distance to the corner goal
    for b in range(2):
        _check_rollouts(cost, goal, o, b)
    starts = np.array([H * W - 1, 0], np.int32)
    o = _oracle(cost, goal, start_idx=starts)
    for b in range(2):
        s = starts[b]
        assert o["path_maps"][b].sum() == o["hops"][b, 0].ravel()[s] + 1
        assert o["path_costs"][b] == np.float32(cost[b].ravel()[s] + _D(o, b)[s])


def test_news_oracle_reduces_to_news_unit_labels_on_fixtures():
    """cost = (map != 0), passable = map, a passable goal: -D equals the NEWS unit labels' dists on every reachable
    cell, hop equals D, and the policy equals their max set (and first member) on every reachable non-goal cell."""
    n = 0
    for name in labels_golden.NAMES:
        maps, goal_idx, _, _ = labels_golden.load(name)
        B = maps.shape[0]
        keep = maps.reshape(B, -1)[np.arange(B), goal_idx] != 0
        maps, goal_idx = maps[keep], goal_idx[keep]
        B, H, W = maps.shape
        ud, um, ua = label_oracle.opt_labels(maps, goal_idx, mechanism="news")
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


def test_news_oracle_status_and_edge_cases():
    H, W = 6, 7
    cost = np.ones((7, H, W), np.float32)
    passable = np.ones_like(cost)
    goal = np.array([10, 10, 99, 10, 10, 10, 10], np.int32)     # map 2: no goal
    starts = np.array([0, 0, 0, 0, 10, 0, 0], np.int32)         # map 4: start == goal
    cost[0, 3, 3] = -1.0                                        # a negative cost on a passable cell
    cost[1, 3, 3] = np.inf
    passable[1, 3, 3] = 0.0                                     # ... on an obstacle it is never charged
    passable[3, :, 2] = 0.0                                     # map 3: a wall between the start and the goal
    passable[5, 1, 3] = 0.0                                     # map 5: a goal that is not passable is still the
    cost[5, 1, 3] = 2.5                                         # source, and its cost is charged on entering it
    passable[6, 0, 3] = passable[6, 2, 3] = 0.0                 # map 6: the goal's 4 neighbours blocked, its
    passable[6, 1, 2] = passable[6, 1, 4] = 0.0                 # diagonal neighbours open: unreachable in NEWS
    o = _oracle(cost, goal, passable, starts)
    assert o["status"].tolist() == [1 | 4, 0, 2 | 4, 4, 0, 0, 4]
    assert np.isneginf(o["dists"][0]).all() and (o["hops"][0] == -1).all() and (o["action"][0] == -1).all()
    assert (o["act_mask"][0] == 0).all() and np.isinf(o["path_costs"][0]) and o["path_maps"][0].sum() == 0
    assert np.isneginf(o["dists"][2]).all() and (o["hops"][2] == -1).all()
    assert o["path_costs"][4] == cost[4, 1, 3] and o["path_maps"][4].sum() == 1
    assert np.isinf(o["path_costs"][3]) and o["path_maps"][3].sum() == 0
    assert o["path_maps"][1].sum() == o["hops"][1, 0, 0, 0] + 1 == 5      # (0,0) -> (1,3): Manhattan 4
    assert o["path_costs"][1] == 5.0
    assert o["hops"][5, 0, 0, 0] == 4 and o["path_costs"][5] == np.float32(1 + 3 + 2.5)
    reach6 = o["hops"][6, 0] >= 0
    assert reach6.sum() == 1 and reach6[1, 3]                               # only the goal itself
    # the Moore labels reach map 6's goal diagonally
    assert wlabels.weighted_labels(cost, goal, passable, starts)["status"][6] == 0
    with pytest.raises(ValueError):
        wlabels.weighted_labels(cost, goal, passable, starts, mechanism="hex")


def test_weighted_labels_mech_rejects_bad_arguments_without_a_gpu(built_lib):
    L = built_lib.lib()
    f = L.nastar_b200_weighted_labels_mech
    assert "nastar_b200_weighted_labels_mech" in built_lib.EXPORTS and hasattr(L, "nastar_b200_weighted_labels_mech")
    c, p, g, s = 0x10000, 0x20000, 0x30000, 0x40000
    d, h, m, a, pm, pc, st = 0x50000, 0x60000, 0x70000, 0x80000, 0x90000, 0xA0000, 0xB0000
    EINVAL, EUNSUPPORTED = 1, 2
    before = L.nastar_b200_launch_count()

    def call(**kw):
        args = dict(c=c, cs=144, p=p, ps=144, g=g, s=s, B=1, H=12, W=12, mech=1, d=d, h=h, m=m, a=a, pm=pm, pc=pc,
                    st=st)
        args.update(kw)
        return f(*args.values(), None)

    for bad in (-1, 2, 7, 1 << 30):
        assert call(mech=bad) == EINVAL             # neither NASTAR_MECH_MOORE nor NASTAR_MECH_NEWS
    assert call(mech=2, H=129, W=8, cs=129 * 8, ps=129 * 8) == EINVAL      # every argument is checked first
    assert call(c=None) == EINVAL and call(g=None) == EINVAL
    for k in ("d", "h", "m", "a", "st"):
        assert call(**{k: None}) == EINVAL
    assert call(B=0) == EINVAL and call(H=0) == EINVAL and call(W=-1) == EINVAL
    assert call(cs=143) == EINVAL and call(ps=100) == EINVAL
    assert call(pm=None) == EINVAL and call(pc=None) == EINVAL and call(s=None) == EINVAL
    for mech in (0, 1):
        assert call(mech=mech, H=129, W=8, cs=129 * 8, ps=129 * 8) == EUNSUPPORTED
        assert call(mech=mech, H=8, W=200, cs=1600, ps=1600) == EUNSUPPORTED
    assert L.nastar_b200_launch_count() == before   # nothing above was launched
    # the binding refuses an unknown mechanism name before anything else, like opt_labels
    with pytest.raises(ValueError, match="mechanism"):
        built_lib.weighted_labels(torch.ones(1, 12, 12), torch.zeros(1, dtype=torch.int32), mechanism="hex")
    with pytest.raises(RuntimeError):
        built_lib.weighted_labels(torch.ones(1, 12, 12), torch.zeros(1, dtype=torch.int32), mechanism="news")
    from neural_astar.utils.data import compute_weighted_opt_labels, shortest_path_maps

    with pytest.raises(RuntimeError):
        compute_weighted_opt_labels(torch.ones(1, 1, 12, 12), torch.zeros(1, 1, 12, 12), mechanism="news")
    with pytest.raises(RuntimeError):
        shortest_path_maps(torch.ones(1, 1, 12, 12), torch.zeros(1, 1, 12, 12), torch.zeros(1, 1, 12, 12),
                           mechanism="news")


def test_public_signatures_keep_their_positions():
    """The new keyword comes last; every earlier parameter keeps its position and default."""
    import inspect

    from neural_astar import _native
    from neural_astar.utils import data

    for fn, names in ((_native.weighted_labels, ["cost", "goal_idx", "passable", "start_idx", "mechanism"]),
                      (data.compute_weighted_opt_labels, ["cost_maps", "goal_maps", "passable", "mechanism"]),
                      (data.shortest_path_maps, ["cost_maps", "start_maps", "goal_maps", "passable", "mechanism"])):
        params = inspect.signature(fn).parameters
        assert list(params) == names
        assert params["mechanism"].default == "moore" and params["passable"].default is None
