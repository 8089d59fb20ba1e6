"""Search GIFs on the GPU (utils.data.search_gifs, DESIGN.md §19): the decoded frames equal visualize_results of the
planner's own intermediate_results, frame for frame, plus the hold frames."""
from __future__ import annotations

import io
import os
import sys
import warnings

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "neural-astar_b200"), os.path.join(ROOT, "tests")]

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(ROOT, "tests", "golden")


@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    return torch.device("cuda:0")


def _decode(gif: bytes):
    from PIL import Image

    im = Image.open(io.BytesIO(gif))
    frames = []
    for k in range(im.n_frames):
        im.seek(k)
        frames.append(np.asarray(im.convert("RGB")))
    return frames, im


def _expected(planner, maps, starts, goals, scale, hold):
    from neural_astar.utils.data import visualize_results

    out = planner(maps, starts, goals, store_intermediate_results=True)
    frames = [visualize_results(maps, f, scale) for f in out.intermediate_results]
    return frames + [frames[-1]] * hold


def _check(gif, want, duration=30):
    got, im = _decode(gif)
    assert len(got) == len(want)
    for k, (a, b) in enumerate(zip(got, want)):
        assert a.shape == b.shape and np.array_equal(a, b), f"frame {k} differs"
    assert im.info.get("loop") == 0
    for k in range(len(got)):
        im.seek(k)
        assert im.info.get("duration") == duration, k


def _oracle(planner, maps, starts, goals, layout="each", scale=4, fps=30, hold=15, loop=0):
    """oracle/gif_oracle.c's GIFs of the search the planner runs for search_gifs."""
    from neural_astar.planner.differentiable_astar import _recording
    from oracle import gif as G

    token = _recording.set("batch" if layout == "grid" else "each")
    try:
        with torch.no_grad():
            rec = planner(maps, starts, goals, store_intermediate_results=True).intermediate_results
    finally:
        _recording.reset(token)
    B = maps.shape[0]
    m, hist, paths, trace = (t.detach().cpu().numpy() for t in (maps, rec.histories, rec.paths, rec.trace))
    goal = goals.reshape(B, -1).argmax(-1).cpu().numpy()
    T = trace.shape[1]
    ts = rec.t_solve.cpu().numpy()
    own = np.where(ts >= 0, np.minimum(ts + 1, T), T)
    kw = dict(scale=scale, fps=fps, hold=hold, loop=loop)
    if layout == "grid":
        steps = rec.T_batch if rec.T_batch is not None else int(own.max())
        return [G.gif(m, hist, paths, trace, goal, steps, grid=True, **kw)]
    return [G.gif(m[b:b + 1], hist[b:b + 1], paths[b:b + 1], trace[b:b + 1], goal[b:b + 1], int(own[b]), **kw)
            for b in range(B)]


def _gifs(planner, maps, starts, goals, **kw):
    """search_gifs, checked byte for byte against the oracle."""
    from neural_astar.utils.data import search_gifs

    gifs = search_gifs(planner, maps, starts, goals, **kw)
    want = _oracle(planner, maps, starts, goals, **kw)
    assert len(gifs) == len(want)
    for b, (a, w) in enumerate(zip(gifs, want)):
        assert a == w, f"GIF {b}: {len(a)} bytes, the oracle's {len(w)}"
    return gifs


def _random_problem(dev, B, H, W, seed, density=0.25):
    g = np.random.RandomState(seed)
    maps = (g.rand(B, 1, H, W) > density).astype(np.float32)
    starts = np.zeros_like(maps)
    goals = np.zeros_like(maps)
    for b in range(B):
        s, t = g.choice(H * W, 2, replace=False)
        maps[b, 0].flat[s] = maps[b, 0].flat[t] = 1
        starts[b, 0].flat[s] = 1
        goals[b, 0].flat[t] = 1
    return tuple(torch.from_numpy(x).to(dev) for x in (maps, starts, goals))


@pytest.mark.parametrize("g_ratio", [0.5, 0.2, 0.8])
@pytest.mark.parametrize("mechanism", ["moore", "news"])
def test_each_equals_per_map_calls(dev, g_ratio, mechanism):
    from neural_astar.planner import VanillaAstar
    from neural_astar.utils.data import search_gifs

    maps, starts, goals = _random_problem(dev, 6, 20, 20, 1)
    planner = VanillaAstar(g_ratio=g_ratio, mechanism=mechanism).to(dev).eval()
    gifs = _gifs(planner, maps, starts, goals, scale=2, hold=3)
    assert len(gifs) == 6
    for b, gif in enumerate(gifs):
        _check(gif, _expected(planner, maps[b:b + 1], starts[b:b + 1], goals[b:b + 1], 2, 3))


@pytest.mark.parametrize("B", [1, 8, 11])
@pytest.mark.parametrize("g_ratio", [0.5, 0.2])
def test_grid_equals_batched_call(dev, B, g_ratio):
    from neural_astar.planner import VanillaAstar
    from neural_astar.utils.data import search_gifs

    maps, starts, goals = _random_problem(dev, B, 16, 16, 2)
    planner = VanillaAstar(g_ratio=g_ratio).to(dev).eval()
    (gif,) = _gifs(planner, maps, starts, goals, scale=3, hold=2, layout="grid")
    _check(gif, _expected(planner, maps, starts, goals, 3, 2))


@pytest.mark.parametrize("HW,scale", [((20, 12), 1), ((20, 12), 3), ((12, 20), 4), ((64, 128), 1), ((5, 40), 2)])
def test_non_square(dev, HW, scale):
    from neural_astar.planner import VanillaAstar
    from neural_astar.utils.data import search_gifs

    maps, starts, goals = _random_problem(dev, 3, HW[0], HW[1], 3)
    planner = VanillaAstar().to(dev).eval()
    for layout in ("each", "grid"):
        gifs = _gifs(planner, maps, starts, goals, scale=scale, hold=1, layout=layout)
        if layout == "grid":
            _check(gifs[0], _expected(planner, maps, starts, goals, scale, 1))
        else:
            for b, gif in enumerate(gifs):
                _check(gif, _expected(planner, maps[b:b + 1], starts[b:b + 1], goals[b:b + 1], scale, 1))


def test_edge_maps_and_grey_levels(dev):
    """Unreachable goal, start == goal, a step-capped search (train mode, Tmax), many grey levels."""
    from neural_astar.planner import NeuralAstar, VanillaAstar
    from neural_astar.utils.data import search_gifs

    maps, starts, goals = _random_problem(dev, 4, 24, 24, 4)
    maps[0, 0, :, 12] = 0                      # a wall between start and goal
    starts[0].zero_(); goals[0].zero_()
    starts[0, 0, 3, 3] = 1; goals[0, 0, 20, 20] = 1
    maps[0, 0, 3, 3] = maps[0, 0, 20, 20] = 1
    starts[1] = goals[1]                       # start == goal
    g = torch.Generator(device="cpu").manual_seed(0)
    maps[2] = torch.where(maps[2] > 0, torch.randint(60, 256, (1, 24, 24), generator=g).float().to(dev) / 255, maps[2])
    planner = VanillaAstar().to(dev).eval()
    for b, gif in enumerate(_gifs(planner, maps, starts, goals, scale=2, hold=2)):
        _check(gif, _expected(planner, maps[b:b + 1], starts[b:b + 1], goals[b:b + 1], 2, 2))
    # train mode caps the search at Tmax * W * W steps; its batch norm makes the costs depend on the batch, so the
    # grid is checked against the same batch and "each" against one map
    torch.manual_seed(0)
    na = NeuralAstar(Tmax=0.25).to(dev).train()
    with torch.no_grad():
        (gif,) = _gifs(na, maps, starts, goals, scale=1, hold=0, layout="grid")
        _check(gif, _expected(na, maps, starts, goals, 1, 0))
        (gif,) = _gifs(na, maps[3:], starts[3:], goals[3:], scale=1, hold=0)
        _check(gif, _expected(na, maps[3:], starts[3:], goals[3:], 1, 0))


def test_checkpoint_neural_astar_mazes(dev):
    """All 100 mazes_032 test problems with VanillaAstar and the checkpoint's NeuralAstar (fused encoder path)."""
    from neural_astar.planner import NeuralAstar, VanillaAstar
    from neural_astar.utils.data import search_gifs

    from golden_util import Golden

    z = Golden("mazes032_vanilla_test")
    maps, starts, goals = (torch.from_numpy(x).to(dev) for x in (z.obst, z.start, z.goal))
    state = np.load(os.path.join(GOLDEN, "mazes032_ckpt_planner_state.npz"))
    na = NeuralAstar(encoder_arch="CNN", encoder_depth=4).to(dev).eval()
    na.load_state_dict({k: torch.from_numpy(state[k]) for k in state.files})
    for planner in (VanillaAstar().to(dev).eval(), na):
        with torch.no_grad():
            gifs = _gifs(planner, maps, starts, goals, scale=4, hold=15)
            assert len(gifs) == len(maps)
            for b, gif in enumerate(gifs):
                _check(gif, _expected(planner, maps[b:b + 1], starts[b:b + 1], goals[b:b + 1], 4, 15))
            (grid,) = _gifs(planner, maps, starts, goals, scale=4, hold=15, layout="grid")
            _check(grid, _expected(planner, maps, starts, goals, 4, 15))


@pytest.mark.parametrize("HW", [(96, 96), (256, 256)])
def test_large_maps(dev, HW):
    """96x96 and 256x256 maps (T = 65 536 steps on the latter) in both layouts."""
    from neural_astar.planner import VanillaAstar

    H, W = HW
    g = np.random.RandomState(5)
    maps = (g.rand(3, 1, H, W) > 0.2).astype(np.float32)
    starts, goals = np.zeros_like(maps), np.zeros_like(maps)
    for b, (s, t) in enumerate([((H // 3, W // 3), (H // 3 + 40, W // 3 + 30)), ((5, 5), (60, 20)),
                                ((H - 20, W - 50), (H - 60, W - 10))]):
        lo, hi = sorted((s[1], t[1]))
        maps[b, 0, s[0], lo:hi + 1] = 1   # an L-shaped corridor: the goal is reachable
        lo, hi = sorted((s[0], t[0]))
        maps[b, 0, lo:hi + 1, t[1]] = 1
        starts[b, 0][s] = 1
        goals[b, 0][t] = 1
    maps, starts, goals = (torch.from_numpy(x).to(dev) for x in (maps, starts, goals))
    planner = VanillaAstar().to(dev).eval()
    for b, gif in enumerate(_gifs(planner, maps, starts, goals, scale=1, hold=1)):
        _check(gif, _expected(planner, maps[b:b + 1], starts[b:b + 1], goals[b:b + 1], 1, 1))
    (gif,) = _gifs(planner, maps, starts, goals, scale=1, hold=1, layout="grid")
    _check(gif, _expected(planner, maps, starts, goals, 1, 1))


def test_two_launches_three_waits_and_repeatable(dev, monkeypatch):
    from neural_astar import _native
    from neural_astar.planner import VanillaAstar
    from neural_astar.utils.data import search_gifs

    maps, starts, goals = _random_problem(dev, 5, 32, 32, 6)
    planner = VanillaAstar().to(dev).eval()
    first = search_gifs(planner, maps, starts, goals)
    n0 = _native.launch_count()
    planner(maps, starts, goals, store_intermediate_results=False)
    torch.cuda.synchronize()
    search_launches = _native.launch_count() - n0
    waits = []
    real = torch.cuda.Stream.synchronize
    monkeypatch.setattr(torch.cuda.Stream, "synchronize", lambda self: (waits.append(self), real(self))[1])
    n0 = _native.launch_count()
    with warnings.catch_warnings(record=True) as seen:
        warnings.simplefilter("always")
        torch.cuda.set_sync_debug_mode("warn")
        try:
            again = search_gifs(planner, maps, starts, goals)
        finally:
            torch.cuda.set_sync_debug_mode("default")
    syncs = [w for w in seen if str(w.message).startswith("called a synchronizing CUDA operation")]
    assert _native.launch_count() - n0 - search_launches == 2
    assert len(waits) == 3 and len(syncs) <= len(waits), [str(w.message) for w in syncs]
    assert again == first


def test_many_frames_reuse_workers(dev):
    """More frames than resident warps: 64 maps of 64x64 give thousands of frame items."""
    from neural_astar.planner import VanillaAstar
    from neural_astar.utils.data import search_gifs

    maps, starts, goals = _random_problem(dev, 64, 64, 64, 7, density=0.1)
    planner = VanillaAstar().to(dev).eval()
    gifs = _gifs(planner, maps, starts, goals, scale=1, hold=0)
    n = sum(_decode(g)[1].n_frames for g in gifs)
    assert n > 4 * torch.cuda.get_device_properties(dev).multi_processor_count * 4
    for b in (0, 31, 63):
        _check(gifs[b], _expected(planner, maps[b:b + 1], starts[b:b + 1], goals[b:b + 1], 1, 0))


def test_forward_outputs_unchanged(dev):
    from neural_astar.planner import VanillaAstar
    from neural_astar.utils.data import search_gifs

    maps, starts, goals = _random_problem(dev, 4, 32, 32, 8)
    planner = VanillaAstar(g_ratio=0.2).to(dev).eval()
    before = planner(maps, starts, goals, store_intermediate_results=True)
    search_gifs(planner, maps, starts, goals, layout="each")
    after = planner(maps, starts, goals, store_intermediate_results=True)
    assert torch.equal(before.histories, after.histories) and torch.equal(before.paths, after.paths)
    assert len(before.intermediate_results) == len(after.intermediate_results)
    assert isinstance(after.intermediate_results, list)


def test_palette_overflow_and_range_raise_before_the_search(dev):
    from neural_astar import _native
    from neural_astar.planner import VanillaAstar
    from neural_astar.utils.data import search_gifs

    maps, starts, goals = _random_problem(dev, 1, 32, 32, 9)
    planner = VanillaAstar().to(dev).eval()
    many = (torch.arange(32 * 32, device=dev).reshape(1, 1, 32, 32) % 254 + 1).float() / 255   # 254 greys + 0
    n0 = _native.launch_count()
    with pytest.raises(ValueError, match="palette"):
        search_gifs(planner, many, starts, goals)
    with pytest.raises(ValueError, match=r"\[0, 1\]"):
        search_gifs(planner, maps * 2, starts, goals)
    assert _native.launch_count() == n0
    fits = (torch.arange(32 * 32, device=dev).reshape(1, 1, 32, 32) % 252 + 1).float() / 255   # 252 greys + 0
    (gif,) = _gifs(planner, fits, starts, goals, scale=1, hold=0)
    _check(gif, _expected(planner, fits, starts, goals, 1, 0))
