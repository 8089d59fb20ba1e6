"""Search GIFs without a GPU: the C ABI's argument checks (nothing is launched), the record size, and the rejections
of search_gifs that precede any device work."""
from __future__ import annotations

import ctypes
import os
import subprocess
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "neural-astar_b200")]


@pytest.fixture(scope="module")
def native():
    subprocess.check_call(["make", "-C", os.path.join(ROOT, "neural-astar_b200"), "-s", "all"])
    from neural_astar import _native

    return _native


@pytest.fixture
def no_launch(native):
    L = native.lib()
    before = L.nastar_b200_launch_count()
    yield L
    assert L.nastar_b200_launch_count() == before, "a rejected call launched something"


def _params(native, **kw):
    p = native.GifParams()
    p.maps, p.histories, p.paths, p.goal_maps, p.trace, p.t_solve = 0x10000, 0x20000, 0x30000, 0x40000, 0x50000, 0x60000
    p.B, p.H, p.W, p.T = 4, 32, 32, 1024
    p.layout, p.steps_mode = native.GIF_EACH, native.GIF_STEPS_MAP
    p.screen_w, p.screen_h, p.delay_cs = 128, 128, 3
    p.tables = 0x70000
    for k, v in kw.items():
        setattr(p, k, v)
    return p


BAD = [dict(maps=None), dict(trace=None), dict(tables=None), dict(B=0), dict(H=0), dict(T=0), dict(layout=2),
       dict(steps_mode=1), dict(layout=1, steps_mode=0), dict(screen_w=0), dict(screen_h=65536), dict(delay_cs=-1),
       dict(delay_cs=65536)]


@pytest.mark.parametrize("kw", BAD)
def test_plan_rejects_before_launch(native, no_launch, kw):
    p = _params(native, **kw)
    assert no_launch.nastar_b200_gif_workspace_bytes(ctypes.byref(p)) == 0
    assert no_launch.nastar_b200_gif_plan(ctypes.byref(p), 0x80000, 0x90000, 0xA0000, 1 << 30, None) == 1


def test_plan_status_codes(native, no_launch):
    p = _params(native)
    need = no_launch.nastar_b200_gif_workspace_bytes(ctypes.byref(p))
    assert need > 4 * 32 * 32 * 4
    assert no_launch.nastar_b200_gif_plan(ctypes.byref(p), None, 0x90000, 0xA0000, need, None) == 1
    assert no_launch.nastar_b200_gif_plan(ctypes.byref(p), 0x80000, 0x90000, 0xA0000, need - 1, None) == 4
    assert no_launch.nastar_b200_gif_plan(ctypes.byref(p), 0x80000, 0x90000, 0xA0010, need, None) == 1  # alignment
    big = _params(native, H=4097, W=4097)
    assert no_launch.nastar_b200_gif_plan(ctypes.byref(big), 0x80000, 0x90000, 0xA0000, 1 << 40, None) == 2
    grid = _params(native, layout=native.GIF_GRID, steps_mode=native.GIF_STEPS_BATCH)
    # 4 maps in one row of make_grid: 36 x 138 image
    assert no_launch.nastar_b200_gif_tables_bytes(ctypes.byref(grid)) == 4 * (128 + 128 + 2 * 138 + 2 * 36) + 258


def test_encode_checks_offsets(native, no_launch):
    import numpy as np

    p = _params(native)
    need = no_launch.nastar_b200_gif_workspace_bytes(ctypes.byref(p))
    nb = np.array([300, 5, 1], np.int32)
    off = np.concatenate([[0], np.cumsum(native.gif_record_bytes(nb))]).astype(np.int64)

    def enc(nb, off, n, out_bytes, ws=need):
        return no_launch.nastar_b200_gif_encode(ctypes.byref(p), 0x80000, nb.ctypes.data, off.ctypes.data, 0x90000,
                                                n, 0xB0000, out_bytes, 0xA0000, ws, None)

    assert enc(nb, off, 3, int(off[-1]) - 1) == 1
    bad = off.copy()
    bad[2] += 1
    assert enc(nb, bad, 3, 1 << 20) == 1
    assert enc(nb, off, 0, 1 << 20) == 1
    assert enc(nb, off, 4 * 1025 + 1, 1 << 20) == 1
    assert enc(np.array([300, 0, 1], np.int32), off, 3, 1 << 20) == 1
    assert enc(nb, off, 3, int(off[-1]), ws=need - 1) == 4


def test_record_bytes(native):
    L = native.lib()
    for n in (1, 254, 255, 256, 510, 511, 100000):
        assert L.nastar_b200_gif_record_bytes(n) == 19 + n + -(-n // 255) + 1 == native.gif_record_bytes(n)
    assert L.nastar_b200_gif_record_bytes(0) == -1


def test_lzw_of_one_pixel_decodes():
    """The hold frame's stream (clear, index, end) decodes with Pillow to the index."""
    import io

    import numpy as np
    from PIL import Image

    from neural_astar.utils.data import _gif_lzw_pixel

    for m in (2, 3, 8):
        P = 1 << m
        idx = P - 1
        lzw = _gif_lzw_pixel(m, idx)
        gif = (b"GIF89a\x01\x00\x01\x00" + bytes([0x80 | (m - 1) << 4 | (m - 1), 0, 0]) + bytes(3 * P)
               + b"\x2c\x00\x00\x00\x00\x01\x00\x01\x00\x00" + bytes([m, len(lzw)]) + lzw + b"\x00;")
        im = Image.open(io.BytesIO(gif))
        assert np.asarray(im)[0, 0] == idx


def test_search_gifs_rejections_precede_device_work():
    from neural_astar.planner import NeuralAstar, VanillaAstar
    from neural_astar.utils.data import _gif_geometry, search_gifs

    maps = torch.ones(2, 1, 8, 8)
    marks = torch.zeros(2, 1, 8, 8)
    with pytest.raises(ValueError, match="intermediate"):
        search_gifs(VanillaAstar(use_differentiable_astar=False), maps, marks, marks)
    with pytest.raises(TypeError):
        search_gifs(object(), maps, marks, marks)
    with pytest.raises(ValueError, match=r"\[B,1,H,W\]"):
        search_gifs(NeuralAstar(encoder_input="rgb+"), torch.ones(2, 3, 8, 8), marks, marks)
    with pytest.raises(ValueError, match="layout"):
        search_gifs(VanillaAstar(), maps, marks, marks, layout="row")
    with pytest.raises(ValueError):
        search_gifs(VanillaAstar(), maps, marks, marks, scale=0)
    with pytest.raises(ValueError, match="65535"):
        search_gifs(VanillaAstar(), torch.ones(1, 1, 8, 20000), marks, marks, scale=4)
    with pytest.raises(RuntimeError, match="CUDA"):
        search_gifs(VanillaAstar(), maps, marks, marks)
    assert _gif_geometry(100, 32, 32, 4, True) == (13 * 34 + 2, 8 * 34 + 2, (13 * 34 + 2) * 4, (8 * 34 + 2) * 4)
    assert _gif_geometry(1, 20, 12, 3, True) == (20, 12, 60, 36)
    assert _gif_geometry(1, 20, 12, 1, False) == (20, 12, 12, 20)


# ---- the oracle's GIFs, decoded by Pillow, against visualize_results of the frames of golden traces ---------------
def _decode(gif: bytes):
    import io

    import numpy as np
    from PIL import Image

    im = Image.open(io.BytesIO(gif))
    frames, durations = [], []
    for k in range(im.n_frames):
        im.seek(k)
        frames.append(np.asarray(im.convert("RGB")))
        durations.append(im.info.get("duration"))
    return frames, durations, im.info.get("loop")


def _frames(maps, hist, paths, trace, goal, steps):
    """The frames _materialise_frames builds, from a trace: closed set before step t and the cell selected at t, then
    the final histories and paths."""
    import numpy as np

    n, _, H, W = maps.shape
    tr = np.asarray(trace[:, :steps], np.int64)
    tr = np.where(tr < 0, np.asarray(goal)[:, None], tr)
    closed = np.zeros((n, H * W), np.float32)
    frames = []
    for t in range(steps):
        sel = np.zeros((n, H * W), np.float32)
        sel[np.arange(n), tr[:, t]] = 1
        frames.append({"histories": torch.from_numpy(closed.reshape(n, 1, H, W).copy()),
                       "paths": torch.from_numpy(sel.reshape(n, 1, H, W))})
        closed[np.arange(n), tr[:, t]] = 1
    frames.append({"histories": torch.from_numpy(np.asarray(hist, np.float32)), "paths": torch.from_numpy(paths)})
    return frames


def _check_oracle(maps, hist, paths, trace, goal, steps, grid, scale, hold=3, fps=30):
    import numpy as np

    from neural_astar.utils.data import visualize_results
    from oracle import gif as G

    g = G.gif(maps, hist, paths, trace, goal, steps, grid=grid, scale=scale, fps=fps, hold=hold)
    got, durations, loop = _decode(g)
    want = [visualize_results(torch.from_numpy(maps), f, scale)
            for f in _frames(maps, hist, paths, trace, goal, steps)]
    want += [want[-1]] * hold
    assert len(got) == len(want) == steps + 1 + hold
    for k, (a, b) in enumerate(zip(got, want)):
        assert a.shape == b.shape and np.array_equal(a, b), f"frame {k}"
    assert durations == [10 * round(100 / fps)] * len(got) and loop == 0
    return g


def _golden(name, n=None):
    from golden_util import Golden

    z = Golden(name)
    sl = slice(None) if n is None else slice(0, n)
    return (z.obst[sl], z.bits("hist_bits")[sl].astype("float32"), z.bits("path_bits")[sl].astype("int64"),
            z.z["trace"][sl], z.z["goal_idx"][sl], int(z.z["T_batch"]))


def _own_steps(trace, goal, T):
    """A map's steps searched alone (uncoupled): through its first selection of the goal."""
    import numpy as np

    hit = np.flatnonzero(np.asarray(trace) == goal)
    return int(hit[0]) + 1 if len(hit) else T


@pytest.mark.parametrize("name,n,scales", [("mazes032_vanilla_test", 12, (4,)), ("rect64x128_vanilla", None, (1, 3, 4)),
                                           ("news/news_mazes032_vanilla", 10, (2,)), ("mazes032_lowg_gr02", 16, (1,))])
def test_oracle_frames_equal_visualize_results(name, n, scales):
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    maps, hist, paths, trace, goal, T_batch = _golden(name, n)
    for scale in scales:
        # one GIF of the batch (for the g_ratio < 0.5 golden: the coupled T_batch), and one map alone
        _check_oracle(maps, hist, paths, trace, goal, T_batch, True, scale)
        if "lowg" not in name:
            s = _own_steps(trace[0], goal[0], T_batch)
            _check_oracle(maps[:1], hist[:1], paths[:1], trace[:1], goal[:1], s, False, scale)


def _synthetic(H, W, steps, seed, greys=None):
    import numpy as np

    g = np.random.RandomState(seed)
    maps = (np.ones((1, 1, H, W), np.float32) if greys is None else
            (g.choice(greys, (1, 1, H, W)).astype(np.float32) / np.float32(255)))
    trace = g.randint(0, H * W, (1, steps)).astype(np.int32)
    trace[0, steps // 2:] = -1   # past the map's own search: the goal
    goal = np.array([H * W - 1])
    hist = np.zeros((1, 1, H, W), np.float32)
    hist.reshape(-1)[trace[0, : steps // 2]] = 1
    paths = np.zeros((1, 1, H, W), np.int64)
    paths.reshape(-1)[[0, H * W - 1]] = 1
    return maps, hist, paths, trace, goal


def test_lzw_edge_cases():
    import numpy as np

    # a 1x1 map: every frame is one pixel
    maps, hist, paths, trace, goal = _synthetic(1, 1, 4, 0)
    _check_oracle(maps, hist, paths, trace, goal, 4, False, 1)
    # a 4-entry palette (grey 0 only) and a 256-entry one (252 greys and 0)
    maps, hist, paths, trace, goal = _synthetic(8, 8, 6, 1, greys=[0])
    g = _check_oracle(maps, hist, paths, trace, goal, 6, False, 2)
    assert g[10] & 7 == 1
    maps, hist, paths, trace, goal = _synthetic(32, 32, 6, 2, greys=np.arange(1, 253))
    g = _check_oracle(maps, hist, paths, trace, goal, 6, False, 1)
    assert g[10] & 7 == 7
    # a noisy 256x256 map with many grey levels at scale 1: frame 0 fills the 4096-entry table many times
    maps, hist, paths, trace, goal = _synthetic(256, 256, 4, 3, greys=np.arange(0, 250))
    g = _check_oracle(maps, hist, paths, trace, goal, 4, False, 1, hold=1)
    assert len(g) > 65536
    # all-transparent strips: a grid whose frames change two far-apart maps only
    maps, hist, paths, trace, goal = _synthetic(16, 16, 6, 4)
    maps = np.repeat(maps, 16, 0)
    hist, paths = np.repeat(hist, 16, 0), np.repeat(paths, 16, 0)
    trace = np.repeat(trace, 16, 0)
    trace[1:15] = goal[0]
    goal = np.repeat(goal, 16)
    _check_oracle(maps, hist, paths, trace, goal, 6, True, 3)


def test_oracle_palette_overflow():
    import numpy as np

    from oracle import gif as G

    maps, hist, paths, trace, goal = _synthetic(64, 64, 2, 5, greys=np.arange(1, 255))   # 254 greys + 0
    with pytest.raises(ValueError):
        G.gif(maps, hist, paths, trace, goal, 2)
