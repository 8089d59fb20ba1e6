"""Dataset readers with the reference's interface (host-side I/O; not part of the GPU hot path), and the labels
that turn new maps into a planning dataset (optimal distances and policies computed on the GPU).

Same public names and return conventions as /root/reference/src/neural_astar/utils/data.py:
`create_dataloader` / `MazeDataset` (:54-245), `create_warcraft_dataloader` / `WarCraftDataset`
(:248-295), `visualize_results` (:16-51).  File formats: the planning-datasets `.npz`
(arr_0..11 = {train,valid,test} x {maps, goals, optimal policies, optimal distances}, :127-150)
and the WarCraft `.npy` pairs (:273-282).
"""
from __future__ import annotations

import functools
import os

import numpy as np
import torch
import torch.utils.data as data

from .. import _native
from ..planner.differentiable_astar import AstarOutput

# Moore-neighbourhood action order used by the dataset's optimal policies (reference :234-243)
_ACTION_TO_MOVE = ((0, -1, 0), (0, 0, +1), (0, 0, -1), (0, +1, 0), (0, -1, +1), (0, -1, -1), (0, +1, +1), (0, +1, -1))
_SPLIT_OFFSET = {"train": 0, "valid": 4, "test": 8}


def _make_grid(x: torch.Tensor, nrow: int = 8, padding: int = 2) -> torch.Tensor:
    """torchvision.utils.make_grid(x) with its defaults, without the torchvision dependency: a [B,C,H,W] batch
    (single-channel images repeated to RGB) tiled 8 per row with a 2-pixel zero border; a batch of ONE image is
    returned as is, unpadded — exactly like torchvision."""
    x = x.detach().cpu()
    if x.dim() == 3:
        x = x.unsqueeze(0)
    if x.shape[1] == 1:
        x = x.repeat(1, 3, 1, 1)
    B, C, H, W = x.shape
    if B == 1:
        return x[0]
    xmaps = min(nrow, B)
    ymaps = -(-B // xmaps)
    hh, ww = H + padding, W + padding
    grid = x.new_zeros((C, hh * ymaps + padding, ww * xmaps + padding))
    for k in range(B):
        yy, xx = divmod(k, xmaps)
        grid[:, yy * hh + padding:yy * hh + padding + H, xx * ww + padding:xx * ww + padding + W] = x[k]
    return grid


def visualize_results(map_designs: torch.Tensor, planner_outputs, scale: int = 1) -> np.ndarray:
    """Search results as one uint8 RGB image [Hg, Wg, 3] (reference :16-51): the maps tiled like
    torchvision's make_grid (8 per row, 2-pixel border), explored nodes painted (0.2, 0.8, 0), path cells
    (1, 0, 0), values * 255 — the format scripts/create_gif.py hands to moviepy.  `scale` > 1 enlarges with
    nearest-neighbour resampling (the reference passes (rows*scale, cols*scale) to PIL as (width, height);
    kept as is)."""
    if isinstance(planner_outputs, dict):
        histories, paths = planner_outputs["histories"], planner_outputs["paths"]
    else:
        histories, paths = planner_outputs.histories, planner_outputs.paths
    results = _make_grid(map_designs.float()).permute(1, 2, 0).clone()
    h = _make_grid(histories.float()).permute(1, 2, 0)
    p = _make_grid(paths.float()).permute(1, 2, 0)
    results[h[..., 0] == 1] = torch.tensor([0.2, 0.8, 0.0])
    results[p[..., 0] == 1] = torch.tensor([1.0, 0.0, 0.0])
    results = (results.numpy() * 255.0).astype("uint8")
    if scale > 1:
        from PIL import Image

        results = np.asarray(Image.fromarray(results).resize([x * scale for x in results.shape[:2]],
                                                             resample=Image.NEAREST))
    return results


_GIF_GREEN, _GIF_RED = (51, 204, 0), (255, 0, 0)   # uint8 of visualize_results' (0.2, 0.8, 0) * 255 and (1, 0, 0)


def _gif_index_map(n_in: int, n_out: int) -> np.ndarray:
    """The source index of each of n_out samples that Pillow's NEAREST resize takes from n_in, read from Pillow
    itself by resizing a row of indices."""
    if n_in == n_out:
        return np.arange(n_in, dtype=np.int32)
    from PIL import Image

    row = Image.fromarray(np.arange(n_in, dtype=np.int32)[None, :])
    return np.asarray(row.resize((n_out, 1), resample=Image.NEAREST), dtype=np.int32)[0]


def _gif_geometry(B: int, H: int, W: int, scale: int, grid: bool):
    """(image rows, image columns, screen width, screen height) of visualize_results(maps, ., scale): the
    make_grid image, enlarged to (rows * scale, cols * scale) given to Pillow as (width, height)."""
    if grid and B > 1:
        xmaps = min(8, B)
        Hi, Wi = (H + 2) * (-(-B // xmaps)) + 2, (W + 2) * xmaps + 2
    else:
        Hi, Wi = H, W
    SW, SH = (Hi * scale, Wi * scale) if scale > 1 else (Wi, Hi)
    if SW > 0xFFFF or SH > 0xFFFF:
        raise ValueError(f"search_gifs: the {SW}x{SH} screen has a side above 65535")
    return Hi, Wi, SW, SH


def _gif_lzw_pixel(m: int, index: int) -> bytes:
    """The LZW stream of one pixel: clear, the index, end of information, each m + 1 bits, LSB first."""
    v = (1 << m) | (index << (m + 1)) | (((1 << m) + 1) << (2 * (m + 1)))
    return v.to_bytes(-(-3 * (m + 1) // 8), "little")


def search_gifs(planner, map_designs: torch.Tensor, start_maps: torch.Tensor, goal_maps: torch.Tensor,
                scale: int = 4, fps: float = 30, hold: int = 15, layout: str = "each", loop: int = 0):
    """Animated GIFs of the planner's search, as bytes (DESIGN.md §19).

    The planner (VanillaAstar or NeuralAstar with the differentiable search) runs once with a trace, then two kernel
    launches draw and LZW-encode every frame on the device.  layout "each": one GIF per map, whose frames are
    visualize_results(map_designs[b:b+1], f, scale) for f in the intermediate_results of the planner run on map b
    alone, then the last frame `hold` more times.  layout "grid": one GIF whose frames are visualize_results of the
    whole batch over the batched call's intermediate_results, then `hold` copies of the last.  Exact colours: the
    maps' grey levels, (51, 204, 0) explored, (255, 0, 0) selected or on the path, black border.  Each frame after the
    first covers only the pixels that changed, the rest transparent; a frame equal to the previous one is one
    transparent pixel.  map_designs: [B,1,H,W] CUDA tensor with values in [0, 1].  A NeuralAstar in train mode
    normalises its encoder's batch with the batch's own statistics, so there GIF b of "each" shows map b searched within
    the batch, which equals map b searched alone only for a batch of one.  The search runs in the caller's autograd mode,
    because a NeuralAstar's encoder takes its folded inference path only without autograd, and the frames are those of
    a plain call in the same mode; call it under torch.no_grad() for inference (any graph is freed on return).  The host waits three times: for the
    maps' grey levels, for the frame sizes and for the bytes (a batch-coupled grid search waits once more itself)."""
    from ..planner.astar import VanillaAstar
    from ..planner.differentiable_astar import _recording

    if not isinstance(planner, VanillaAstar):
        raise TypeError("search_gifs: the planner must be a VanillaAstar or a NeuralAstar")
    if not planner.use_differentiable_astar:
        raise ValueError("search_gifs: use_differentiable_astar=False (pq_astar) has no intermediate results")
    if layout not in ("each", "grid"):
        raise ValueError(f"search_gifs: layout must be 'each' or 'grid' (got {layout!r})")
    if map_designs.ndim != 4 or map_designs.shape[1] != 1:
        raise ValueError(f"search_gifs: map_designs must be [B,1,H,W] grey maps (got {tuple(map_designs.shape)})")
    if int(scale) != scale or scale < 1 or hold < 0 or int(hold) != hold or not fps > 0 or not 0 <= loop <= 0xFFFF:
        raise ValueError("search_gifs: scale >= 1 and hold >= 0 are integers, fps > 0, 0 <= loop <= 65535")
    delay = round(100 / fps)
    if delay > 0xFFFF:
        raise ValueError("search_gifs: fps is too low for a 16-bit delay")
    B, _, H, W = map_designs.shape
    grid = layout == "grid"
    Hi, Wi, SW, SH = _gif_geometry(B, H, W, int(scale), grid)
    if not map_designs.is_cuda:
        raise RuntimeError("search_gifs: map_designs must be a CUDA tensor (there is no CPU fallback)")
    dev = map_designs.device
    maps = map_designs.detach().float()
    G = 1 if grid else B
    with torch.cuda.device(dev):
        stream = torch.cuda.current_stream(dev)
        # wait 1: the grey levels of each GIF's maps and their range, before anything runs
        grey = (maps * 255).to(torch.uint8).reshape(B, -1).long()
        present = torch.zeros((B, 256), dtype=torch.bool, device=dev).scatter_(1, grey, True)
        if grid:
            present = present.any(0, keepdim=True)
        lo_hi = torch.stack(torch.aminmax(maps)).reshape(1, 2)
        probe = torch.cat([present.float(), lo_hi.expand(G, 2)], 1).to("cpu", non_blocking=True)
        stream.synchronize()
        probe = probe.numpy()
        if not (probe[0, 256] >= 0 and probe[0, 257] <= 1):
            raise ValueError("search_gifs: map_designs must hold values in [0, 1]")
        present = probe[:, :256] > 0
        present[:, 0] = True
        n_grey = present.sum(1)
        bits = np.maximum(2, np.ceil(np.log2(n_grey + 3))).astype(np.int64)
        if bits.max() > 8:
            raise ValueError(f"search_gifs: {int(n_grey.max())} grey levels and 3 more colours do not fit a "
                             "256-entry palette")
        token = _recording.set("batch" if grid else "each")
        try:
            rec = planner(map_designs, start_maps, goal_maps, store_intermediate_results=True).intermediate_results
        finally:
            _recording.reset(token)
        if grid:
            steps_mode = _native.GIF_STEPS_ALL if rec.T_batch is not None else _native.GIF_STEPS_BATCH
        else:
            steps_mode = _native.GIF_STEPS_MAP
        p, keep = _native.gif_params(maps, rec.histories, rec.paths, rec.goal_maps.float(), rec.trace,
                                     rec.t_solve, _native.GIF_GRID if grid else _native.GIF_EACH, steps_mode, SW, SH,
                                     delay)
        xmap = _gif_index_map(Wi, SW)
        ymap = _gif_index_map(Hi, SH)
        xspan = np.stack([np.searchsorted(xmap, np.arange(Wi), "left"), np.searchsorted(xmap, np.arange(Wi), "right")],
                         1)
        yspan = np.stack([np.searchsorted(ymap, np.arange(Hi), "left"), np.searchsorted(ymap, np.arange(Hi), "right")],
                         1)
        lut = np.zeros((G, 256), np.uint8)
        for g in range(G):
            levels = np.flatnonzero(present[g])
            lut[g, levels] = np.arange(len(levels))
        colors = np.stack([n_grey, bits], 1).astype(np.uint8)
        host = np.concatenate([np.concatenate([xmap, ymap, xspan.ravel(), yspan.ravel()]).astype("<i4").view(np.uint8),
                               lut.ravel(), colors.ravel()])
        assert len(host) == _native.gif_tables_bytes(p)
        tables_h = torch.from_numpy(host).pin_memory()
        tables = tables_h.to(dev, non_blocking=True)
        p.tables = tables.data_ptr()
        steps, nbytes, ws = _native.gif_plan(p, dev)
        # wait 2: the steps of each GIF and the size of every frame's LZW stream
        steps_h = steps.to("cpu", non_blocking=True)
        nbytes_h = nbytes.to("cpu", non_blocking=True)
        stream.synchronize()
        steps_h = steps_h.numpy().astype(np.int64)
        F = int((steps_h + 1).sum())
        nb = nbytes_h.numpy()[:F]
        offset = np.concatenate([[0], np.cumsum(_native.gif_record_bytes(nb))]).astype(np.int64)
        offset_h = torch.from_numpy(offset).pin_memory()
        offset_d = offset_h.to(dev, non_blocking=True)
        out = _native.gif_encode(p, nbytes, nb, offset, offset_d, ws)
        # wait 3: exactly the records' bytes
        image = torch.empty((int(offset[-1]),), dtype=torch.uint8, pin_memory=True)
        image.copy_(out[:int(offset[-1])], non_blocking=True)
        stream.synchronize()
        del keep, tables_h, offset_h
    img = image.numpy().tobytes()
    frame0 = np.concatenate([[0], np.cumsum(steps_h + 1)])
    gifs = []
    for g in range(G):
        P = 1 << int(bits[g])
        levels = np.flatnonzero(present[g])
        pal = np.zeros((P, 3), np.uint8)
        pal[:len(levels)] = levels[:, None]
        pal[len(levels)] = _GIF_GREEN
        pal[len(levels) + 1] = _GIF_RED
        m = int(bits[g])
        head = (b"GIF89a" + SW.to_bytes(2, "little") + SH.to_bytes(2, "little") + bytes([0x80 | (m - 1) << 4 | (m - 1), 0, 0])
                + pal.tobytes() + b"\x21\xff\x0bNETSCAPE2.0\x03\x01" + int(loop).to_bytes(2, "little") + b"\x00")
        lzw = _gif_lzw_pixel(m, len(levels) + 2)
        still = (b"\x21\xf9\x04\x05" + delay.to_bytes(2, "little") + bytes([len(levels) + 2, 0])
                 + b"\x2c\x00\x00\x00\x00\x01\x00\x01\x00\x00" + bytes([m, len(lzw)]) + lzw + b"\x00")
        gifs.append(head + img[offset[frame0[g]]:offset[frame0[g + 1]]] + still * int(hold) + b";")
    return gifs


def save_search_gifs(paths, planner, map_designs: torch.Tensor, start_maps: torch.Tensor, goal_maps: torch.Tensor,
                     **kwargs) -> None:
    """search_gifs(planner, map_designs, start_maps, goal_maps, **kwargs), each GIF written to its path (one path for
    layout "grid", one per map for "each")."""
    paths = [paths] if isinstance(paths, (str, os.PathLike)) else list(paths)
    G = 1 if kwargs.get("layout", "each") == "grid" else map_designs.shape[0]
    if len(paths) != G:
        raise ValueError(f"save_search_gifs: {G} GIFs, {len(paths)} paths")
    for path, gif in zip(paths, search_gifs(planner, map_designs, start_maps, goal_maps, **kwargs)):
        with open(path, "wb") as f:
            f.write(gif)


class MazeDataset(data.Dataset):
    def __init__(self, filename: str, split: str, pct1: float = 0.55, pct2: float = 0.70, pct3: float = 0.85,
                 num_starts: int = 1):
        """Shortest-path problems from a planning-datasets .npz (reference :82-125).

        __getitem__ returns (map_design [1,W,W], start_map [num_starts,W,W], goal_map [1,W,W],
        opt_traj [num_starts,W,W]) as float32 arrays.
        """
        assert filename.endswith("npz")
        self.filename = filename
        self.dataset_type = split
        self.pcts = np.array([pct1, pct2, pct3, 1.0])
        self.num_starts = num_starts
        with np.load(filename) as f:
            k = _SPLIT_OFFSET[split]
            self.map_designs, self.goal_maps, self.opt_policies, self.opt_dists = (
                f[f"arr_{k + j}"].astype(np.float32) for j in range(4))
        label = {"train": "Train", "valid": "Validation", "test": "Test"}[split]
        print(f"Number of {label} Samples: {self.map_designs.shape[0]}")
        print(f"\tSize: {self.map_designs.shape[1]}x{self.map_designs.shape[2]}")
        self.num_actions = self.opt_policies.shape[1]
        self.num_orient = self.opt_policies.shape[2]

    def __len__(self):
        return self.map_designs.shape[0]

    def __getitem__(self, index: int):
        """Same samples and the same np.random consumption as the reference (:152-166), but the per-map work
        that does not depend on the draw (percentile bands, the policy's successor table) is computed once
        and cached — at GPU training speeds the reference's per-sample NumPy work is the bottleneck
        (SURVEY.md 8(f) rank 4)."""
        map_design = self.map_designs[index][np.newaxis]
        goal_map = self.goal_maps[index]
        bands, succ = self._prepared(index)
        H, W = goal_map.shape[-2:]
        goal_flat = int(np.argmax(goal_map.reshape(-1)))
        starts = np.zeros((self.num_starts, H, W), np.float32)
        trajs = np.zeros((self.num_starts, H, W), np.float32)
        for k in range(self.num_starts):
            r = np.random.randint(0, len(bands))          # same draw order as get_random_start_map
            loc = int(np.random.choice(bands[r]))
            starts[k].reshape(-1)[loc] = 1.0
            flat = trajs[k].reshape(-1)
            while loc != goal_flat:
                flat[loc] = 1.0
                loc = int(succ[loc])
                assert flat[loc] == 0.0, "Revisiting the same position while following the optimal policy"
        return map_design, starts, goal_map, trajs

    def _prepared(self, index: int):
        cache = self.__dict__.setdefault("_cache", {})
        hit = cache.get(index)
        if hit is None:
            od = self.opt_dists[index].flatten()
            th = np.percentile(od[od > od.min()], 100.0 * (1 - self.pcts))
            bands = [np.where((od >= th[r + 1]) & (od <= th[r]))[0] for r in range(len(th) - 1)]
            policy = self.opt_policies[index]                       # [A, 1, H, W] one-hot over actions
            H, W = policy.shape[-2:]
            act = policy.reshape(policy.shape[0], -1).argmax(0)      # first maximal action, like np.argmax
            moves = np.array([m[1] * W + m[2] for m in _ACTION_TO_MOVE])
            succ = np.arange(H * W) + moves[act]
            hit = cache[index] = (bands, succ)
        return hit

    def get_random_start_map(self, opt_dist: np.ndarray) -> np.ndarray:
        """Pick a start uniformly inside one of the 55-70 / 70-85 / 85-100 percentile bands of the optimal
        distance (reference :200-221; consumes np.random in the same order: randint then choice)."""
        od = opt_dist.flatten()
        th = np.percentile(od[od > od.min()], 100.0 * (1 - self.pcts))
        r = np.random.randint(0, len(th) - 1)
        candidates = np.where((od >= th[r + 1]) & (od <= th[r]))[0]
        start = np.zeros_like(opt_dist)
        start.ravel()[np.random.choice(candidates)] = 1.0
        return start

    def get_opt_traj(self, start_map: np.ndarray, goal_map: np.ndarray, opt_policy: np.ndarray) -> np.ndarray:
        """Roll the optimal policy out from the start until the goal (reference :171-198)."""
        traj = np.zeros_like(start_map)
        policy = opt_policy.transpose((1, 2, 3, 0))
        loc = tuple(np.array(np.nonzero(start_map)).squeeze())
        goal = tuple(np.array(np.nonzero(goal_map)).squeeze())
        while loc != goal:
            traj[loc] = 1.0
            nxt = self.next_loc(loc, policy[loc])
            assert traj[nxt] == 0.0, "Revisiting the same position while following the optimal policy"
            loc = nxt
        return traj

    def next_loc(self, current_loc: tuple, one_hot_action: np.ndarray) -> tuple:
        return tuple(np.add(current_loc, _ACTION_TO_MOVE[int(np.argmax(one_hot_action))]))


def create_dataloader(filename: str, split: str, batch_size: int, num_starts: int = 1,
                      shuffle: bool = False) -> data.DataLoader:
    """reference :54-78"""
    return data.DataLoader(MazeDataset(filename, split, num_starts=num_starts), batch_size=batch_size,
                           shuffle=shuffle, num_workers=0)


def _percentile_fractions(pcts) -> np.ndarray:
    """The fp64 fractions np.percentile(a, 100 * (1 - pcts)) evaluates for a float32 `a` (it divides by float32(100))."""
    return np.true_divide(100.0 * (1 - np.asarray(pcts, np.float64)), np.float32(100))


_SAMPLER_STATUS = ((1, "distances that are not integers in [-(H*W), 0]"), (2, "no cell above the minimum distance"),
                   (4, "an empty percentile band"),
                   (8, "a policy action that does not lead to a cell one step closer to the goal"),
                   (16, "a goal that is not the only cell at distance 0"))


class DeviceMazeDataset:
    def __init__(self, filename: str, split: str, pct1: float = 0.55, pct2: float = 0.70, pct3: float = 0.85,
                 num_starts: int = 1, device=None):
        """MazeDataset's shortest-path problems, drawn as whole batches on the GPU (csrc/nastar_sampler.cuh).

        Same file, same bands and the same trajectory rule as MazeDataset, but the draws come from a torch.Generator
        on the device, so the starts are not np.random's.  The per-map work (bands, goal, first-max actions) runs once,
        here, in one kernel launch; `sample` then writes a collated batch in one launch, without host synchronisation.
        Raises ValueError naming the maps that cannot be sampled (see `from_labels`)."""
        assert filename.endswith("npz")
        with np.load(filename) as f:
            k = _SPLIT_OFFSET[split]
            maps, goals, policies, dists = (f[f"arr_{k + j}"].astype(np.float32) for j in range(4))
        dev = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
        self._setup(*(torch.from_numpy(x).to(dev) for x in (maps[:, None], goals, policies, dists)),
                    (pct1, pct2, pct3), num_starts)

    @classmethod
    def from_labels(cls, map_designs: torch.Tensor, goal_maps: torch.Tensor, opt_policies: torch.Tensor,
                    opt_dists: torch.Tensor, pct1: float = 0.55, pct2: float = 0.70, pct3: float = 0.85,
                    num_starts: int = 1) -> "DeviceMazeDataset":
        """A dataset over device tensors, e.g. from compute_opt_labels / sample_goal_maps, without a file or a host
        copy of the planes: map_designs [N,H,W] or [N,1,H,W], goal_maps [N,1,H,W], opt_policies [N,8,1,H,W] (or
        [N,4,1,H,W] for the NEWS mechanism), opt_dists [N,1,H,W], on one CUDA device.

        Every map must have integer distances in [-(H*W), 0] with the goal as the only 0, cells above the minimum
        distance, three non-empty bands, and a first-max action that moves every cell that reaches the goal onto the
        grid cell exactly one step closer.  This is stricter than MazeDataset, which only asserts against revisiting a
        cell during a walk; it guarantees that every walk ends at the goal after exactly -opt_dists[start] moves.
        Every compute_opt_labels policy and every shipped planning dataset satisfies it."""
        self = cls.__new__(cls)
        maps = map_designs.detach().float()
        if maps.ndim == 3:
            maps = maps[:, None]
        self._setup(maps, goal_maps.detach().float(), opt_policies.detach().float(), opt_dists.detach().float(),
                    (pct1, pct2, pct3), num_starts)
        return self

    def _setup(self, maps, goals, policies, dists, pcts, num_starts):
        if not maps.is_cuda:
            raise RuntimeError("DeviceMazeDataset runs on CUDA tensors only (there is no CPU fallback)")
        if int(num_starts) <= 0:
            raise ValueError("num_starts must be positive")
        self.map_designs = maps.contiguous()
        self.goal_maps = goals.contiguous()
        self.num_starts = int(num_starts)
        self.pcts = np.array([*pcts, 1.0])
        self.device = maps.device
        if policies.ndim == 5 and policies.shape[1] == 4:
            # NEWS policies: actions 0..3 are the sampler's first four moves (N, E, W, S), so zero planes 4..7 make them
            # the 8-plane policies it reads, with the same first maximal action on every cell
            policies = torch.cat((policies, torch.zeros_like(policies)), 1)
        self._tables = _native.sampler_prepare(dists, policies, self.goal_maps, _percentile_fractions(self.pcts))
        status = self._tables[5].cpu().numpy()
        if status.any():
            bad = [f"{why}: maps {np.flatnonzero(status & bit).tolist()[:20]}"
                   for bit, why in _SAMPLER_STATUS if (status & bit).any()]
            raise ValueError(f"{int((status != 0).sum())} of {len(status)} maps cannot be sampled; " + "; ".join(bad))

    def __len__(self):
        return self.map_designs.shape[0]

    @property
    def thresholds(self) -> torch.Tensor:
        """[N,4] fp64: np.percentile(od[od > od.min()], 100 * (1 - [pct1, pct2, pct3, 1])) per map."""
        return self._tables[4]

    def sample(self, indices, generator: torch.Generator = None, draws: torch.Tensor = None):
        """(map_designs [B,1,H,W], start_maps [B,S,H,W], goal_maps [B,1,H,W], opt_trajs [B,S,H,W]) as fp32 tensors on
        the device, S = num_starts: a collated create_dataloader batch of the maps `indices` (host or device, B
        of them).  Each start picks one of the three bands uniformly, then a candidate of that band uniformly in
        raster order: with u32 draws (d0, d1), band (d0*3) >> 32 and candidate (d1*count) >> 32.  The draws are
        torch.randint on the device with `generator` (a CUDA generator; the default one when None), or the given
        int32 [B,S,2] tensor `draws`.  One kernel launch; host indices are range-checked, device indices must lie in
        [0, len(self)) (a row outside comes back all zero)."""
        idx = torch.as_tensor(indices)
        if idx.device.type == "cpu":
            if idx.numel() and (int(idx.min()) < 0 or int(idx.max()) >= len(self)):
                raise IndexError(f"indices must lie in [0, {len(self)})")
            idx = idx.to(self.device)
        idx = idx.reshape(-1).to(torch.int64).contiguous()
        B, S = idx.numel(), self.num_starts
        if draws is None:
            draws = torch.randint(-2 ** 31, 2 ** 31, (B, S, 2), dtype=torch.int32, device=self.device,
                                  generator=generator)
        elif tuple(draws.shape) != (B, S, 2):
            raise ValueError(f"draws must be [B, num_starts, 2] = {[B, S, 2]}")
        return _native.sampler_sample(self.map_designs, self.goal_maps, self._tables, idx,
                                      draws.to(self.device, torch.int32).contiguous())


class DeviceDataLoader:
    """Batches of a DeviceMazeDataset in DataLoader order: consecutive slices of range(len(dataset)), or of one
    torch.randperm per pass with `shuffle`, the last batch kept partial."""

    def __init__(self, dataset: DeviceMazeDataset, batch_size: int, shuffle: bool = False,
                 generator: torch.Generator = None):
        self.dataset, self.batch_size, self.shuffle, self.generator = dataset, int(batch_size), shuffle, generator

    def __len__(self):
        return -(-len(self.dataset) // self.batch_size)

    def __iter__(self):
        n, dev = len(self.dataset), self.dataset.device
        order = (torch.randperm(n, device=dev, generator=self.generator) if self.shuffle
                 else torch.arange(n, device=dev))
        for i in range(0, n, self.batch_size):
            yield self.dataset.sample(order[i:i + self.batch_size], generator=self.generator)


def create_device_dataloader(filename: str, split: str, batch_size: int, num_starts: int = 1, shuffle: bool = False,
                             generator: torch.Generator = None) -> DeviceDataLoader:
    """create_dataloader's batches drawn on the GPU (DeviceMazeDataset): an iterable of device batches that
    GraphedTrainStep and PlannerModule.fit take as they are."""
    return DeviceDataLoader(DeviceMazeDataset(filename, split, num_starts=num_starts), batch_size, shuffle, generator)


class WarCraftDataset(data.Dataset):
    def __init__(self, dirname: str, split: str):
        """WarCraft terrain maps: `<split>_maps.npy` (uint8 HWC) and `<split>_shortest_paths.npy` (reference :273-295)."""
        maps = np.load(f"{dirname}/{split}_maps.npy")
        self.map_designs = (maps.transpose(0, 3, 1, 2) / 255.0).astype(np.float32)
        self.paths = np.load(f"{dirname}/{split}_shortest_paths.npy").astype(np.float32)

    def __len__(self):
        return self.map_designs.shape[0]

    def __getitem__(self, index: int):
        opt_traj = self.paths[index][np.newaxis]
        start = np.zeros_like(opt_traj)
        start[:, 0, 0] = 1
        goal = np.zeros_like(opt_traj)
        goal[:, -1, -1] = 1
        return self.map_designs[index], start, goal, opt_traj


def create_warcraft_dataloader(dirname: str, split: str, batch_size: int, shuffle: bool = False) -> data.DataLoader:
    """reference :248-270"""
    return data.DataLoader(WarCraftDataset(dirname, split), batch_size=batch_size, shuffle=shuffle, num_workers=0)


def compute_opt_labels(map_designs: torch.Tensor, goal_maps: torch.Tensor, mechanism: str = "moore"):
    """Optimal policies and distances of the planning-datasets generator (get_goalMaps_optPolicies_optDists,
    planning_datasets_utils/data.py:154-159: dijkstra_dist + extract_policy), computed on the GPU in one kernel launch.

    map_designs: CUDA [B,H,W] or [B,1,H,W] (a cell is passable iff its value != 0); goal_maps: CUDA [B,1,H,W] or
    [B,H,W] with one 1 per map (the first maximum is taken).  H, W <= 512.  mechanism: the generator's --mechanism,
    "moore" (8 actions N, E, W, S, NE, NW, SE, SW) or "news" (4 actions N, E, W, S and 4-connected distances).
    Returns, on the maps' device, with A = 8 (moore) or 4 (news):
      opt_policies [B,A,1,H,W] float32 one-hot of the FIRST maximal action per cell (the reference draws one member
                   of the maximal set at random; MazeDataset rolls a policy out with the same first-maximum rule);
      opt_dists    [B,1,H,W] float32: 0 at the goal, -(moves to the goal), -(H*W) where the goal is not reachable;
      act_mask     [B,1,H,W] uint8: bit a set iff action a is maximal (the set the reference draws from)."""
    if not map_designs.is_cuda or not goal_maps.is_cuda:
        raise RuntimeError("compute_opt_labels runs on CUDA tensors only (there is no CPU fallback)")
    maps = map_designs.detach().float()
    if maps.ndim == 4:
        maps = maps[:, 0]
    B, H, W = maps.shape
    goal_idx = goal_maps.detach().reshape(B, H * W).argmax(1).to(torch.int32)
    dists, act_mask, action = _native.opt_labels(maps, goal_idx, mechanism)
    policies = torch.zeros((B, 4 if mechanism == "news" else 8, 1, H, W), dtype=torch.float32, device=maps.device)
    policies.scatter_(1, action.long().view(B, 1, 1, H, W), 1.0)
    return policies, dists, act_mask


def _weighted_inputs(cost_maps: torch.Tensor, goal_maps: torch.Tensor, passable, what: str):
    if not cost_maps.is_cuda or not goal_maps.is_cuda or (passable is not None and not passable.is_cuda):
        raise RuntimeError(f"{what} runs on CUDA tensors only (there is no CPU fallback)")
    cost = cost_maps.detach().float()
    if cost.ndim == 4:
        cost = cost[:, 0]
    B, H, W = cost.shape
    goal_idx = goal_maps.detach().reshape(B, H * W).argmax(1).to(torch.int32)
    pas = None if passable is None else passable.detach().float().reshape(B, H, W)
    return cost, pas, goal_idx


def _raise_on_bad_costs(status: torch.Tensor, what: str) -> None:
    bad = torch.nonzero(status & 1).flatten().tolist()
    if bad:
        raise ValueError(f"{what}: the goal or a passable cell has a negative, NaN or infinite cost in maps {bad}")


def compute_weighted_opt_labels(cost_maps: torch.Tensor, goal_maps: torch.Tensor, passable: torch.Tensor = None,
                                mechanism: str = "moore"):
    """Exact vertex-weighted shortest-path labels of cost maps, computed on the GPU in one kernel launch
    (DESIGN.md §11).  A move (8-connected, no corner check; 4-connected with mechanism="news") leaves a passable cell,
    enters an in-grid cell that is passable or is the goal, and costs the cost of the cell it enters; every sum is the
    fp32 fold from the goal.

    cost_maps: CUDA [B,H,W] or [B,1,H,W], every cost that can be charged finite and >= 0; goal_maps: CUDA [B,1,H,W] or
    [B,H,W] with one 1 per map (the first maximum is taken); passable: CUDA maps of the same shape (a cell is passable
    iff != 0), None = every cell.  H, W <= 128.  mechanism: "moore" (8 actions N, E, W, S, NE, NW, SE, SW) or "news"
    (4 actions N, E, W, S: 4-connected moves, the optimum a 4-connected planner can reach).
    Returns, on the maps' device, with A = 8 (moore) or 4 (news):
      opt_policies [B,A,1,H,W] float32 one-hot of the first optimal action that leads one hop closer to the goal,
                   all zero at the goal and where the goal is unreachable;
      opt_dists    [B,1,H,W] float32: minus the cost-to-go (0 at the goal, -inf where the goal is unreachable);
      act_mask     [B,1,H,W] uint8: bit a set iff action a is optimal and leads one hop closer;
      hops         [B,1,H,W] int32: moves along the policy to the goal, -1 where unreachable.
    Raises ValueError naming the maps with a negative, NaN or infinite cost on the goal or a passable cell (this
    reads the per-map status back to the host)."""
    cost, pas, goal_idx = _weighted_inputs(cost_maps, goal_maps, passable, "compute_weighted_opt_labels")
    B, H, W = cost.shape
    dists, hops, act_mask, action, _, _, status = _native.weighted_labels(cost, goal_idx, pas, mechanism=mechanism)
    _raise_on_bad_costs(status, "compute_weighted_opt_labels")
    A = 4 if mechanism == "news" else 8
    policies = torch.zeros((B, A + 1, 1, H, W), dtype=torch.float32, device=cost.device)
    policies.scatter_(1, (action.long() % (A + 1)).view(B, 1, 1, H, W), 1.0)   # action -1 lands in the dropped slot A
    return policies[:, :A].contiguous(), dists, act_mask, hops


def shortest_path_maps(cost_maps: torch.Tensor, start_maps: torch.Tensor, goal_maps: torch.Tensor,
                       passable: torch.Tensor = None, mechanism: str = "moore"):
    """Minimum-cost paths from the start to the goal of every map, in one kernel launch (the inputs, moves and
    `mechanism` of compute_weighted_opt_labels; start_maps [B,1,H,W] or [B,H,W] with one 1 per map).  Judge a
    planner against the optimum of its own mechanism: a 4-connected path never costs less than the "news" optimum,
    which can be strictly dearer than the "moore" one.

    Returns (path_maps [B,1,H,W] float32: the cells of the path, start and goal included -- the layout of WarCraft's
    shortest_paths and of DifferentiableAstar's paths; path_costs [B] float32: the sum of the costs of every cell of
    the path, as the fp32 fold from the goal).  A start that cannot reach the goal gives an empty mask and +inf; a
    start on the goal gives the goal alone and its cost.  Raises ValueError like compute_weighted_opt_labels."""
    cost, pas, goal_idx = _weighted_inputs(cost_maps, goal_maps, passable, "shortest_path_maps")
    B, H, W = cost.shape
    start_idx = start_maps.detach().reshape(B, H * W).argmax(1).to(torch.int32)
    out = _native.weighted_labels(cost, goal_idx, pas, start_idx, mechanism)
    _raise_on_bad_costs(out[6], "shortest_path_maps")
    return out[4], out[5]


def save_warcraft_dataset(dirname: str, split: str, map_images, shortest_paths) -> None:
    """Write `{split}_maps.npy` and `{split}_shortest_paths.npy` under `dirname`, the files WarCraftDataset /
    create_warcraft_dataloader read.  map_images: uint8 [N,H,W,C] (stored as is) or float [N,C,H,W] in [0, 1] (the
    layout WarCraftDataset returns; stored as round(255 * x) in uint8 [N,H,W,C]); shortest_paths: [N,h,w] or
    [N,1,h,w] masks, e.g. shortest_path_maps' path_maps, stored as float32 [N,h,w]."""
    import os

    imgs, paths = _np(map_images), _np(shortest_paths)
    if imgs.dtype != np.uint8:
        if imgs.ndim != 4:
            raise ValueError(f"map_images: expected [N,C,H,W] floats in [0, 1] or uint8 [N,H,W,C] (got {imgs.shape})")
        imgs = np.rint(np.clip(imgs.transpose(0, 2, 3, 1), 0.0, 1.0) * 255.0).astype(np.uint8)
    if paths.ndim == 4:
        if paths.shape[1] != 1:
            raise ValueError(f"shortest_paths: expected [N,h,w] or [N,1,h,w] (got {paths.shape})")
        paths = paths[:, 0]
    if imgs.ndim != 4 or paths.ndim != 3 or imgs.shape[0] != paths.shape[0]:
        raise ValueError(f"expected N images [N,H,W,C] and N masks [N,h,w] (got {imgs.shape}, {paths.shape})")
    os.makedirs(dirname, exist_ok=True)
    np.save(os.path.join(dirname, f"{split}_maps.npy"), np.ascontiguousarray(imgs))
    np.save(os.path.join(dirname, f"{split}_shortest_paths.npy"), paths.astype(np.float32))


def _largest_component(maze: np.ndarray) -> np.ndarray:
    """Cells of the largest 4-connected passable region; ties go to the region whose first cell comes first in
    raster order (reference data.py:129-132, skimage label(connectivity=1) + np.argmax of the pixel counts).  Any
    non-zero value is passable here, so a non-binary map forms regions by passability, not by equal values."""
    from scipy import ndimage

    lab, _ = ndimage.label(maze != 0)
    counts = np.bincount(lab.ravel())
    counts[0] = 0
    return lab == np.argmax(counts)


def sample_goal_maps(map_designs, edge_size: int = 0, rng=None) -> np.ndarray:
    """Goal maps for new maps, drawn like the planning-datasets generator (reference data.py:127-152).

    For every map, in order: take the cells of its largest 4-connected passable region; with edge_size > 0 keep only
    the cells inside the four edge_size x edge_size corner squares when that leaves any; draw one cell with
    `rng.choice` over them in raster order.  `rng` is a `random.Random` (or the `random` module, as in the
    reference, which seeds it with random.seed); each map makes exactly one `choice` call.  map_designs: [B,H,W] or
    [B,1,H,W] array or tensor.  Returns float32 [B,1,H,W] with one 1 per map."""
    import random as _random

    rng = _random.Random() if rng is None else rng
    maps = map_designs.detach().cpu().numpy() if isinstance(map_designs, torch.Tensor) else np.asarray(map_designs)
    if maps.ndim == 4:
        maps = maps[:, 0]
    B, H, W = maps.shape
    goals = np.zeros((B, 1, H, W), np.float32)
    for i in range(B):
        cond = _largest_component(maps[i])
        if edge_size > 0:
            corner = np.ones_like(cond)
            corner[edge_size:-edge_size, :] = False
            corner[:, edge_size:-edge_size] = False
            if np.any(cond & corner):
                cond = cond & corner
        cells = np.flatnonzero(cond)
        goals[i, 0].reshape(-1)[int(rng.choice(cells))] = 1.0
    return goals


def sample_device_goal_maps(map_designs: torch.Tensor, edge_size: int = 0, generator: torch.Generator = None,
                            draws: torch.Tensor = None) -> torch.Tensor:
    """sample_goal_maps' rule on the GPU, one kernel launch for the whole batch (DESIGN.md §12).

    For every map: the largest 4-connected passable region (a cell is passable iff its value != 0; ties go to the
    region whose first cell comes first in raster order), restricted to the four edge_size x edge_size corner squares
    when that leaves any cell (edge_size = 0: no restriction); then candidate (d * count) >> 32 in raster order, d the
    map's u32 draw.  The draws are torch.randint on the device with `generator` (a CUDA generator; the default one when
    None), or the given int32 [B] tensor `draws`, so the goals are not `random.choice`'s: sample_goal_maps stays the
    path that follows the `random` module.

    map_designs: CUDA [B,H,W] or [B,1,H,W], H, W <= 512.  Returns float32 [B,1,H,W] goal maps with one 1 per map on the
    maps' device, ready for compute_opt_labels, compute_weighted_opt_labels and DeviceMazeDataset.from_labels.  Raises
    ValueError naming the maps without a passable cell (this reads the per-map status back to the host)."""
    if not map_designs.is_cuda:
        raise RuntimeError("sample_device_goal_maps runs on CUDA tensors only (there is no CPU fallback)")
    maps = map_designs.detach().float()
    B = maps.shape[0]
    if draws is None:
        draws = torch.randint(-2 ** 31, 2 ** 31, (B,), dtype=torch.int32, device=maps.device, generator=generator)
    elif tuple(draws.shape) != (B,):
        raise ValueError(f"draws must be [B] = [{B}]")
    _, goal_maps, status = _native.sample_goals(maps, draws.to(maps.device, torch.int32), edge_size)
    bad = torch.nonzero(status & 1).flatten().tolist()
    if bad:
        raise ValueError(f"sample_device_goal_maps: maps {bad[:20]} have no passable cell")
    return goal_maps


def _natural_key(s: str):
    """natsort's default ordering for file names: runs of digits compare as integers."""
    import re

    return [int(p) if p.isdigit() else p for p in re.split(r"(\d+)", s)]


def load_map_images(input_path: str, split: str):
    """Decode the map images `<input_path>/<split>/*.png` on the host, as the planning-datasets generator does
    (load_maze_from_directory): natural-sort order of the paths, `*` allowed in input_path, each image converted to L.

    split: "train", "validation" or "test".  Returns a list of (positions int64 [n], images uint8 [n,H0,W0]) NumPy
    pairs, one per source size: positions are the images' places in the sorted file list.  maps_from_images takes the
    list as it is and returns the maps in file order."""
    import glob
    import os

    from PIL import Image

    if split not in ("train", "validation", "test"):
        raise ValueError(f"split must be train, validation or test (got {split!r})")
    paths = sorted(glob.glob(os.path.join(input_path, split, "*.png")), key=_natural_key)
    if not paths:
        raise FileNotFoundError(f"no PNG images match {os.path.join(input_path, split, '*.png')}")
    groups = {}
    for i, path in enumerate(paths):
        with Image.open(path) as im:
            img = np.asarray(im.convert("L"), dtype=np.uint8)
        groups.setdefault(img.shape, []).append((i, img))
    return [(np.array([i for i, _ in g], np.int64), np.stack([img for _, img in g])) for g in groups.values()]


class PngInfo(tuple):
    """What load_map_pngs needs of one PNG file: (W0, H0, bit_depth, color_type, interlace, idat, plte), idat the
    (offset, length) ranges of the IDAT payloads in the file's bytes, plte the PLTE payload's (offset, length) or
    None."""


_PNG_SIGNATURE = b"\x89PNG\r\n\x1a\n"
# the (bit depth, colour type) pairs of the PNG specification, every one of which Pillow opens
_PNG_MODES = {(1, 0), (2, 0), (4, 0), (8, 0), (16, 0), (8, 2), (16, 2), (1, 3), (2, 3), (4, 3), (8, 3), (8, 4), (16, 4),
              (8, 6), (16, 6)}


def parse_png(data: bytes, name: str = "<bytes>") -> PngInfo:
    """The chunks of a PNG file that its decode needs, checked as Pillow 12.2 checks them when it opens and loads the
    file; anything it refuses, and a file without IHDR or IDAT, raises ValueError naming `name`.

    The signature must match; every chunk before the first IDAT needs a valid type and CRC, and IHDR a known bit depth
    / colour type pair and filter method 0.  The image data is the first run of consecutive IDAT chunks, whose CRCs
    are not checked; later chunks (IEND included, which may be missing) are not read.  Beyond Pillow, a palette image
    without PLTE, an interlace method above 1 and a side of 0 or above 2048 (maps_from_images' source limit) are
    refused too."""
    import re
    import struct
    import zlib

    def bad(why):
        return ValueError(f"{name}: {why}")

    if data[:8] != _PNG_SIGNATURE:
        raise bad("not a PNG file")
    pos, ihdr, plte, idat, n = 8, None, None, [], len(data)
    while True:
        if pos + 8 > n:
            if idat:
                break
            raise bad("truncated PNG file (no IDAT chunk)")
        length, cid = struct.unpack(">I", data[pos:pos + 4])[0], data[pos + 4:pos + 8]
        if idat and cid != b"IDAT":
            break   # the end of the first IDAT run: the decode reads nothing further
        if re.fullmatch(rb"\w\w\w\w", cid) is None:
            raise bad(f"broken PNG file (chunk {cid!r})")
        body = pos + 8
        if body + length > n:
            raise bad(f"truncated {cid.decode('latin-1')} chunk")
        if cid == b"IDAT":
            if ihdr is None:
                raise bad("IDAT before IHDR")
            idat.append((body, length))
            pos = body + length + 4
            continue
        if body + length + 4 > n:
            raise bad(f"incomplete checksum in {cid!r}")
        if zlib.crc32(data[pos + 4:body + length]) & 0xFFFFFFFF != struct.unpack(">I", data[body + length:body + length + 4])[0]:
            raise bad(f"broken PNG file (bad header checksum in {cid!r})")
        if cid == b"IEND":
            raise bad("no IDAT chunk")
        if cid == b"IHDR":
            if length < 13:
                raise bad("truncated IHDR chunk")
            W, H, depth, ct, _, filt, il = struct.unpack(">IIBBBBB", data[body:body + 13])
            if (depth, ct) not in _PNG_MODES:
                raise bad(f"unsupported bit depth {depth} / colour type {ct}")
            if filt:
                raise bad("unknown filter category")
            if il > 1:
                raise bad(f"unknown interlace method {il}")
            if not (1 <= W <= _native.PNG_MAX_SIDE and 1 <= H <= _native.PNG_MAX_SIDE):
                raise bad(f"size {W}x{H} outside 1..{_native.PNG_MAX_SIDE}")
            ihdr = (W, H, depth, ct, il)
        elif cid == b"PLTE" and ihdr is not None and ihdr[3] == 3:
            plte = (body, length)
        pos = body + length + 4
    if ihdr is None:
        raise bad("no IHDR chunk")
    if ihdr[3] == 3 and plte is None:
        raise bad("palette image without PLTE chunk")
    return PngInfo((*ihdr, idat, plte))


def decode_pngs(blobs, names=None, device=None, check: bool = True):
    """PNG files held in memory (a list of bytes) decoded to L by one kernel launch (nastar_b200_decode_png,
    DESIGN.md §16), bit-equal to Pillow's Image.open(f).convert("L").

    The host parses each file (parse_png: one Pillow refuses raises ValueError naming it, before any launch), packs
    descriptors, zlib streams and palettes into one pinned buffer and copies it to `device` (the current CUDA device
    when None) in one transfer.  Returns (groups, status): groups is a list of (positions int64 [n], images CUDA uint8
    [n,H0,W0]) pairs, one per image size in order of first appearance, whose planes are contiguous in one output
    buffer; status is the kernel's int32 [B] NumPy array (include/nastar_b200.h).  Reading it is the call's one host
    synchronisation.  With `check`, a non-zero status raises ValueError naming the files and the reasons."""
    names = [f"<png {i}>" for i in range(len(blobs))] if names is None else list(names)
    infos = [parse_png(b, n) for b, n in zip(blobs, names)]
    groups = {}
    for i, info in enumerate(infos):
        groups.setdefault((info[1], info[0]), []).append(i)
    B = len(blobs)
    desc = np.zeros(B, _native.PNG_DESC_DTYPE)
    head = desc.nbytes
    total = head + sum(sum(n for _, n in info[5]) + (info[6][1] if info[6] else 0) for info in infos)
    dev = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
    buf = torch.empty((total,), dtype=torch.uint8).pin_memory()
    host = buf.numpy()
    pos, out_pos = head, 0
    for (H0, W0), members in groups.items():
        for i in members:
            W, H, depth, ct, il, idat, plte = infos[i]
            blob = np.frombuffer(blobs[i], np.uint8)
            d = desc[i]
            d["in_off"], d["out_off"] = pos, out_pos
            for off, n in idat:
                host[pos:pos + n] = blob[off:off + n]
                pos += n
            d["in_len"] = pos - d["in_off"]
            if plte:
                d["plte_off"], d["plte_len"] = pos, plte[1]
                host[pos:pos + plte[1]] = blob[plte[0]:plte[0] + plte[1]]
                pos += plte[1]
            d["W0"], d["H0"], d["bit_depth"], d["color_type"], d["interlace"] = W, H, depth, ct, il
            out_pos += H0 * W0
    host[:head] = desc.view(np.uint8)
    with torch.cuda.device(dev):
        data = buf.to(dev, non_blocking=True)
        out, status = _native.decode_png(data, desc, data[:head], out_pos)
        status = status.cpu().numpy()
    if check and status.any():
        bad = [f"{names[i]}: " + ", ".join(why for bit, why in _native.PNG_STATUS.items() if status[i] & bit)
               for i in np.flatnonzero(status)]
        raise ValueError("corrupt PNG data in " + "; ".join(bad[:20]))
    result, base = [], 0
    for (H0, W0), members in groups.items():
        n = len(members)
        result.append((np.array(members, np.int64), out[base:base + n * H0 * W0].view(n, H0, W0)))
        base += n * H0 * W0
    return result, status


def load_map_pngs(input_path: str, split: str, device=None):
    """load_map_images on the GPU: the same files (`<input_path>/<split>/*.png`, natural-sort order, `*` allowed) and
    the same result, a list of (positions int64 [n], images) pairs, one per source size, but with the images decoded
    by one kernel launch (decode_pngs) into CUDA uint8 [n,H0,W0] tensors on `device`, bit-equal to Pillow's
    Image.open(f).convert("L").  maps_from_images takes the list as it is.

    A file Pillow refuses, or one without IHDR or IDAT, raises ValueError naming it before any launch; a stream the
    kernel finds corrupt raises ValueError naming the files and the reasons."""
    import glob
    import os

    if split not in ("train", "validation", "test"):
        raise ValueError(f"split must be train, validation or test (got {split!r})")
    paths = sorted(glob.glob(os.path.join(input_path, split, "*.png")), key=_natural_key)
    if not paths:
        raise FileNotFoundError(f"no PNG images match {os.path.join(input_path, split, '*.png')}")
    blobs = []
    for path in paths:
        with open(path, "rb") as fh:
            blobs.append(fh.read())
    return decode_pngs(blobs, paths, device)[0]


def maps_from_images(images, size, device=None) -> torch.Tensor:
    """Planning maps from decoded map images on the GPU, as the planning-datasets generator makes them
    (load_maze_from_directory, DESIGN.md §13): Pillow's bicubic Image.resize to H x W, skimage's threshold_otsu of the
    resized levels, 1.0 where level > threshold, else 0.0.  Bit-equal to the generator; a uniform resized image gives
    an all-zero map, as there.

    images: CUDA uint8 [B,H0,W0] (one kernel launch), or the list load_map_images or load_map_pngs returns (one launch
    per source size, moved to `device`, the current CUDA device when None; a group's images may be a NumPy array or a
    CUDA tensor).  H0, W0 <= 2048.  size: int or (H, W), H, W <= 512.
    Returns float32 [B,1,H,W] on the device, in the images' order, ready for sample_device_goal_maps."""
    H, W = (int(size), int(size)) if np.ndim(size) == 0 else (int(size[0]), int(size[1]))
    if isinstance(images, torch.Tensor):
        if not images.is_cuda:
            raise RuntimeError("maps_from_images runs on CUDA tensors only (there is no CPU fallback)")
        return _native.maps_from_images(images, H, W)[0]
    dev = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
    n = sum(len(pos) for pos, _ in images)
    out = torch.empty((n, 1, H, W), dtype=torch.float32, device=dev)
    for pos, imgs in images:
        if isinstance(imgs, torch.Tensor):
            if not imgs.is_cuda:
                raise RuntimeError("maps_from_images: a group's images are a NumPy array or a CUDA tensor")
            x = imgs.to(dev)
        else:
            x = torch.from_numpy(imgs).to(dev)
        out[torch.from_numpy(pos).to(dev)] = _native.maps_from_images(x, H, W)[0]
    return out


def tile_maps(maps: torch.Tensor, tile_size: int, indices=None, generator: torch.Generator = None,
              num: int = None) -> torch.Tensor:
    """Tiled maps, skimage.util.montage of tile_size**2 maps each, as the planning-datasets generator lays them out
    with --tile-size (Tiled MP): map k of a tile goes to grid cell (k // tile_size, k % tile_size).

    maps: [N,h,w] or [N,1,h,w]; indices: [M, tile_size**2] map indices (a tensor or array), or None to draw `num`
    tiles (N when None) uniformly with torch.randint on the maps' device with `generator`.  The generator's own tiles
    come from np.random.choice: pass those indices to replay them.  Returns [M,1,t*h,t*w] in the maps' dtype."""
    t = int(tile_size)
    m = maps[:, 0] if maps.ndim == 4 else maps
    N, h, w = m.shape
    if indices is None:
        idx = torch.randint(0, N, (N if num is None else int(num), t * t), device=m.device, generator=generator)
    else:
        idx = torch.as_tensor(np.asarray(indices) if not isinstance(indices, torch.Tensor) else indices)
        if idx.ndim != 2 or idx.shape[1] != t * t:
            raise ValueError(f"indices must be [M, tile_size**2] = [M, {t * t}] (got {tuple(idx.shape)})")
        if idx.numel() and (int(idx.min()) < 0 or int(idx.max()) >= N):
            raise IndexError(f"indices must lie in [0, {N})")
        idx = idx.to(m.device, torch.int64)
    M = idx.shape[0]
    return m[idx].reshape(M, t, t, h, w).permute(0, 1, 3, 2, 4).reshape(M, 1, t * h, t * w)


def draw_opt_policies(act_mask: torch.Tensor, generator: torch.Generator = None,
                      draws: torch.Tensor = None, num_actions: int = 8) -> torch.Tensor:
    """One-hot optimal policies with the planning-datasets generator's rule (extract_policy): every cell takes one
    member of its maximal action set uniformly, instead of compute_opt_labels' first maximum.  One kernel launch.

    act_mask: CUDA uint8 [B,1,H,W] from compute_opt_labels (bit a set iff action a is maximal).  Cell c takes set bit
    (d * popc) >> 32 in action order, d its u32 draw: torch.randint on the device with `generator` (a CUDA generator;
    the default one when None), or the given int32 [B,1,H,W] / [B,H,W] tensor `draws`.  Returns float32
    [B,num_actions,1,H,W] (a cell with an empty mask gets an all-zero column).  num_actions = 4 is for the masks of
    compute_opt_labels(..., mechanism="news"), which never set bits 4..7: the draw then lies in planes 0..3."""
    if not act_mask.is_cuda:
        raise RuntimeError("draw_opt_policies runs on CUDA tensors only (there is no CPU fallback)")
    if num_actions not in (4, 8):
        raise ValueError(f"num_actions must be 4 (news) or 8 (moore) (got {num_actions})")
    mask = act_mask[:, 0] if act_mask.ndim == 4 else act_mask
    if draws is None:
        draws = torch.randint(-2 ** 31, 2 ** 31, tuple(mask.shape), dtype=torch.int32, device=mask.device,
                              generator=generator)
    elif draws.numel() != mask.numel():
        raise ValueError(f"draws must have one entry per cell, {list(mask.shape)}")
    policies = _native.draw_policies(mask, draws.to(mask.device, torch.int32))
    return policies if num_actions == 8 else policies[:, :num_actions].contiguous()


def _np(x) -> np.ndarray:
    return x.detach().cpu().numpy() if isinstance(x, torch.Tensor) else np.asarray(x)


_ZIP_DOS_DATE = (0 << 9) | (1 << 5) | 1   # 1980-01-01 00:00:00: archives do not depend on the write time
_U32 = 0xFFFFFFFF


@functools.lru_cache(maxsize=None)
def _npy_header(dtype: np.dtype, shape) -> bytes:
    """The header np.save writes for a C-order array of this dtype and shape (format 1.0, or 2.0 when it must)."""
    import io

    d = {"descr": np.lib.format.dtype_to_descr(dtype), "fortran_order": False, "shape": tuple(int(s) for s in shape)}
    buf = io.BytesIO()
    try:
        np.lib.format.write_array_header_1_0(buf, d)
    except ValueError:
        buf = io.BytesIO()
        np.lib.format.write_array_header_2_0(buf, d)
    return buf.getvalue()


def _zip_local_header_bytes(name: bytes) -> int:
    return 30 + len(name) + 20


def _zip_finish(image, names, offs, csizes, usizes, crcs, force_zip64: bool = False) -> bytes:
    """Write each member's local header (ZIP64 extra with both sizes, as np.savez writes them) into `image` just
    before its stream at offs[i], and return the central directory, ZIP64 end records where needed, and the end
    record, which follow image's bytes in the file.  Timestamps are fixed; members are stored with method 8."""
    import struct

    cd = []
    for name, off, cs, us, crc in zip(names, offs, csizes, usizes, crcs):
        lh = off - _zip_local_header_bytes(name)
        image[lh:off] = np.frombuffer(
            struct.pack("<IHHHHHIIIHH", 0x04034B50, 45, 0, 8, 0, _ZIP_DOS_DATE, crc, _U32, _U32, len(name), 20) + name
            + struct.pack("<HHQQ", 1, 16, us, cs), np.uint8)
        ext = [v for v in (us, cs, lh) if force_zip64 or v >= _U32]
        extra = struct.pack("<HH", 1, 8 * len(ext)) + struct.pack(f"<{len(ext)}Q", *ext) if ext else b""
        big = force_zip64 or us >= _U32, force_zip64 or cs >= _U32, force_zip64 or lh >= _U32
        cd.append(struct.pack("<IHHHHHHIIIHHHHHII", 0x02014B50, 45 | (3 << 8), 45, 0, 8, 0, _ZIP_DOS_DATE, crc,
                              _U32 if big[1] else cs, _U32 if big[0] else us, len(name), len(extra), 0, 0, 0,
                              0o600 << 16, _U32 if big[2] else lh) + name + extra)
    cd = b"".join(cd)
    cd_off, n = len(image), len(names)
    tail = b""
    if force_zip64 or n > 0xFFFF or cd_off >= _U32 or len(cd) >= _U32:
        z64 = cd_off + len(cd)
        tail = (struct.pack("<IQHHIIQQQQ", 0x06064B50, 44, 45, 45, 0, 0, n, n, len(cd), cd_off)
                + struct.pack("<IIQI", 0x07064B50, 0, z64, 1))
        eocd = struct.pack("<IHHHHIIH", 0x06054B50, 0, 0, 0xFFFF, 0xFFFF, _U32, _U32, 0)
    else:
        eocd = struct.pack("<IHHHHIIH", 0x06054B50, 0, 0, n, n, len(cd), cd_off, 0)
    return cd + tail + eocd


def savez_compressed_device(file, *args, **kwds) -> None:
    """np.savez_compressed for CUDA tensors: members arr_0.npy, ... for positional arrays and <name>.npy for keywords,
    each inflating to the bytes np.save writes for tensor.cpu().numpy().  The members are deflated on the device in one
    kernel launch (include/nastar_b200.h, nastar_b200_deflate; DESIGN.md §18) with the CRC-32 of their raw bytes;
    only the compressed bytes are copied to the host, and the archive (fixed timestamps, ZIP64 where needed) is
    written at once.  `file`: a path (".npz" is appended when missing, as numpy does) or a writable binary file.
    Non-CUDA arguments raise RuntimeError: there is no CPU fallback."""
    members = {}
    for i, a in enumerate(args):
        members[f"arr_{i}"] = a
    for k, a in kwds.items():
        if k in members:
            raise ValueError(f"Cannot use un-named variables and keyword {k}")
        members[k] = a
    if not members:
        raise ValueError("savez_compressed_device: nothing to save")
    _savez_compressed_many([(file, members)])


_NP_DTYPE = {}


def _np_dtype(dtype: torch.dtype) -> np.dtype:
    if dtype not in _NP_DTYPE:
        _NP_DTYPE[dtype] = torch.empty(0, dtype=dtype).numpy().dtype
    return _NP_DTYPE[dtype]


def _savez_compressed_many(files) -> None:
    """savez_compressed_device for many archives at once: files is a list of (file, members), members a dict of
    member name (without ".npy") -> CUDA tensor, every tensor of every file on one device.  All members of all files
    are deflated in one nastar_b200_deflate launch, and the host waits twice in all, once for the compressed sizes and
    CRCs and once for exactly the compressed bytes; each archive is then finished (_zip_finish) and written.  `file`:
    a path (".npz" is appended when missing) or a writable binary file."""
    names, tensors, first = [], [], [0]
    for _, members in files:
        if not members:
            raise ValueError("savez_compressed_device: nothing to save")
        names += [(k + ".npy").encode() for k in members]
        tensors += list(members.values())
        first.append(len(tensors))
    if not all(isinstance(t, torch.Tensor) and t.is_cuda for t in tensors):
        raise RuntimeError("savez_compressed_device: every array must be a CUDA tensor (there is no CPU fallback)")
    dev = tensors[0].device
    if any(t.device != dev for t in tensors):
        raise ValueError("savez_compressed_device: every tensor must be on one device")
    flat = [t.detach().contiguous().reshape(-1) for t in tensors]
    heads = [_npy_header(_np_dtype(t.dtype), tuple(t.shape)) for t in tensors]
    data = [f.view(torch.uint8) if f.numel() else f for f in flat]
    M = len(tensors)
    desc = np.zeros(M, _native.DEFLATE_DESC_DTYPE)
    hlen = np.array([len(h) for h in heads], np.int64)
    dlen = np.array([f.numel() * f.element_size() for f in flat], np.int64)
    hoff = np.concatenate([[0], np.cumsum(hlen)])
    ctl = torch.empty((int(hoff[-1]) + desc.nbytes,), dtype=torch.uint8, pin_memory=True)
    ctl_dev = torch.empty((ctl.numel(),), dtype=torch.uint8, device=dev)
    gaps = np.array([_zip_local_header_bytes(n) for n in names], np.int64)
    desc["head"] = ctl_dev.data_ptr() + hoff[:-1]
    desc["head_len"] = hlen
    desc["data"] = [d.data_ptr() if n else 0 for d, n in zip(data, dlen)]
    desc["data_len"] = dlen
    desc["gap"] = gaps
    desc["chunk0"] = np.concatenate([[0], np.cumsum(_native.deflate_chunk_counts(dlen))[:-1]])
    c = ctl.numpy()
    c[:hoff[-1]] = np.frombuffer(b"".join(heads), np.uint8)
    c[hoff[-1]:] = desc.view(np.uint8)
    with torch.cuda.device(dev):
        ctl_dev.copy_(ctl, non_blocking=True)
        out, out_off, out_len, crc = _native.deflate(desc, ctl_dev[int(hoff[-1]):])
        meta = torch.cat([out_off, out_len, crc.to(torch.int64) & _U32]).to("cpu", non_blocking=True)
        torch.cuda.current_stream(dev).synchronize()   # the compressed sizes and CRCs
        meta = meta.numpy().reshape(3, M)
        offs, csizes, crcs = meta[0].tolist(), meta[1].tolist(), meta[2].tolist()
        end = offs[-1] + csizes[-1]
        image = torch.empty((end,), dtype=torch.uint8, pin_memory=True)
        image.copy_(out[:end], non_blocking=True)
        torch.cuda.current_stream(dev).synchronize()   # exactly the compressed bytes, known only after the first wait
    del flat, data, ctl
    img = image.numpy()
    usizes = (hlen + dlen).tolist()
    for f, (file, _) in enumerate(files):
        a, b = first[f], first[f + 1]
        start = offs[a] - int(gaps[a])   # the archive's first local header; the archives lie back to back
        part = img[start:offs[b - 1] + csizes[b - 1]]
        tail = _zip_finish(part, names[a:b], [o - start for o in offs[a:b]], csizes[a:b], usizes[a:b], crcs[a:b])
        if isinstance(file, (str, os.PathLike)):
            file = os.fspath(file)
            if not file.endswith(".npz"):
                file += ".npz"
            with open(file, "wb") as fh:
                fh.write(memoryview(part))
                fh.write(tail)
        else:
            file.write(memoryview(part))
            file.write(tail)


def save_planning_dataset(path: str, train, valid, test) -> None:
    """Write a planning-datasets .npz (np.savez_compressed arr_0..arr_11, reference generate_spp_instances.py:48-62)
    that MazeDataset / create_dataloader read.  Each split is (maps [N,H,W] or [N,1,H,W], goal_maps [N,1,H,W],
    opt_policies [N,8,1,H,W] (moore) or [N,4,1,H,W] (news), opt_dists [N,1,H,W]), NumPy arrays or tensors; they are
    stored in the dtype given.  When all 12 arrays are CUDA tensors on one device, the file is compressed there
    (savez_compressed_device); otherwise np.savez_compressed writes it.  np.load reads the same arrays either way."""
    splits = [tuple(split) for split in (train, valid, test)]
    flat = [x for split in splits for x in split]
    device = all(isinstance(x, torch.Tensor) and x.is_cuda for x in flat) and len({x.device for x in flat}) == 1
    arrays = []
    for name, split in zip(("train", "valid", "test"), splits):
        maps, goals, policies, dists = (x.detach() if device else _np(x) for x in split)
        if maps.ndim == 4:
            maps = maps[:, 0]
        N, H, W = maps.shape
        if (goals.shape != (N, 1, H, W) or policies.shape not in ((N, 8, 1, H, W), (N, 4, 1, H, W))
                or dists.shape != (N, 1, H, W)):
            raise ValueError(f"{name}: expected maps [N,H,W], goals / dists [N,1,H,W], policies [N,8|4,1,H,W] "
                             f"(got {maps.shape}, {goals.shape}, {policies.shape}, {dists.shape})")
        arrays += [maps, goals, policies, dists]
    if device:
        savez_compressed_device(path, *arrays)
    else:
        np.savez_compressed(path, *arrays)


def encode_pngs(images) -> list:
    """PNG files of 8-bit grey images, encoded on the GPU (DESIGN.md §21): colour type 0, not interlaced, one IDAT
    chunk each.  Every scanline takes the filter type 0..4 with the least sum of |byte as int8| (libpng's heuristic,
    ties to the lowest type), the filtered streams are deflated by nastar_b200_deflate and each file's chunks, CRCs and
    Adler-32 are written around its stream on the device: three kernel launches in all.  The host waits twice, once
    for the files' offsets and once for exactly their bytes.

    images: a CUDA uint8 tensor [B,H,W], or a list of CUDA uint8 [H,W] tensors of any sizes on one device; sides
    1 .. 2048.  Returns one `bytes` per image, in order.  Non-CUDA images raise RuntimeError: there is no CPU
    fallback."""
    if isinstance(images, torch.Tensor):
        if not images.is_cuda:
            raise RuntimeError("encode_pngs runs on CUDA tensors only (there is no CPU fallback)")
        if images.ndim != 3:
            raise ValueError(f"encode_pngs: images are [B,H,W] (got {tuple(images.shape)})")
        planes = list(images.detach().contiguous().unbind(0))
    else:
        planes = list(images)
    if not planes:
        return []
    if not all(isinstance(p, torch.Tensor) and p.is_cuda for p in planes):
        raise RuntimeError("encode_pngs runs on CUDA tensors only (there is no CPU fallback)")
    dev = planes[0].device
    for p in planes:
        if p.dtype != torch.uint8:
            raise TypeError(f"encode_pngs: images are uint8 grey levels (got {p.dtype})")
        if p.ndim != 2 or not (1 <= p.shape[0] <= _native.PNG_MAX_SIDE and 1 <= p.shape[1] <= _native.PNG_MAX_SIDE):
            raise ValueError(f"encode_pngs: images are [H,W] with sides 1..{_native.PNG_MAX_SIDE} "
                             f"(got {tuple(p.shape)})")
        if p.device != dev:
            raise ValueError("encode_pngs: every image must be on one device")
    planes = [p.detach().contiguous() for p in planes]
    B = len(planes)
    H = np.array([p.shape[0] for p in planes], np.int64)
    W = np.array([p.shape[1] for p in planes], np.int64)
    n = H * (W + 1)
    foff = np.concatenate([[0], np.cumsum(n)[:-1]])
    enc = np.zeros(B, _native.PNG_ENC_DESC_DTYPE)
    enc["pixels"] = [p.data_ptr() for p in planes]
    enc["filt_off"], enc["W"], enc["H"] = foff, W, H
    filt = torch.empty((int(n.sum()),), dtype=torch.uint8, device=dev)
    desc = np.zeros(B, _native.DEFLATE_DESC_DTYPE)
    desc["data"] = filt.data_ptr() + foff
    desc["data_len"] = n
    desc["gap"] = _native.png_gaps(B)
    desc["chunk0"] = np.concatenate([[0], np.cumsum(_native.deflate_chunk_counts(n))[:-1]])
    ctl = torch.empty((enc.nbytes + desc.nbytes,), dtype=torch.uint8, pin_memory=True)
    c = ctl.numpy()
    c[:enc.nbytes] = enc.view(np.uint8)
    c[enc.nbytes:] = desc.view(np.uint8)
    with torch.cuda.device(dev):
        ctl_dev = torch.empty((ctl.numel(),), dtype=torch.uint8, device=dev)
        ctl_dev.copy_(ctl, non_blocking=True)
        enc_dev = ctl_dev[:enc.nbytes]
        adler = _native.png_filter(enc, enc_dev, filt)
        out, out_off, out_len, _ = _native.deflate(desc, ctl_dev[enc.nbytes:], tail=_native.PNG_ENC_TAIL)
        _native.png_finish(enc, enc_dev, out_off, out_len, adler, out)
        meta = torch.cat([out_off, out_len]).to("cpu", non_blocking=True)
        torch.cuda.current_stream(dev).synchronize()   # the files' offsets
        meta = meta.numpy().reshape(2, B)
        starts = meta[0] - _native.PNG_ENC_HEAD
        ends = meta[0] + meta[1] + _native.PNG_ENC_TAIL
        image = torch.empty((int(ends[-1]),), dtype=torch.uint8, pin_memory=True)
        image.copy_(out[:int(ends[-1])], non_blocking=True)
        torch.cuda.current_stream(dev).synchronize()   # exactly the files' bytes, known only after the first wait
    del planes, filt, ctl
    img = image.numpy()
    return [img[a:b].tobytes() for a, b in zip(starts.tolist(), ends.tolist())]


def save_pngs(paths, images) -> None:
    """Write image i of `images` (what encode_pngs takes) as a PNG file to paths[i], every file encoded on the GPU in
    one encode_pngs call."""
    paths = list(paths)
    n = images.shape[0] if isinstance(images, torch.Tensor) and images.ndim == 3 else len(images)
    if len(paths) != n:
        raise ValueError(f"save_pngs: {len(paths)} paths for {n} images")
    for path, blob in zip(paths, encode_pngs(images)):
        with open(path, "wb") as f:
            f.write(blob)


STREET_SPLITS = ("train", "validation", "test")


def street_crop_boxes(train_files, test_files, size: int = 128, counts=(160, 20, 40), seed: int = 1372,
                      source_size: int = 256):
    """The crop boxes of the CSM street maps (planning-datasets' preprocess_street_dataset.py, crop_images), replayed
    on the host: np.random.RandomState(seed) draws randint(0, source_size - size, [count, 2]) per file, first for
    every train file (counts[0] each), then for the same train files again (validation, counts[1] each), then for every
    test file (counts[2] each).  A draw's row (left, top) is the box (left, top, left + size, top + size) of the
    source resized to source_size x source_size, saved as "<fileid>_<n:05d>.png" with fileid the file name before
    "_256.png".

    train_files, test_files: the sources in the order the draws take them (the generator takes glob order).  Returns
    {split: dict(source int64 [N] (index into that split's file list), n, left, top int64 [N], name list of str)}."""
    import re

    rng = np.random.RandomState(seed)
    result = {}
    for split, files, count in zip(STREET_SPLITS, (train_files, train_files, test_files), counts):
        src, n, lt, names = [], [], [], []
        for k, f in enumerate(files):
            fileid = re.split("_256.png", re.split("/", os.fspath(f))[-1])[0]
            draw = rng.randint(0, source_size - size, [int(count), 2])
            src += [k] * int(count)
            n += list(range(int(count)))
            lt.append(draw)
            names += ["%s_%05d.png" % (fileid, i) for i in range(int(count))]
        lt = np.concatenate(lt).astype(np.int64) if lt else np.zeros((0, 2), np.int64)
        result[split] = dict(source=np.array(src, np.int64), n=np.array(n, np.int64), left=lt[:, 0], top=lt[:, 1],
                             name=names)
    return result


SDD_LABELS = {"Pedestrian": 0, "Biker": 1, "Skater": 2, "Car": 3, "Cart": 4, "Bus": 5}


def read_sdd_annotations(path: str):
    """A Stanford Drone `annotations.txt`: space-separated rows `id xmin ymin xmax ymax frame lost occluded generated
    "label"` (the label quoted).  Returns (int64 [n, 9] of the first nine columns, list of the n labels without their
    quotes)."""
    with open(path, "rb") as f:
        text = f.read()
    tok = text.split()
    if len(tok) != 10 * sum(1 for ln in text.splitlines() if ln.strip()):
        raise ValueError(f"{path}: every annotation row has 10 space-separated columns")
    tok = np.array(tok).reshape(-1, 10)
    names, which = np.unique(tok[:, 9], return_inverse=True)
    names = np.array([n.decode().strip('"') for n in names] or [""])
    return tok[:, :9].astype(np.int64), list(names[which.reshape(-1)])


def sdd_sample_plan(video_dir: str, W: int = 64, min_len_ratio: float = 0.5, min_max_size: int = 128,
                    max_step: int = 600, rng=None) -> dict:
    """The samples planning-datasets' SDD.py (create_sample_from_dataset) makes of one Stanford Drone video directory
    (`reference.jpg` and `annotations.txt`), planned on the host without decoding the scene (DESIGN.md §22).

    Ids are visited in order of first appearance; each id's visible segments are its maximal runs of rows with
    lost == 0, numbered 1, 2, ...  A segment longer than max_step takes a window of max_step rows starting at
    rng.randint(0, len - max_step), drawn before the segment is judged, so rejected segments draw too.  The segment is
    kept when its start-to-goal length is > 0, its length ratio > min_len_ratio and its larger extent > min_max_size;
    the ROI, the resized trajectory and the ratio are the reference's float64 expressions, evaluated with the same
    NumPy calls.  rng: a np.random.RandomState shared across videos (None: NumPy's global state, as the reference).

    Returns dict(scene, video (the directory's last two components), name list of "%08d_%02d.npz", box int64 [K, 4]
    (Image.crop's box after Python's round, half to even), traj list of float64 [n, 2] (traj_resized), label int64
    [K], length_ratio float64 [K], start, goal int64 [K, 2] (row, column), cells list of int64 [m, 2] (row, column)
    of the trajectory image's set cells)."""
    from PIL import Image

    rng = np.random if rng is None else rng
    parts = os.path.normpath(os.fspath(video_dir)).split(os.sep)
    with Image.open(os.path.join(video_dir, "reference.jpg")) as im:
        size = im.size
    cols, labels = read_sdd_annotations(os.path.join(video_dir, "annotations.txt"))
    ids = cols[:, 0]
    uniq, first = np.unique(ids, return_index=True)
    perm = np.argsort(ids, kind="stable")   # each id's rows, in file order
    bounds = np.searchsorted(ids[perm], uniq)
    rows_of = {int(u): perm[b:e] for u, b, e in zip(uniq, bounds, np.append(bounds[1:], len(ids)))}
    plan = dict(scene=parts[-2], video=parts[-1], name=[], box=[], traj=[], label=[], length_ratio=[], start=[],
                goal=[], cells=[])
    for id_ in uniq[np.argsort(first)]:
        rows = rows_of[int(id_)]
        sample = cols[rows]
        visible = sample[:, 6] == 0
        starts = np.flatnonzero(visible & ~np.concatenate([[False], visible[:-1]]))
        ends = np.flatnonzero(visible & ~np.concatenate([visible[1:], [False]])) + 1
        for vl, (a, b) in enumerate(zip(starts, ends), 1):
            seg = sample[a:b]
            traj = (seg[:, 1:3] + seg[:, 3:5]) / 2.
            if len(traj) > max_step:
                s0 = rng.randint(0, len(traj) - max_step)
                traj = traj[s0:s0 + max_step, :]
            max_size = np.max(traj.max(axis=0) - traj.min(axis=0), 0)
            mean_loc = traj.min(axis=0) + (traj.max(axis=0) - traj.min(axis=0)) / 2
            if np.all(mean_loc - max_size / 2 - 50 > 0):
                min_loc = np.maximum(mean_loc - max_size / 2 - 50, 0)
                max_loc = min_loc + max_size + 100
            else:
                max_loc = np.minimum(mean_loc + max_size / 2 + 50, size)
                min_loc = max_loc - max_size - 100
            all_length = np.abs(np.diff(traj, axis=0)).sum()
            sg_length = np.abs(np.diff(traj[[0, -1]], axis=0)).sum()
            length_ratio = sg_length / (all_length + 1e-5)
            if not ((sg_length > 0) & (length_ratio > min_len_ratio) & (max_size > min_max_size)):
                continue
            label = labels[rows[0]]
            if label not in SDD_LABELS:
                raise ValueError(f"{video_dir}: unknown label {label!r} (id {int(id_)})")
            tr = (traj - min_loc) / (max_size + 100) * W
            tr[tr > W - 1] = W - 1
            tr[tr < 0] = 0
            dense = np.arange(len(tr) * 5)
            knots = np.arange(0, 5 * len(tr), 5)
            t0, t1 = np.interp(dense, knots, tr[:, 0]), np.interp(dense, knots, tr[:, 1])
            # np.histogram2d(t1, t0, range(W + 1)) puts v in [0, W - 1] in bin floor(v)
            cell = np.unique(np.floor(t1).astype(np.int64) * W + np.floor(t0).astype(np.int64))
            plan["name"].append("%08d_%02d.npz" % (id_, vl))
            plan["box"].append([round(float(v)) for v in (min_loc[0], min_loc[1], max_loc[0], max_loc[1])])
            plan["traj"].append(tr)
            plan["label"].append(SDD_LABELS[label])
            plan["length_ratio"].append(length_ratio)
            plan["start"].append([int(tr[0, 1]), int(tr[0, 0])])
            plan["goal"].append([int(tr[-1, 1]), int(tr[-1, 0])])
            plan["cells"].append(np.stack([cell // W, cell % W], axis=1))
    plan["box"] = np.array(plan["box"], np.int64).reshape(-1, 4)
    plan["label"] = np.array(plan["label"], np.int64)
    plan["length_ratio"] = np.array(plan["length_ratio"], np.float64)
    plan["start"] = np.array(plan["start"], np.int64).reshape(-1, 2)
    plan["goal"] = np.array(plan["goal"], np.int64).reshape(-1, 2)
    return plan


def sdd_crops(scenes, boxes, size, src=None) -> torch.Tensor:
    """RGB crops of scenes resized on the GPU, bit-equal to Pillow's np.array(scene.crop(box).resize(size)) (BICUBIC)
    for an RGB scene: one kernel launch for all crops (include/nastar_b200.h, nastar_b200_crop_resize_rgb).

    scenes: a CUDA uint8 [H,W,3] tensor or a list of them on one device (sides <= 4096); boxes: int [N, 4]
    (left, top, right, bottom) in pixels, non-empty, sides <= 4096, past any edge allowed (those pixels are 0);
    size: int or Pillow's (width, height), each <= 1024; src: [N] scene index of each box (None: all 0).  Returns
    uint8 [N, height, width, 3] on the scenes' device."""
    scenes = [scenes] if isinstance(scenes, torch.Tensor) else list(scenes)
    Wo, Ho = (int(size), int(size)) if np.ndim(size) == 0 else (int(size[0]), int(size[1]))
    boxes = np.asarray(boxes, np.int64).reshape(-1, 4)
    src = np.zeros(len(boxes), np.int64) if src is None else np.asarray(src, np.int64).reshape(-1)
    return _native.crop_resize_rgb(scenes, src, boxes, Ho, Wo)


def _sdd_scene(video_dir: str, device) -> torch.Tensor:
    """reference.jpg decoded by Pillow on the host and uploaded, uint8 [H, W, 3]."""
    from PIL import Image

    path = os.path.join(video_dir, "reference.jpg")
    with Image.open(path) as im:
        if im.mode != "RGB":
            raise ValueError(f"{path}: the scene decodes to mode {im.mode!r}, not RGB")
        pixels = np.array(im)
    return torch.from_numpy(pixels).to(device)


def _write_sdd_samples(batch, W: int, device) -> None:
    """One batch of (plan, scene, directory) of save_sdd_samples: one crop launch, planes built on the device, one
    deflate launch for all files."""
    plans = [p for p, _, _ in batch]
    K = sum(len(p["name"]) for p in plans)
    if K == 0:
        return
    scenes = [s for _, s, _ in batch]
    src = np.concatenate([np.full(len(p["name"]), i, np.int64) for i, p in enumerate(plans)])
    images = sdd_crops(scenes, np.concatenate([p["box"] for p in plans]), W, src)
    # start_image, goal_image and traj_image of every sample: 1.0 at the plan's cells
    k_traj = np.concatenate([np.full(len(c), k, np.int64) for k, c in
                             enumerate(c for p in plans for c in p["cells"])])
    cells = np.concatenate([c for p in plans for c in p["cells"]])
    start = np.concatenate([p["start"] for p in plans])
    goal = np.concatenate([p["goal"] for p in plans])
    k = np.arange(K)
    idx = np.concatenate([np.stack([np.zeros(K, np.int64), k, start[:, 0], start[:, 1]]),
                          np.stack([np.ones(K, np.int64), k, goal[:, 0], goal[:, 1]]),
                          np.stack([np.full(len(cells), 2, np.int64), k_traj, cells[:, 0], cells[:, 1]])], axis=1)
    trajs = [t for p in plans for t in p["traj"]]
    toff = np.concatenate([[0], np.cumsum([len(t) for t in trajs])])
    host = np.concatenate([idx.reshape(-1).view(np.float64), np.concatenate(trajs).reshape(-1),
                           np.concatenate([p["label"] for p in plans]).view(np.float64),
                           np.concatenate([p["length_ratio"] for p in plans])])
    up = torch.from_numpy(host).pin_memory().to(device, non_blocking=True)
    n_idx = idx.size
    idx_d = up[:n_idx].view(torch.int64).view(4, -1)
    traj_d = up[n_idx:n_idx + 2 * int(toff[-1])].view(-1, 2)
    label_d = up[n_idx + 2 * int(toff[-1]):n_idx + 2 * int(toff[-1]) + K].view(torch.int64)
    ratio_d = up[n_idx + 2 * int(toff[-1]) + K:]
    planes = torch.zeros((3, K, W, W), dtype=torch.float64, device=device)
    planes[idx_d[0], idx_d[1], idx_d[2], idx_d[3]] = 1.0
    files, k = [], 0
    for p, _, out_dir in batch:
        for name in p["name"]:
            files.append((os.path.join(out_dir, name), dict(
                image=images[k], start_image=planes[0, k], goal_image=planes[1, k], traj_image=planes[2, k],
                traj=traj_d[toff[k]:toff[k + 1]], label=label_d[k], length_ratio=ratio_d[k])))
            k += 1
    _savez_compressed_many(files)


def save_sdd_samples(video_dirs, save_dir: str, W: int = 64, min_len_ratio: float = 0.5, min_max_size: int = 128,
                     max_step: int = 300, rng=None, device=None, batch_samples: int = 4096) -> int:
    """planning-datasets' SDD samples (create_sample_from_dataset over `video_dirs`, in the order given) written on the
    GPU (DESIGN.md §22): for each video directory, `<save_dir>/<scene>/<video>/` is created (also when it gets no
    samples) and every kept sample of sdd_sample_plan is written there as `%08d_%02d.npz` with members image (uint8
    [W, W, 3]), start_image, goal_image, traj_image (float64 [W, W]), traj (float64 [n, 2]), label (int64) and
    length_ratio (float64), loading equal to the reference's files.  Scenes are decoded by Pillow on the host and
    must be RGB; the crops are resized by one kernel launch and the files deflated by one more per batch of about
    `batch_samples` samples.  rng: a np.random.RandomState (None: RandomState(0), the generator script's
    np.random.seed(0)).  device: a CUDA device (None: the current one).  Returns the number of files written."""
    rng = np.random.RandomState(0) if rng is None else rng
    dev = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
    if dev.type != "cuda":
        raise RuntimeError("save_sdd_samples runs on a CUDA device (there is no CPU fallback)")
    batch, n, total = [], 0, 0
    for video_dir in video_dirs:
        plan = sdd_sample_plan(video_dir, W, min_len_ratio, min_max_size, max_step, rng)
        out_dir = os.path.join(save_dir, plan["scene"], plan["video"])
        os.makedirs(out_dir, exist_ok=True)
        if not plan["name"]:
            continue
        batch.append((plan, _sdd_scene(video_dir, dev), out_dir))
        n += len(plan["name"])
        if n >= batch_samples:
            _write_sdd_samples(batch, W, dev)
            total += n
            batch, n = [], 0
    _write_sdd_samples(batch, W, dev)
    return total + n


# the .npy dtypes load_npz_device reads: NumPy's descr -> the torch dtype of the same bytes
_NPY_TORCH_DTYPE = {"|b1": torch.bool, "|u1": torch.uint8, "|i1": torch.int8, "<i2": torch.int16, "<i4": torch.int32,
                    "<i8": torch.int64, "<f2": torch.float16, "<f4": torch.float32, "<f8": torch.float64}
_NPY_MAGIC = b"\x93NUMPY"


class NpzMember(tuple):
    """One member of a .npz file as load_npz_device reads it: (key, method, data_off, csize, usize, crc, descr, shape,
    header_len).  data_off / csize: the stored or deflated bytes in the file; usize: the inflated .npy size;
    header_len: the bytes of its .npy header, after which the array's C-order bytes follow."""


def _npz_plan(blob, name: str = "<bytes>") -> list:
    """The members of a .npz file held in memory, parsed on the host as zipfile and np.lib.format read them: the end
    record (ZIP64 where present), the central directory (sizes and CRC from there, with ZIP64 extras, so members
    written with data descriptors work) and each local header's length.  Each member's .npy header (format 1, 2 or 3)
    comes from its first bytes alone, inflated with zlib.decompressobj(-15) when it is deflated.  Returns a list of
    NpzMember in central-directory order.  Anything load_npz_device does not read raises ValueError naming the file and
    the member: methods other than stored (0) and deflated (8), encryption, members that are not .npy files, dtypes
    other than |b1 |u1 |i1 <i2 <i4 <i8 <f2 <f4 <f8 (object, structured and big-endian ones among them), Fortran order,
    and sizes that do not add up."""
    import ast
    import struct
    import zlib

    blob = memoryview(blob).cast("B")
    n = len(blob)

    def bad(why, member=None):
        return ValueError(f"{name}: {why}" if member is None else f"{name}: member {member!r}: {why}")

    tail = bytes(blob[max(0, n - 22 - 0xFFFF):])
    e = tail.rfind(b"PK\x05\x06")
    if e < 0 or len(tail) - e < 22:
        raise bad("not a zip file (no end of central directory record)")
    eocd = n - len(tail) + e
    _, _, _, _, count, cd_size, cd_off, _ = struct.unpack("<IHHHHIIH", blob[eocd:eocd + 22])
    if eocd >= 20 and bytes(blob[eocd - 20:eocd - 16]) == b"PK\x06\x07":
        z64 = struct.unpack("<Q", blob[eocd - 12:eocd - 4])[0]
        if z64 + 56 > n or bytes(blob[z64:z64 + 4]) != b"PK\x06\x06":
            raise bad("corrupt ZIP64 end of central directory record")
        count, _, cd_size, cd_off = struct.unpack("<QQQQ", blob[z64 + 24:z64 + 56])
    if cd_off + cd_size > n:
        raise bad("central directory outside the file")
    members, pos = [], cd_off
    for _ in range(count):
        if pos + 46 > n or bytes(blob[pos:pos + 4]) != b"PK\x01\x02":
            raise bad("corrupt central directory")
        (_, _, _, flags, method, _, _, crc, csize, usize, nlen, elen, clen, _, _, _,
         lh) = struct.unpack("<IHHHHHHIIIHHHHHII", blob[pos:pos + 46])
        member = bytes(blob[pos + 46:pos + 46 + nlen]).decode("utf-8" if flags & 0x800 else "cp437")
        extra = bytes(blob[pos + 46 + nlen:pos + 46 + nlen + elen])
        pos += 46 + nlen + elen + clen
        x = 0
        while x + 4 <= len(extra):   # ZIP64 extra: the 64-bit values of the fields that hold 0xFFFFFFFF, in order
            tag, size = struct.unpack("<HH", extra[x:x + 4])
            if tag == 1:
                vals = list(struct.unpack(f"<{size // 8}Q", extra[x + 4:x + 4 + size // 8 * 8]))
                if usize == _U32 and vals:
                    usize = vals.pop(0)
                if csize == _U32 and vals:
                    csize = vals.pop(0)
                if lh == _U32 and vals:
                    lh = vals.pop(0)
            x += 4 + size
        if flags & 1:
            raise bad("encrypted members are not supported", member)
        if method not in (0, 8):
            raise bad(f"compression method {method} is not supported (only stored and deflated)", member)
        if not member.endswith(".npy"):
            raise bad("not a .npy member", member)
        if lh + 30 > n or bytes(blob[lh:lh + 4]) != b"PK\x03\x04":
            raise bad("corrupt local header", member)
        lnlen, lelen = struct.unpack("<HH", blob[lh + 26:lh + 30])
        data_off = lh + 30 + lnlen + lelen
        if data_off + csize > n or (method == 0 and csize != usize):
            raise bad("member data outside the file or of the wrong size", member)
        comp = blob[data_off:data_off + csize]

        def first(k):   # the member's first k inflated bytes (fewer at its end)
            if method == 0:
                return bytes(comp[:k])
            try:
                return zlib.decompressobj(-15).decompress(comp, k)
            except zlib.error as err:
                raise bad(f"corrupt deflate stream ({err})", member) from None

        head = first(12)
        if len(head) < 10 or head[:6] != _NPY_MAGIC or head[6] not in (1, 2, 3):
            raise bad("not a .npy file of format 1, 2 or 3", member)
        start = 10 if head[6] == 1 else 12
        hl = struct.unpack("<H" if head[6] == 1 else "<I", head[8:start])[0]
        text = first(start + hl)[start:]
        if len(text) != hl:
            raise bad("truncated .npy header", member)
        try:
            d = ast.literal_eval(text.decode("utf-8" if head[6] == 3 else "latin-1"))
        except (ValueError, SyntaxError, UnicodeDecodeError):
            raise bad("unreadable .npy header", member) from None
        if not isinstance(d, dict) or set(d) != {"descr", "fortran_order", "shape"}:
            raise bad("unreadable .npy header", member)
        descr, shape = d["descr"], d["shape"]
        try:
            dt = np.dtype(descr).str if isinstance(descr, str) else None
        except TypeError:
            dt = None
        if dt not in _NPY_TORCH_DTYPE:
            raise bad(f"dtype {descr!r} is not supported (only {' '.join(_NPY_TORCH_DTYPE)})", member)
        if d["fortran_order"]:
            raise bad("Fortran-order arrays are not supported", member)
        if not isinstance(shape, tuple) or not all(isinstance(v, int) and v >= 0 for v in shape):
            raise bad(f"bad shape {shape!r}", member)
        descr = dt
        if start + hl + int(np.prod(shape, dtype=np.int64)) * np.dtype(descr).itemsize != usize:
            raise bad("the .npy header does not match the member's size", member)
        members.append(NpzMember((member[:-4], method, data_off, csize, usize, crc, descr, tuple(shape), start + hl)))
    return members


def load_npz_device(files, device=None) -> list:
    """np.load for many .npz files at once, with the members inflated on the GPU (include/nastar_b200.h,
    nastar_b200_inflate; DESIGN.md §23).  files: paths or `bytes`.  Returns one dict per file of what np.load(f) gives,
    {member name without ".npy": CUDA tensor} with the same dtypes, shapes and values.

    The host parses the zip records and each member's .npy header (_npz_plan: anything it does not read raises
    ValueError naming the file and member before any launch), copies every member's stored or deflated bytes to
    `device` (the current CUDA device when None) in one transfer and allocates one output buffer, each array's bytes
    starting 64-byte aligned, so every array is a typed view of it.  One launch inflates every member of every file;
    one synchronisation then reads the statuses and CRC-32s: a corrupt stream or a CRC-32 that differs from the zip's
    raises ValueError naming the file and member, whose `arrays` attribute holds the result, exact for every member it
    does not name.  One warp inflates one member, so this suits many small members
    (such as the SDD samples), not a few huge ones."""
    names, blobs = [], []
    for f in files:
        if isinstance(f, (bytes, bytearray, memoryview)):
            names.append(f"<npz {len(names)}>")
            blobs.append(f)
        else:
            names.append(os.fspath(f))
            with open(f, "rb") as fh:
                blobs.append(fh.read())
    plans = [_npz_plan(b, n) for b, n in zip(blobs, names)]
    if not blobs:
        return []
    dev = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
    if dev.type != "cuda":
        raise RuntimeError("load_npz_device runs on a CUDA device (there is no CPU fallback)")
    M = sum(len(p) for p in plans)
    desc = np.zeros(M, _native.INFLATE_DESC_DTYPE)
    head = (desc.nbytes + 63) // 64 * 64
    total = head + sum(m[3] for p in plans for m in p)
    buf = torch.empty((max(total, 1),), dtype=torch.uint8).pin_memory()
    host = buf.numpy()
    pos, out_pos, i = head, 0, 0
    for blob, plan in zip(blobs, plans):
        b = np.frombuffer(blob, np.uint8)
        for key, method, off, csize, usize, _, _, _, hl in plan:
            out_pos = (out_pos + hl + 63) // 64 * 64 - hl   # the array's bytes start 64-byte aligned
            host[pos:pos + csize] = b[off:off + csize]
            desc[i] = (pos, csize, out_pos, usize, method, 0)
            pos += csize
            out_pos += usize
            i += 1
    host[:desc.nbytes] = desc.view(np.uint8)
    with torch.cuda.device(dev):
        data = buf.to(dev, non_blocking=True)
        out = torch.empty((max(out_pos, 1),), dtype=torch.uint8, device=dev)
        if M:
            status, crc = _native.inflate(data, desc, data[:desc.nbytes], out)
            meta = torch.cat([status.to(torch.int64), crc.to(torch.int64) & _U32]).cpu().numpy().reshape(2, M)
        else:
            meta = np.zeros((2, 0), np.int64)
    result, i, errors = [], 0, []
    for name, plan in zip(names, plans):
        arrays = {}
        for key, _, _, _, usize, crc, descr, shape, hl in plan:
            st, got = int(meta[0, i]), int(meta[1, i])
            if st:
                why = ", ".join(w for bit, w in _native.INFLATE_STATUS.items() if st & bit)
                errors.append(f"{name}: member {key + '.npy'!r}: corrupt deflate stream ({why})")
            elif got != crc:
                errors.append(f"{name}: Bad CRC-32 for file {key + '.npy'!r}")
            a = int(desc[i]["out_off"]) + hl
            arrays[key] = out[a:a + usize - hl].view(_NPY_TORCH_DTYPE[descr]).view(shape)
            i += 1
        result.append(arrays)
    if errors:
        err = ValueError("; ".join(errors[:20]))
        err.arrays = result   # what the call read: exact for every member the message does not name
        raise err
    return result


class DeviceSDDDataset:
    def __init__(self, root: str, scenes=None, device=None):
        """The Stanford Drone planning samples that save_sdd_samples / tools/make_sdd_dataset.py write, read back onto
        the GPU for training Neural A* on raw RGB images (DESIGN.md §23): every `<root>/<scene>/<video>/*.npz`, in
        sorted (scene, video, file) order, of the given `scenes` only when given, read by one load_npz_device call.

        Keeps map_designs fp32 [N,3,W,W] = (image.transpose(2, 0, 1) / 255.0).astype(np.float32) (WarCraftDataset's
        rule), start_maps / goal_maps / traj_images fp32 [N,1,W,W] (start_image, goal_image, traj_image), label int64
        [N], length_ratio fp64 [N], the ragged trajectories as traj fp64 [T,2] with traj_offsets int64 [N+1] (sample i
        is traj[traj_offsets[i]:traj_offsets[i+1]]), all on the device, and per sample the host lists scene and name
        ("<video>/<file>").  A scene that is not in the tree, or a selection without samples, raises ValueError."""
        import glob

        root = os.fspath(root)
        present = sorted(d for d in os.listdir(root) if os.path.isdir(os.path.join(root, d)))
        scenes = present if scenes is None else sorted(set(scenes))
        unknown = [s for s in scenes if s not in present]
        if unknown:
            raise ValueError(f"{root}: no scene {unknown} (scenes: {present})")
        files = []
        for s in scenes:   # within a scene, the paths sort as (video, file): "/" sorts before any name character
            files += sorted(glob.glob(os.path.join(glob.escape(root), glob.escape(s), "*", "*.npz")))
        if not files:
            raise ValueError(f"{root}: no samples in scenes {scenes}")
        arrays = load_npz_device(files, device)
        self.scene = [os.path.basename(os.path.dirname(os.path.dirname(f))) for f in files]
        self.name = [os.path.relpath(f, os.path.dirname(os.path.dirname(f))) for f in files]
        images = torch.stack([a["image"] for a in arrays])
        self.device = images.device
        self.map_designs = (images.permute(0, 3, 1, 2).double() / 255.0).float().contiguous()
        self.start_maps, self.goal_maps, self.traj_images = (
            torch.stack([a[k] for a in arrays])[:, None].float() for k in ("start_image", "goal_image", "traj_image"))
        self.label = torch.stack([a["label"] for a in arrays])
        self.length_ratio = torch.stack([a["length_ratio"] for a in arrays])
        self.traj = torch.cat([a["traj"] for a in arrays])
        self.traj_offsets = torch.tensor(np.concatenate([[0], np.cumsum([a["traj"].shape[0] for a in arrays])]),
                                         dtype=torch.int64, device=self.device)

    def __len__(self):
        return self.map_designs.shape[0]

    def sample(self, indices, generator: torch.Generator = None):
        """(map_designs [B,3,W,W], start_maps, goal_maps, traj_images [B,1,W,W]) of the samples `indices` (host or
        device), the batch PlannerModule and GraphedTrainStep take (traj_images is the target, as opt_trajs is for
        mazes).  The samples are fixed: `generator` is accepted for DeviceDataLoader and not used."""
        idx = torch.as_tensor(indices)
        if idx.device.type == "cpu":
            if idx.numel() and (int(idx.min()) < 0 or int(idx.max()) >= len(self)):
                raise IndexError(f"indices must lie in [0, {len(self)})")
        idx = idx.to(self.device).reshape(-1).to(torch.int64)
        return self.map_designs[idx], self.start_maps[idx], self.goal_maps[idx], self.traj_images[idx]


def sdd_leave_one_scene_out(root: str, test_scene: str, device=None):
    """(train, test) DeviceSDDDatasets of the SDD sample tree at `root`: test holds the samples of `test_scene`, train
    those of every other scene.  An unknown scene raises ValueError."""
    root = os.fspath(root)
    scenes = sorted(d for d in os.listdir(root) if os.path.isdir(os.path.join(root, d)))
    if test_scene not in scenes:
        raise ValueError(f"{root}: no scene {test_scene!r} (scenes: {scenes})")
    return (DeviceSDDDataset(root, [s for s in scenes if s != test_scene], device),
            DeviceSDDDataset(root, [test_scene], device))


__all__ = ["AstarOutput", "DeviceDataLoader", "DeviceMazeDataset", "DeviceSDDDataset", "MazeDataset",
           "WarCraftDataset", "compute_opt_labels", "compute_weighted_opt_labels", "create_dataloader",
           "create_device_dataloader", "create_warcraft_dataloader", "draw_opt_policies", "encode_pngs",
           "load_map_images", "load_npz_device", "maps_from_images",
           "read_sdd_annotations", "sample_device_goal_maps", "sample_goal_maps", "save_planning_dataset",
           "save_pngs", "save_sdd_samples", "save_search_gifs",
           "savez_compressed_device", "save_warcraft_dataset", "search_gifs",
           "sdd_crops", "sdd_leave_one_scene_out", "sdd_sample_plan", "shortest_path_maps", "street_crop_boxes",
           "tile_maps", "visualize_results"]
