#!/usr/bin/env python
"""Make a planning-datasets .npz from map images on the GPU, with generate_spp_instances.py's arguments and file name
(`<name>_<size:03d>_<mechanism>_c<edge>.npz`, name = the last part of --input-path, `all` when it holds a `*`).

Per split (train, validation, test): decode the PNGs on the GPU (load_map_pngs, bit-equal to Pillow) -> maps_from_images (bicubic
resize + Otsu, bit-equal to the generator) -> with --tile-size t > 1, split-size tiles of t x t maps whose indices
come from np.random.RandomState(seed).choice, as the generator draws them (its train tiles replay exactly; its
validation and test tiles follow label draws and do not) -> sample_device_goal_maps (largest region, corner squares of
int(edge_ratio * size * t)) -> compute_opt_labels + draw_opt_policies (a uniform member of each maximal action set) ->
save_planning_dataset, which deflates the twelve arrays on the GPU too (savez_compressed_device, DESIGN.md §18), so only
the compressed file crosses to the host.  --mechanism moore (8 actions, the default) or news (4 actions, 4-connected
distances) is the generator's transition mechanism; the goals are the same for both.  Goals and policies come from a CUDA
torch.Generator seeded with --seed, so they are not the generator's random draws.  With --tile-size 1 the split sizes are ignored and every image is used, as there.

    python tools/make_planning_dataset.py --input-path data/mpd/original/mazes --output-path out --maze-size 32 \\
        --edge-ratio 0.25
"""
import argparse
import os
import re
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "neural-astar_b200"))


MECHANISMS = ("news", "moore")


def output_name(input_path: str, maze_size: int, tile_size: int, edge_size: int, mechanism: str = "moore") -> str:
    name = re.split("/", input_path.rstrip("/"))[-1]
    return "{}_{:03d}_{}_c{}.npz".format("all" if "*" in name else name, maze_size * tile_size, mechanism, edge_size)


def make(args) -> str:
    import torch

    from neural_astar.utils.data import (compute_opt_labels, draw_opt_policies, load_map_pngs, maps_from_images,
                                         sample_device_goal_maps, save_planning_dataset, tile_maps)

    if args.mechanism not in MECHANISMS:
        raise SystemExit(f"--mechanism must be one of {', '.join(MECHANISMS)} (got {args.mechanism!r})")
    num_actions = 4 if args.mechanism == "news" else 8
    dev = torch.device("cuda", torch.cuda.current_device())
    t = int(args.tile_size)
    edge = int(args.edge_ratio * args.maze_size * t)
    rng = np.random.RandomState(args.seed)
    gen = torch.Generator(dev).manual_seed(args.seed)
    splits, t0 = [], time.time()
    for split, n in (("train", args.train_size), ("validation", args.valid_size), ("test", args.test_size)):
        maps = maps_from_images(load_map_pngs(args.input_path, split, device=dev), args.maze_size, device=dev)
        if t > 1:
            maps = tile_maps(maps, t, indices=np.stack([rng.choice(len(maps), t * t) for _ in range(n)]))
        goals = sample_device_goal_maps(maps, edge, generator=gen)
        _, dists, mask = compute_opt_labels(maps, goals, args.mechanism)
        splits.append((maps, goals, draw_opt_policies(mask, generator=gen, num_actions=num_actions), dists))
        print(f"{split}: {maps.shape[0]} maps {maps.shape[-2]}x{maps.shape[-1]}")
    os.makedirs(args.output_path, exist_ok=True)
    path = os.path.join(args.output_path, output_name(args.input_path, args.maze_size, t, edge, args.mechanism))
    save_planning_dataset(path, *splits)
    print(f"wrote {path} in {time.time() - t0:.1f} s")
    return path


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--input-path", required=True, help="directory with train/validation/test PNGs ('*' allowed)")
    ap.add_argument("--output-path", required=True, help="directory for the .npz")
    ap.add_argument("--maze-size", type=int, required=True, help="map side after the resize")
    ap.add_argument("--mechanism", default="moore", help="transition mechanism: news or moore")
    ap.add_argument("--edge-ratio", type=float, default=0, help="goal corner squares, as a share of the side")
    ap.add_argument("--train-size", type=int, default=800)
    ap.add_argument("--valid-size", type=int, default=100)
    ap.add_argument("--test-size", type=int, default=100)
    ap.add_argument("--seed", type=int, default=1372)
    ap.add_argument("--tile-size", type=int, default=1)
    make(ap.parse_args())


if __name__ == "__main__":
    main()
