#!/usr/bin/env python
"""Search animations of a planning dataset's test problems, as the reference's scripts/create_gif.py makes them, with
the frames drawn and encoded on the GPU (utils.data.save_search_gifs, DESIGN.md §19).

The first 100 test problems are loaded as the reference does (create_dataloader, one random start each, no shuffle);
the chosen planner searches them and GIFs are written to {resultdir}/{planner}/video_{dataname}_{problem_id:04d}.gif
(scale 4, 30 fps, the last frame held for 15 more).  --all-problems writes one file per problem, --grid one file of
all 100 (video_{dataname}_grid.gif).

    python tools/create_gif.py --dataset planning-datasets/data/mpd/mazes_032_moore_c8 --planner na \\
        --modeldir model --problem-id 0
"""
import argparse
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "neural-astar_b200")]

import torch  # noqa: E402


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--dataset", required=True, help="dataset path without .npz")
    ap.add_argument("--planner", choices=("na", "va"), default="na")
    ap.add_argument("--problem-id", type=int, default=0)
    ap.add_argument("--modeldir", default="model")
    ap.add_argument("--resultdir", default="results")
    ap.add_argument("--encoder-input", default="m+")
    ap.add_argument("--encoder-arch", default="CNN")
    ap.add_argument("--encoder-depth", type=int, default=4)
    ap.add_argument("--all-problems", action="store_true", help="one GIF per test problem")
    ap.add_argument("--grid", action="store_true", help="one GIF of all problems in make_grid's layout")
    args = ap.parse_args(argv)

    from neural_astar.planner import NeuralAstar, VanillaAstar
    from neural_astar.utils.data import create_dataloader, save_search_gifs
    from neural_astar.utils.training import load_from_ptl_checkpoint

    dataname = os.path.basename(args.dataset)
    if args.planner == "na":
        planner = NeuralAstar(encoder_input=args.encoder_input, encoder_arch=args.encoder_arch,
                              encoder_depth=args.encoder_depth, learn_obstacles=False, Tmax=1.0)
        planner.load_state_dict(load_from_ptl_checkpoint(f"{args.modeldir}/{dataname}"))
    else:
        planner = VanillaAstar()
    dev = torch.device("cuda")
    planner = planner.to(dev).eval()
    savedir = f"{args.resultdir}/{args.planner}"
    os.makedirs(savedir, exist_ok=True)
    maps, starts, goals, _ = next(iter(create_dataloader(args.dataset + ".npz", "test", 100, shuffle=False,
                                                         num_starts=1)))
    maps, starts, goals = maps.to(dev), starts.to(dev), goals.to(dev)
    kw = dict(scale=4, fps=30, hold=15)
    with torch.no_grad():
        if args.grid:
            path = f"{savedir}/video_{dataname}_grid.gif"
            save_search_gifs([path], planner, maps, starts, goals, layout="grid", **kw)
            print(path)
        ids = range(len(maps)) if args.all_problems else ([] if args.grid else [args.problem_id])
        ids = list(ids)
        if ids:
            paths = [f"{savedir}/video_{dataname}_{i:04d}.gif" for i in ids]
            save_search_gifs(paths, planner, maps[ids], starts[ids], goals[ids], **kw)
            print("\n".join(paths))


if __name__ == "__main__":
    main()
