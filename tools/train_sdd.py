#!/usr/bin/env python
"""Neural A* on the Stanford Drone planning samples (the paper's planning on raw image inputs), leave one scene out:
for each held-out scene, train NeuralAstar(encoder_input="rgb+", learn_obstacles=True) on every other scene to imitate
the pedestrian trajectories (traj_images, as opt_trajs for mazes), then score it on the held-out scene by the Chamfer
distance between its paths and the trajectories, beside VanillaAstar on all-passable maps (the straight-path
baseline).  The samples are those tools/make_sdd_dataset.py writes, read onto the GPU by DeviceSDDDataset.

Training replays GraphedTrainStep on full batches of a shuffled DeviceDataLoader; the partial last batch of each epoch
is dropped (reported on stderr).  Evaluation runs in eval mode under no_grad.  One JSON line per scene on stdout.

    python tools/train_sdd.py --data-dir data/sdd/s064_0.5_128_300 --test-scene <scene> [--epochs 20] ...
    python tools/train_sdd.py --data-dir data/sdd/s064_0.5_128_300 --all-scenes
"""
import argparse
import json
import os
import sys
import time
from types import SimpleNamespace

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "neural-astar_b200"))

import torch  # noqa: E402


def run_scene(args, scene, dev):
    from neural_astar.planner import NeuralAstar
    from neural_astar.utils.data import DeviceDataLoader, sdd_leave_one_scene_out
    from neural_astar.utils.training import GraphedTrainStep, PlannerModule, chamfer_distance, set_global_seeds

    train, test = sdd_leave_one_scene_out(args.data_dir, scene, dev)
    bs = args.batch_size
    batches = len(train) // bs
    if batches == 0:
        raise SystemExit(f"{scene}: {len(train)} training samples, fewer than one batch of {bs}")
    print(f"{scene}: {len(train)} training samples, {batches} batches of {bs} per epoch; the last "
          f"{len(train) - batches * bs} samples of each shuffled epoch are dropped", file=sys.stderr)
    set_global_seeds(args.seed)
    planner = NeuralAstar(g_ratio=args.g_ratio, Tmax=args.Tmax, encoder_input="rgb+", encoder_arch=args.encoder_arch,
                          encoder_depth=args.encoder_depth, learn_obstacles=True, const=args.const)
    module = PlannerModule(planner, SimpleNamespace(params=SimpleNamespace(lr=args.lr))).to(dev).train()
    step = GraphedTrainStep(module, train.sample(range(bs)))
    loader = DeviceDataLoader(train, bs, shuffle=True, generator=torch.Generator(device=dev).manual_seed(args.seed))
    torch.cuda.synchronize(dev)
    t0 = time.perf_counter()
    loss = None
    for _ in range(args.epochs):
        for batch in loader:
            if batch[0].shape[0] == bs:
                loss = step(batch)
    torch.cuda.synchronize(dev)
    seconds = time.perf_counter() - t0
    module.eval()
    na, va = [], []
    with torch.no_grad():
        for map_designs, start_maps, goal_maps, traj_images in DeviceDataLoader(test, bs):
            na.append(chamfer_distance(planner(map_designs, start_maps, goal_maps).paths, traj_images))
            vanilla = module.vanilla_astar(torch.ones_like(start_maps), start_maps, goal_maps)
            va.append(chamfer_distance(vanilla.paths, traj_images))
    na, va = torch.cat(na).mean().item(), torch.cat(va).mean().item()
    return dict(test_scene=scene, train_samples=len(train), test_samples=len(test), batch_size=bs,
                batches_per_epoch=batches, epochs=args.epochs, encoder_arch=args.encoder_arch,
                final_train_loss=float(loss), seconds=round(seconds, 3), chamfer_neural_astar=na,
                chamfer_vanilla_astar=va)


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--data-dir", required=True, help="a <scene>/<video>/*.npz tree of make_sdd_dataset.py")
    which = ap.add_mutually_exclusive_group(required=True)
    which.add_argument("--test-scene", help="the held-out scene")
    which.add_argument("--all-scenes", action="store_true", help="hold out each scene in turn")
    ap.add_argument("--encoder-arch", choices=("CNN", "Unet"), default="CNN")
    ap.add_argument("--encoder-depth", type=int, default=4)
    ap.add_argument("--Tmax", type=float, default=0.25)
    ap.add_argument("--const", type=float, default=None)
    ap.add_argument("--g-ratio", type=float, default=0.5)
    ap.add_argument("--lr", type=float, default=1e-3)
    ap.add_argument("--batch-size", type=int, default=64)
    ap.add_argument("--epochs", type=int, default=20)
    ap.add_argument("--seed", type=int, default=1234)
    args = ap.parse_args(argv)
    if not torch.cuda.is_available():
        raise SystemExit("train_sdd.py needs a GPU")
    dev = torch.device("cuda", torch.cuda.current_device())
    scenes = (sorted(d for d in os.listdir(args.data_dir) if os.path.isdir(os.path.join(args.data_dir, d)))
              if args.all_scenes else [args.test_scene])
    results = []
    for scene in scenes:
        rec = run_scene(args, scene, dev)
        print(json.dumps(rec), flush=True)
        results.append(rec)
    return results


if __name__ == "__main__":
    main()
