#!/usr/bin/env python
"""Make the CSM street-map dataset on the GPU: planning-datasets' 2_CSM.sh in one process.

1. The crops of preprocess_street_dataset.py (crop_images): the `*[0,1]_256.png` sources of --input-path in glob order
   give the train crops (160 per file) and then the validation crops (20 per file), the `*2_256.png` sources the test
   crops (40 per file), their boxes drawn by np.random.RandomState(--seed) in that order (street_crop_boxes).  The
   sources are decoded on the GPU (decode_pngs, bit-equal to Pillow's convert("L")), a source that is not 256 x 256 is
   resized to it by the maps kernel's bicubic resize (bit-equal to Pillow's), the 128 x 128 crops are gathered on the
   device and written as PNGs encoded there (save_pngs) into --crops-path/{train,validation,test}, named
   "<fileid>_<n:05d>.png" as the reference names them.
2. generate_spp_instances.py --maze-size 64 --mechanism moore --edge-ratio 0.25 --train-size 3200 --valid-size 400
   --test-size 400 on --crops-path: make_planning_dataset.make(), which writes <output-path>/mixed_064_moore_c16.npz
   when --crops-path ends in `mixed`.  Its goals and policies come from make()'s default seed, 1372, as there.

    python tools/make_street_dataset.py --input-path data/street/original/all \\
        --crops-path data/street/original/mixed --output-path data/street
"""
import argparse
import glob
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "neural-astar_b200"))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

SPLITS = ("train", "validation", "test")
SOURCE_SIZE, CROP_SIZE = 256, 128
COUNTS = (160, 20, 40)
DATASET = dict(maze_size=64, mechanism="moore", edge_ratio=0.25, train_size=3200, valid_size=400, test_size=400,
               seed=1372, tile_size=1)


def source_files(input_path: str):
    """The train and test sources in glob order, with crop_images' patterns."""
    return glob.glob("%s/*[0,1]_256.png" % input_path), glob.glob("%s/*2_256.png" % input_path)


def crop_street_maps(train_files, test_files, crops_path: str, seed: int = 1372, counts=COUNTS, device=None) -> dict:
    """Write crop_images' crops of the sources (ordered lists, as the draws take them) into crops_path/<split>/.
    Returns {split: [paths written]}."""
    import torch

    from neural_astar import _native
    from neural_astar.utils.data import decode_pngs, save_pngs, street_crop_boxes

    dev = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
    boxes = street_crop_boxes(train_files, test_files, size=CROP_SIZE, counts=counts, seed=seed,
                              source_size=SOURCE_SIZE)
    files = list(train_files) + list(test_files)
    blobs = []
    for f in files:
        with open(f, "rb") as fh:
            blobs.append(fh.read())
    groups, _ = decode_pngs(blobs, files, device=dev)
    sources = torch.empty((len(files), SOURCE_SIZE, SOURCE_SIZE), dtype=torch.uint8, device=dev)
    for pos, imgs in groups:
        if tuple(imgs.shape[1:]) != (SOURCE_SIZE, SOURCE_SIZE):   # Image.resize((256, 256)) is the identity at 256
            imgs = _native.maps_from_images(imgs, SOURCE_SIZE, SOURCE_SIZE, want_resized=True)[1]
        sources[torch.from_numpy(pos).to(dev)] = imgs
    ar = torch.arange(CROP_SIZE, device=dev)
    written = {}
    for split in SPLITS:
        b = boxes[split]
        base = len(train_files) if split == "test" else 0
        src = torch.from_numpy(b["source"] + base).to(dev)
        top, left = torch.from_numpy(b["top"]).to(dev), torch.from_numpy(b["left"]).to(dev)
        crops = sources[src[:, None, None], (top[:, None] + ar)[:, :, None], (left[:, None] + ar)[:, None, :]]
        out_dir = os.path.join(crops_path, split)
        os.makedirs(out_dir, exist_ok=True)
        paths = [os.path.join(out_dir, name) for name in b["name"]]
        if paths:
            save_pngs(paths, crops)
        written[split] = paths
        print(f"{split}: {len(paths)} crops from {len(test_files if split == 'test' else train_files)} sources")
    return written


def make(train_files, test_files, crops_path: str, output_path: str, seed: int = 1372, counts=COUNTS) -> str:
    """Both steps of 2_CSM.sh; returns the .npz path."""
    import make_planning_dataset

    t0 = time.time()
    crop_street_maps(train_files, test_files, crops_path, seed=seed, counts=counts)
    print(f"crops written in {time.time() - t0:.1f} s")
    return make_planning_dataset.make(argparse.Namespace(input_path=crops_path, output_path=output_path, **DATASET))


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--input-path", required=True, help="directory of the street-map sources (*_256.png)")
    ap.add_argument("--crops-path", required=True, help="directory for the train/validation/test crops")
    ap.add_argument("--output-path", required=True, help="directory for the .npz")
    ap.add_argument("--seed", type=int, default=1372, help="seed of the crop boxes")
    args = ap.parse_args()
    train_files, test_files = source_files(args.input_path)
    if not train_files or not test_files:
        raise SystemExit(f"no *[0,1]_256.png and *2_256.png sources in {args.input_path}")
    make(train_files, test_files, args.crops_path, args.output_path, seed=args.seed)


if __name__ == "__main__":
    main()
