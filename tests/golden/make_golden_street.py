#!/usr/bin/env python
"""Fixture for the CSM street crops (tests/golden/street/): synthetic street-map sources and what the reference's own
crop_images (planning-datasets/preprocess_street_dataset.py) does with them.

  sources/*.png    six street-like sources: blocks of buildings (0) between roads (255), parks and yards in a few grey
                   levels; four train files (*0_256.png, *1_256.png) and two test files (*2_256.png).  Boston_1_256.png
                   is 320 wide and 200 high and RGB, so crop_images' convert("L").resize((256, 256)) is not a no-op
  street.npz       glob_train, glob_test   the file names in the glob order crop_images saw
                   <ns>_boxes_<split>      every box crop_images passed to Image.crop, int64 [N, 4] (left, top, right,
                                           bottom), in call order
                   <ns>_names_<split>      the file names it saved, in the same order
                   small_crops_<split>     the saved small crops as Pillow decodes them, uint8 [N, 128, 128]
                   with <ns> "default" (Ns = [160, 20, 40]) and "small" (Ns = [8, 2, 4]), each run after
                   np.random.seed(1372) as the script's __main__ does

    python tests/golden/make_golden_street.py --reference PATH   # PATH: a checkout of the reference repository
"""
import argparse
import glob as globmod
import importlib.util
import os
import tempfile

import numpy as np
from PIL import Image

HERE = os.path.dirname(os.path.abspath(__file__))
OUT = os.path.join(HERE, "street")
SMALL = [8, 2, 4]
SPLITS = ("train", "validation", "test")


def street_map(rng, H, W, levels=(128, 200)):
    """Blocks of 0 between roads of 255; some blocks are parks or yards in the given grey levels."""
    img = np.full((H, W), 255, np.uint8)
    y = int(rng.randint(0, 12))
    while y < H:
        bh = int(rng.randint(14, 40))
        x = int(rng.randint(0, 12))
        while x < W:
            bw = int(rng.randint(14, 48))
            r = rng.rand()
            level = 0 if r < 0.7 else levels[int(rng.randint(len(levels)))]
            img[y:y + bh, x:x + bw] = level
            x += bw + int(rng.choice([3, 4, 6, 8]))
        y += bh + int(rng.choice([3, 4, 6, 8]))
    # a few diagonal roads across the blocks
    for _ in range(int(rng.randint(1, 3))):
        x0, slope = int(rng.randint(0, W)), rng.uniform(-1.5, 1.5)
        for yy in range(H):
            xx = int(x0 + slope * yy)
            img[yy, max(xx, 0):max(xx + 4, 0)] = 255
    return img


def write_sources(src_dir):
    rng = np.random.RandomState(2024)
    specs = [("Berlin_0_256.png", 256, 256, "L"), ("Berlin_1_256.png", 256, 256, "L"),
             ("Boston_0_256.png", 256, 256, "L"), ("Boston_1_256.png", 200, 320, "RGB"),
             ("Berlin_2_256.png", 256, 256, "L"), ("Boston_2_256.png", 256, 256, "L")]
    for name, H, W, mode in specs:
        img = street_map(rng, H, W)
        im = Image.fromarray(img)
        if mode == "RGB":
            rgb = np.stack([img, np.maximum(img, 30), img], axis=-1).astype(np.uint8)   # greenish roads
            im = Image.fromarray(rgb, "RGB")
        im.save(os.path.join(src_dir, name))


def run_reference(module, src_dir, ns):
    """crop_images(src_dir, <tmp>, Ns=ns) after np.random.seed(1372): (glob orders, boxes and names per split, the
    saved crops per split)."""
    seen = {"globs": [], "boxes": [], "saves": []}
    real_glob, real_crop, real_save = module.glob, Image.Image.crop, Image.Image.save

    def glob_(pattern):
        r = real_glob(pattern)
        seen["globs"].append([os.path.basename(f) for f in r])
        return r

    def crop(self, box=None):
        seen["boxes"].append([int(v) for v in box])
        return real_crop(self, box)

    def save(self, fp, *a, **k):
        seen["saves"].append(os.fspath(fp))
        return real_save(self, fp, *a, **k)

    with tempfile.TemporaryDirectory() as out:
        for s in SPLITS:
            os.makedirs(os.path.join(out, s))
        module.glob, Image.Image.crop, Image.Image.save = glob_, crop, save
        try:
            np.random.seed(1372)
            module.crop_images(inputdir=src_dir, outputdir=out, Ns=list(ns))
        finally:
            module.glob, Image.Image.crop, Image.Image.save = real_glob, real_crop, real_save
        boxes = {s: [] for s in SPLITS}
        names = {s: [] for s in SPLITS}
        crops = {s: [] for s in SPLITS}
        for box, path in zip(seen["boxes"], seen["saves"]):
            split = os.path.basename(os.path.dirname(path))
            boxes[split].append(box)
            names[split].append(os.path.basename(path))
            with Image.open(path) as im:
                crops[split].append(np.asarray(im.convert("L"), np.uint8))
    return seen["globs"], boxes, names, crops


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reference", required=True, help="checkout of the reference repository")
    path = os.path.join(ap.parse_args().reference, "planning-datasets", "preprocess_street_dataset.py")
    spec = importlib.util.spec_from_file_location("preprocess_street_dataset", path)
    module = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(module)
    src_dir = os.path.join(OUT, "sources")
    os.makedirs(src_dir, exist_ok=True)
    for f in globmod.glob(os.path.join(src_dir, "*.png")):
        os.remove(f)
    write_sources(src_dir)
    rec = {}
    for tag, ns in (("default", [160, 20, 40]), ("small", SMALL)):
        globs, boxes, names, crops = run_reference(module, src_dir, ns)
        rec["glob_train"], rec["glob_test"] = np.array(globs[0]), np.array(globs[1])
        for s in SPLITS:
            rec[f"{tag}_boxes_{s}"] = np.array(boxes[s], np.int64).reshape(-1, 4)
            rec[f"{tag}_names_{s}"] = np.array(names[s])
            if tag == "small":
                rec[f"small_crops_{s}"] = np.stack(crops[s])
    np.savez_compressed(os.path.join(OUT, "street.npz"), **rec)
    print({k: v.shape for k, v in rec.items()})


if __name__ == "__main__":
    main()
