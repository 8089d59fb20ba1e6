#!/usr/bin/env python
"""planning-datasets' generate_sdd_instances.py (3_SDD.sh) on the GPU: the Stanford Drone planning samples of every
`<input-path>/*/video*` directory, in sorted order after seed 0, written by save_sdd_samples (DESIGN.md §22) to
`<save-dir>/s%03d_%0.1f_%d_%d/<scene>/<video>/%08d_%02d.npz` (size, min-len-ratio, min-max-size, max-step).

    python tools/make_sdd_dataset.py [--input-path data/sdd/original] [--save-dir data/sdd] [--size 64] ...
"""
import argparse
import glob
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "neural-astar_b200"))

import numpy as np  # noqa: E402


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--size", "-w", type=int, default=64)
    ap.add_argument("--min-len-ratio", "-ml", type=float, default=0.5)
    ap.add_argument("--min-max-size", "-mm", type=int, default=128)
    ap.add_argument("--max-step", "-ms", type=int, default=300)
    ap.add_argument("--save-dir", "-s", type=str, default="data/sdd")
    ap.add_argument("--input-path", type=str, default="data/sdd/original")
    args = ap.parse_args(argv)
    from neural_astar.utils.data import save_sdd_samples

    W, ratio, mms, max_step = int(args.size), float(args.min_len_ratio), int(args.min_max_size), int(args.max_step)
    save_dir = "%s/s%03d_%0.1f_%d_%d" % (args.save_dir, W, ratio, mms, max_step)
    videos = sorted(glob.glob(os.path.join(args.input_path, "*", "video*")))
    if not videos:
        raise SystemExit(f"no video directories match {os.path.join(args.input_path, '*', 'video*')}")
    t0 = time.perf_counter()
    n = save_sdd_samples(videos, save_dir, W, ratio, mms, max_step, rng=np.random.RandomState(0))
    print(f"{n} samples from {len(videos)} videos in {time.perf_counter() - t0:.2f} s -> {save_dir}")
    return save_dir


if __name__ == "__main__":
    main()
