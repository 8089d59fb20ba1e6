#!/usr/bin/env python
"""Reading the Stanford Drone samples onto the GPU and scoring paths by the Chamfer distance (DESIGN.md §23), against
the host route, on the seeded synthetic videos of sdd_bench.py (six scenes, about 4 700 samples of 7 members each):

  read      host clock around DeviceSDDDataset(tree) (file reads, host zip parse, one upload, one inflate launch,
            planes built on the device) against np.load of every file, the same arrays built with NumPy and uploaded;
            the files are read once before timing (page cache warm); warm-up then median of 5, alternating
  chamfer   CUDA events around chamfer_distance of VanillaAstar paths on all-passable maps against traj_images, for
            batches of 100 and 4 096 64 x 64 maps (the dataset's samples, tiled), warm-up then median of 20, against
            the scipy oracle (scipy.ndimage.distance_transform_edt per map and direction) on one host core, one pass;
            the two agree to 1e-12 relative
The card's name and power limit are read in the same run.

    python tools/sdd_read_bench.py [--out f.json] [--tracks 450]
"""
import argparse
import glob
import json
import os
import shutil
import statistics
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "neural-astar_b200"))
sys.path.insert(0, os.path.join(ROOT, "tools"))

import numpy as np  # noqa: E402
import torch  # noqa: E402
from scipy import ndimage  # noqa: E402


def host_read(files, dev):
    zs = [np.load(f) for f in files]
    arrays = [np.stack([(z["image"].transpose(2, 0, 1) / 255.0).astype(np.float32) for z in zs])]
    arrays += [np.stack([z[k] for z in zs])[:, None].astype(np.float32)
               for k in ("start_image", "goal_image", "traj_image")]
    arrays += [np.stack([z["label"] for z in zs]), np.stack([z["length_ratio"] for z in zs]),
               np.concatenate([z["traj"] for z in zs])]
    out = [torch.from_numpy(a).to(dev) for a in arrays]
    torch.cuda.synchronize(dev)
    return out


def scipy_chamfer(a, b):
    out = np.full((len(a), 2), np.nan)
    for k, (x, y) in enumerate(zip(a != 0, b != 0)):
        if x.any() and y.any():
            out[k] = ndimage.distance_transform_edt(~y)[x].mean(), ndimage.distance_transform_edt(~x)[y].mean()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--tracks", type=int, default=450, help="tracks per scene")
    args = ap.parse_args()
    from neural_astar.planner import VanillaAstar
    from neural_astar.utils.data import DeviceSDDDataset, save_sdd_samples
    from neural_astar.utils.training import chamfer_distance, chamfer_distances
    from sdd_bench import make_videos
    from wlabels_bench import power_limit_w

    assert torch.cuda.is_available(), "sdd_read_bench needs a GPU"
    dev = torch.device("cuda:0")
    tmp = tempfile.mkdtemp(prefix="sdd_read_bench_")
    try:
        videos = make_videos(os.path.join(tmp, "original"), args.tracks)
        tree = os.path.join(tmp, "samples")
        n = save_sdd_samples(videos, tree, rng=np.random.RandomState(0), device=dev)
        files = sorted(glob.glob(os.path.join(tree, "*", "*", "*.npz")))
        total_bytes = sum(os.path.getsize(f) for f in files)
        ds = DeviceSDDDataset(tree, device=dev)
        host = host_read(files, dev)
        assert torch.equal(ds.map_designs, host[0]) and torch.equal(ds.traj_images, host[3])
        gpu_s, host_s = [], []
        for _ in range(5):
            t0 = time.perf_counter()
            DeviceSDDDataset(tree, device=dev)
            torch.cuda.synchronize(dev)
            gpu_s.append(time.perf_counter() - t0)
            t0 = time.perf_counter()
            host_read(files, dev)
            host_s.append(time.perf_counter() - t0)
        rec = {"bench": "sdd_read", "device": torch.cuda.get_device_name(dev), "power_limit_w": power_limit_w(0),
               "samples": n, "files_bytes": total_bytes,
               "read": {"gpu_dataset_s": statistics.median(gpu_s), "host_np_load_upload_s": statistics.median(host_s)}}
        paths = VanillaAstar().to(dev)(torch.ones_like(ds.start_maps), ds.start_maps, ds.goal_maps).paths
        rec["chamfer"] = {}
        for B in (100, 4096):
            idx = torch.arange(B, device=dev) % len(ds)
            a, b = paths[idx], ds.traj_images[idx]
            got = chamfer_distances(a, b)
            ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
            ms = []
            for _ in range(23):
                ev[0].record()
                chamfer_distance(a, b)
                ev[1].record()
                ev[1].synchronize()
                ms.append(ev[0].elapsed_time(ev[1]))
            an, bn = a.cpu().numpy()[:, 0], b.cpu().numpy()[:, 0]
            t0 = time.perf_counter()
            want = scipy_chamfer(an, bn)
            scipy_s = time.perf_counter() - t0
            np.testing.assert_allclose(got.cpu().numpy(), want, rtol=1e-12, atol=0)
            rec["chamfer"][str(B)] = {"gpu_ms": statistics.median(ms[3:]), "scipy_one_core_ms": scipy_s * 1e3}
    finally:
        shutil.rmtree(tmp, ignore_errors=True)
    line = json.dumps(rec)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
