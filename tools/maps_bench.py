#!/usr/bin/env python
"""Throughput of the map kernel (nastar_maps.cuh; neural_astar.utils.data.maps_from_images) on an H100, with the card's
name and power limit read in the same run, next to the host recipe (Pillow resize + NumPy Otsu) on one host core and
the host PNG decode that both need.

Workloads (decoded uint8 images):
  mp_8000_201to32      8000 201x201 sources -> 32x32, the size of the 8 MP families' 8000 images: the 215 decoded
                       sources of tests/golden/maps/sources.npz, cycled;
  mp_1024_201to256     1024 of those sources -> 256x256;
  random_256_1024to64  256 random 1024x1024 images -> 64x64 (seed 1024), street-photo sized.
Per workload: the kernel alone (images device-resident) and upload + kernel (images in host memory), CUDA events
around back-to-back calls, median of 3 trials.  The host arm times PIL's Image.resize + the NumPy Otsu of
tests/maps_oracle.py + the threshold per image over a subset, host clock.  The decode arm times Image.open +
convert("L") of PNGs that PIL encodes from the same sources in memory (decode is host work either way).
Prints one JSON object; --out also writes it to a file.

    python tools/maps_bench.py [--out profiles/h100_maps_bench.json]
"""
import argparse
import io
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for _p in (ROOT, os.path.join(ROOT, "neural-astar_b200"), os.path.join(ROOT, "tests"), os.path.join(ROOT, "tools")):
    if _p not in sys.path:
        sys.path.insert(0, _p)

import numpy as np  # noqa: E402
import torch  # noqa: E402

from labels_bench import timed  # noqa: E402
from wlabels_bench import power_limit_w  # noqa: E402


def workloads():
    with np.load(os.path.join(ROOT, "tests", "golden", "maps", "sources.npz")) as z:
        src = np.concatenate([z["mp_images"], z["tiled_images"]])
    yield "mp_8000_201to32", src[np.arange(8000) % len(src)], 32, 400
    yield "mp_1024_201to256", src[np.arange(1024) % len(src)], 256, 100
    yield "random_256_1024to64", np.random.RandomState(1024).randint(0, 256, (256, 1024, 1024)).astype(np.uint8), 64, 20


def host_ms_per_image(images, size, n):
    from PIL import Image

    import maps_oracle as mo

    def one(img):
        r = np.asarray(Image.fromarray(img, "L").resize((size, size)), dtype=np.float32)
        th, _ = mo.otsu(r)
        return (r > th).astype(np.float32)

    one(images[0])
    t0 = time.perf_counter()
    for img in images[:n]:
        one(img)
    return (time.perf_counter() - t0) * 1e3 / min(n, len(images))


def decode_ms_per_image(images, n):
    from PIL import Image

    blobs = []
    for img in images[:n]:
        b = io.BytesIO()
        Image.fromarray(img, "L").save(b, format="PNG")
        blobs.append(b.getvalue())
    t0 = time.perf_counter()
    for b in blobs:
        np.asarray(Image.open(io.BytesIO(b)).convert("L"), dtype=np.uint8)
    return (time.perf_counter() - t0) * 1e3 / len(blobs), float(np.mean([len(b) for b in blobs]))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    from neural_astar import _native
    from neural_astar.utils.data import maps_from_images

    assert torch.cuda.is_available(), "maps_bench measures the GPU kernel: no GPU found"
    torch.set_num_threads(1)
    dev = torch.device("cuda:0")
    out = {"kernel": "nastar::maps_from_images_kernel (bicubic resize + Otsu + threshold, one CTA per image)",
           "timing": "CUDA events around back-to-back calls, median of 3 trials",
           "device": torch.cuda.get_device_name(dev), "power_limit_w": power_limit_w(0),
           "host_arm": "PIL Image.resize + NumPy Otsu (tests/maps_oracle.py otsu) + threshold per image, one host "
                       "core, host clock over the first images of the workload",
           "decode_arm": "Image.open + convert('L') of in-memory PNGs that PIL encoded from the same images, one host "
                         "core"}
    for name, imgs, size, n_host in workloads():
        B, H0, W0 = imgs.shape
        x = torch.from_numpy(imgs).to(dev)
        reps = 10 if B * H0 * W0 < 2 ** 30 else 3
        k_ms, k_trials = timed(lambda: _native.maps_from_images(x, size, size), reps)
        pinned = torch.from_numpy(imgs).pin_memory()
        u_ms, _ = timed(lambda: maps_from_images(pinned.to(dev, non_blocking=True), size), reps)
        host = host_ms_per_image(imgs, size, n_host)
        dec, png_bytes = decode_ms_per_image(imgs, n_host)
        out[name] = {"images": B, "source": f"{H0}x{W0}", "target": f"{size}x{size}", "kernel_ms": k_ms,
                     "kernel_ms_trials": k_trials, "kernel_images_per_s": B / (k_ms * 1e-3),
                     "upload_plus_kernel_ms": u_ms,
                     "host_resize_otsu": {"images": min(n_host, B), "ms_per_image": host, "ms_all": host * B},
                     "host_png_decode": {"images": min(n_host, B), "ms_per_image": dec, "ms_all": dec * B,
                                         "png_bytes_mean": png_bytes},
                     "speedup_kernel_vs_host_resize_otsu": host * B / k_ms}
        del x, pinned
    line = json.dumps(out)
    print(line)
    if args.out:
        with open(args.out, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
