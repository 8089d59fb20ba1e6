#!/usr/bin/env python
"""Time of the GPU PNG encoder (nastar_png_encode.cuh + nastar_deflate.cuh; utils.data.encode_pngs) on an H100, with
the card's name and power limit read in the same run, next to Pillow's Image.fromarray(a).save(buf, "PNG") on one
host core.

Workloads (from seeds):
  csm_128      4 000 128x128 street-like crops, the CSM split sizes (3 200 / 400 / 400): 30 synthetic street sources
               (tests/golden/make_golden_street.py's generator), cropped by street_crop_boxes;
  maps_256     1 024 256x256 street-like maps;
  random_2048  64 random 2048x2048 images (each 16 deflate chunks).
Per workload: each of the three kernels alone (CUDA events, median of 3 after warm-up), encode_pngs end to end (host
clock around the call, which returns the files as bytes; warm-up then median of 3), Pillow once per image, and both
total file sizes; 64 of the GPU files, evenly spaced, are checked to decode (Pillow) to their images.  Then make_street_dataset.py's crop step
(decode, resize, crop, encode, write) end to end on the street fixture's sources with the default Ns, against
crop_images' own sequence of Pillow calls (open, convert("L"), resize((256, 256)), crop, save) on one host core.
Prints one JSON object; --out also writes it to a file.  Files go to a temporary directory.

    python tools/png_encode_bench.py [--out profiles/h100_png_encode_bench.json]
"""
import argparse
import io
import json
import os
import shutil
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for _p in (ROOT, os.path.join(ROOT, "neural-astar_b200"), os.path.join(ROOT, "tests"),
           os.path.join(ROOT, "tests", "golden"), os.path.join(ROOT, "tools")):
    if _p not in sys.path:
        sys.path.insert(0, _p)

import numpy as np  # noqa: E402
import torch  # noqa: E402

STREET = os.path.join(ROOT, "tests", "golden", "street")


def workloads():
    """(name, uint8 [B,H,W] NumPy images), built from seeds."""
    from make_golden_street import street_map
    from neural_astar.utils.data import street_crop_boxes

    rng = np.random.RandomState(1234)
    sources = np.stack([street_map(rng, 256, 256) for _ in range(30)])
    boxes = street_crop_boxes([f"s{i}_0_256.png" for i in range(20)], [f"s{i}_2_256.png" for i in range(20, 30)])
    crops = []
    for split in ("train", "validation", "test"):
        b = boxes[split]
        base = 20 if split == "test" else 0
        crops += [sources[base + k, t:t + 128, l:l + 128] for k, l, t in zip(b["source"], b["left"], b["top"])]
    yield "csm_128", np.stack(crops)
    yield "maps_256", np.stack([street_map(rng, 256, 256) for _ in range(1024)])
    yield "random_2048", rng.randint(0, 256, (64, 2048, 2048)).astype(np.uint8)


def kernel_arms(x):
    """Median CUDA-event times (ms) of the three launches of one encode of x (uint8 CUDA [B,H,W])."""
    from labels_bench import timed
    from neural_astar import _native

    B, H, W = x.shape
    n = np.full(B, H * (W + 1), np.int64)
    foff = np.concatenate([[0], np.cumsum(n)[:-1]])
    enc = np.zeros(B, _native.PNG_ENC_DESC_DTYPE)
    enc["pixels"] = x.data_ptr() + np.arange(B, dtype=np.int64) * H * W
    enc["filt_off"], enc["W"], enc["H"] = foff, W, H
    filt = torch.empty((int(n.sum()),), dtype=torch.uint8, device=x.device)
    desc = np.zeros(B, _native.DEFLATE_DESC_DTYPE)
    desc["data"], desc["data_len"], desc["gap"] = filt.data_ptr() + foff, n, _native.png_gaps(B)
    desc["chunk0"] = np.concatenate([[0], np.cumsum(_native.deflate_chunk_counts(n))[:-1]])
    enc_dev = torch.from_numpy(enc.view(np.uint8).copy()).to(x.device)
    desc_dev = torch.from_numpy(desc.view(np.uint8).copy()).to(x.device)
    adler = _native.png_filter(enc, enc_dev, filt)
    out, off, ln, _ = _native.deflate(desc, desc_dev, tail=_native.PNG_ENC_TAIL)
    f_ms, f_tr = timed(lambda: _native.png_filter(enc, enc_dev, filt), 3)
    d_ms, d_tr = timed(lambda: _native.deflate(desc, desc_dev, tail=_native.PNG_ENC_TAIL), 1)
    e_ms, e_tr = timed(lambda: _native.png_finish(enc, enc_dev, off, ln, adler, out), 3)
    return {"filter_ms": f_ms, "filter_ms_trials": f_tr, "deflate_ms": d_ms, "deflate_ms_trials": d_tr,
            "finish_ms": e_ms, "finish_ms_trials": e_tr, "kernels_ms": f_ms + d_ms + e_ms}


def pillow_save(a: np.ndarray) -> bytes:
    from PIL import Image

    buf = io.BytesIO()
    Image.fromarray(a).save(buf, "PNG")
    return buf.getvalue()


def host_crop_images(src_dir, out_dir, Ns=(160, 20, 40)):
    """crop_images' sequence of Pillow calls, in its draw order, on one host core."""
    import glob
    import re

    from PIL import Image

    np.random.seed(1372)
    train, test = glob.glob("%s/*[0,1]_256.png" % src_dir), glob.glob("%s/*2_256.png" % src_dir)
    for split, files, n in (("train", train, Ns[0]), ("validation", train, Ns[1]), ("test", test, Ns[2])):
        os.makedirs(os.path.join(out_dir, split), exist_ok=True)
        for f in files:
            fileid = re.split("_256.png", re.split("/", f)[-1])[0]
            img = Image.open(f).convert("L").resize((256, 256))
            lt = np.random.randint(0, 256 - 128, [n, 2])
            for k, box in enumerate(np.hstack((lt, lt + 128))):
                img.crop(box).save(os.path.join(out_dir, split, "%s_%05d.png" % (fileid, k)))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    from PIL import Image

    import make_street_dataset as msd
    from neural_astar.utils.data import encode_pngs
    from wlabels_bench import power_limit_w

    assert torch.cuda.is_available(), "png_encode_bench measures the GPU kernels: no GPU found"
    torch.set_num_threads(1)
    dev = torch.device("cuda:0")
    out = {"kernels": "nastar::png_filter_kernel, nastar::deflate_kernel, nastar::png_finish_kernel",
           "timing": "kernels: CUDA events, median of 3 after warm-up; encode_pngs: host clock around the call "
                     "(bytes objects returned), warm-up then median of 3; Pillow: one pass, one host core",
           "device": torch.cuda.get_device_name(dev), "power_limit_w": power_limit_w(0),
           "host_arm": "Image.fromarray(a).save(buf, 'PNG') per image (zlib level 6), one host core"}
    for name, imgs in workloads():
        x = torch.from_numpy(imgs).to(dev)
        rec = {"images": int(imgs.shape[0]), "shape": list(imgs.shape[1:]), "raw_bytes": int(imgs.nbytes)}
        rec.update(kernel_arms(x))
        files = encode_pngs(x)
        walls = []
        for _ in range(3):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            files = encode_pngs(x)
            walls.append((time.perf_counter() - t0) * 1e3)
        step = max(1, len(files) // 64)
        for i in range(0, len(files), step):
            with Image.open(io.BytesIO(files[i])) as im:
                assert np.array_equal(np.asarray(im), imgs[i]), (name, i)
        t0 = time.perf_counter()
        pil = [pillow_save(a) for a in imgs]
        host_ms = (time.perf_counter() - t0) * 1e3
        rec.update({"encode_pngs_ms": sorted(walls)[1], "encode_pngs_ms_trials": walls, "pillow_ms": host_ms,
                    "speedup_end_to_end": host_ms / sorted(walls)[1],
                    "gpu_file_bytes": sum(len(f) for f in files), "pillow_file_bytes": sum(len(p) for p in pil)})
        rec["size_ratio_gpu_over_pillow"] = rec["gpu_file_bytes"] / rec["pillow_file_bytes"]
        out[name] = rec
        print(name, json.dumps(rec), flush=True)
        del x, files, pil
        torch.cuda.empty_cache()
    # the crop step of 2_CSM.sh on the fixture's sources, default Ns (640 / 80 / 80 crops)
    src = os.path.join(STREET, "sources")
    train, test = msd.source_files(src)
    tmp = tempfile.mkdtemp(prefix="png_encode_bench_")
    msd.crop_street_maps(train, test, os.path.join(tmp, "warm"))
    walls = []
    for k in range(3):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        msd.crop_street_maps(train, test, os.path.join(tmp, f"gpu{k}"))
        walls.append((time.perf_counter() - t0) * 1e3)
    t0 = time.perf_counter()
    host_crop_images(src, os.path.join(tmp, "host"))
    host_ms = (time.perf_counter() - t0) * 1e3
    n = {s: len(os.listdir(os.path.join(tmp, "host", s))) for s in ("train", "validation", "test")}
    same = all(sorted(os.listdir(os.path.join(tmp, "gpu0", s))) == sorted(os.listdir(os.path.join(tmp, "host", s)))
               for s in n)
    for s in n if same else ():
        for f in os.listdir(os.path.join(tmp, "host", s)):
            with Image.open(os.path.join(tmp, "host", s, f)) as a, Image.open(os.path.join(tmp, "gpu0", s, f)) as b:
                same = same and np.array_equal(np.asarray(a), np.asarray(b))
    out["street_crops"] = {"sources": len(train) + len(test), "crops": n, "same_names_and_pixels": same,
                           "gpu_ms": sorted(walls)[1], "gpu_ms_trials": walls, "host_ms": host_ms,
                           "speedup_end_to_end": host_ms / sorted(walls)[1]}
    print("street_crops", json.dumps(out["street_crops"]), flush=True)
    shutil.rmtree(tmp)
    line = json.dumps(out)
    print(line)
    if args.out:
        with open(args.out, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
