#!/usr/bin/env python
"""Stanford Drone (SDD) samples on the GPU (DESIGN.md §22) against the host route, on seeded synthetic videos at SDD
scale: six scenes of about 1400 x 1900 pixels (SDD's reference images are 1.1 to 2 k on a side), each with a few
hundred mostly straight tracks, giving a few thousand kept samples with crops of about 200 to 2000 pixels.

  kernel       CUDA events around sdd_crops of every kept box (one launch; its descriptor upload included), warm-up
               then median of 20
  gpu e2e      host clock around save_sdd_samples over all videos: host plan, Pillow's JPEG decode and the upload,
               crops, planes, deflate, files on disk; warm-up then median of 3.  Beside it, in the same runs, CUDA
               events around each nastar_b200_deflate launch, and the host clock around the write step alone (crops,
               planes, deflate, files) from plans and scenes made beforehand
  host         the same samples written on one host core the way the generator does it: Pillow crop + resize and
               np.savez_compressed per sample, after the same host plan and JPEG decode; one pass
The two trees are then compared file by file (np.load equal).  The card's name and power limit are read in the same
run.

    python tools/sdd_bench.py [--out f.json] [--tracks 450]
"""
import argparse
import json
import os
import shutil
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "neural-astar_b200"))
sys.path.insert(0, os.path.join(ROOT, "tools"))

import numpy as np  # noqa: E402
import torch  # noqa: E402
from PIL import Image  # noqa: E402

SCENES = [(1424, 1088), (1630, 1948), (1400, 1904), (1422, 1898), (1331, 1962), (1455, 1925)]   # (W, H)
LABELS = ("Pedestrian", "Biker", "Skater", "Car", "Cart", "Bus")


def make_videos(root, n_tracks, seed=0):
    """Seeded scenes (smooth colour fields, blocks, noise) and tracks of 40 to 600 rows: straight walks with jitter,
    some lost rows; a tenth of them zigzag (rejected by the length ratio)."""
    rng = np.random.RandomState(seed)
    videos = []
    for s, (W, H) in enumerate(SCENES):
        d = os.path.join(root, f"scene{s}", "video0")
        os.makedirs(d)
        low = rng.randint(0, 256, (H // 40, W // 40, 3)).astype(np.uint8)
        img = np.asarray(Image.fromarray(low, "RGB").resize((W, H), Image.BICUBIC)).astype(np.int16)
        for _ in range(60):
            x, y = rng.randint(0, W), rng.randint(0, H)
            img[y:y + rng.randint(20, 200), x:x + rng.randint(20, 200)] = rng.randint(0, 256, 3)
        img = np.clip(img + rng.randint(-12, 13, img.shape), 0, 255).astype(np.uint8)
        Image.fromarray(img, "RGB").save(os.path.join(d, "reference.jpg"), quality=90)
        lines = []
        for t in range(n_tracks):
            n = int(rng.randint(40, 600))
            length = rng.uniform(150, 1900)
            ang = rng.uniform(0, 2 * np.pi)
            p0 = np.array([rng.uniform(0, W), rng.uniform(0, H)])
            step = length / n * np.array([np.cos(ang), np.sin(ang)])
            pts = p0 + np.arange(n)[:, None] * step + rng.normal(0, 1.5, (n, 2))
            if t % 10 == 0:
                pts[:, 1] += 80 * (np.arange(n) % 30 < 15)
            lost = (rng.rand(n) < 0.01).astype(int)
            w, h = int(rng.randint(10, 40)), int(rng.randint(10, 40))
            for i, (cx, cy) in enumerate(pts):
                x0, y0 = int(cx - w / 2), int(cy - h / 2)
                lines.append(f'{t} {x0} {y0} {x0 + w} {y0 + h} {i} {lost[i]} {int(rng.rand() < 0.2)} 0 '
                             f'"{LABELS[t % 6]}"')
        with open(os.path.join(d, "annotations.txt"), "w") as f:
            f.write("\n".join(lines) + "\n")
        videos.append(d)
    return videos


def host_route(videos, save_dir, W, ratio, mms, max_step):
    """The generator's per-sample work on one host core, after the same host plan."""
    from neural_astar.utils.data import sdd_sample_plan

    rng = np.random.RandomState(0)
    n = 0
    for v in videos:
        p = sdd_sample_plan(v, W, ratio, mms, max_step, rng)
        out = os.path.join(save_dir, p["scene"], p["video"])
        os.makedirs(out, exist_ok=True)
        ref = Image.open(os.path.join(v, "reference.jpg"))
        for k, name in enumerate(p["name"]):
            planes = np.zeros((3, W, W))
            planes[0][tuple(p["start"][k])] = 1
            planes[1][tuple(p["goal"][k])] = 1
            planes[2][p["cells"][k][:, 0], p["cells"][k][:, 1]] = 1
            image = np.array(ref.crop(tuple(int(b) for b in p["box"][k])).resize((W, W)))
            np.savez_compressed(os.path.join(out, name), image=image, start_image=planes[0], goal_image=planes[1],
                                traj_image=planes[2], traj=p["traj"][k], label=p["label"][k],
                                length_ratio=p["length_ratio"][k])
            n += 1
    return n


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--tracks", type=int, default=450, help="tracks per scene")
    args = ap.parse_args()
    from neural_astar import _native
    from neural_astar.utils.data import _sdd_scene, _write_sdd_samples, save_sdd_samples, sdd_crops, \
        sdd_sample_plan
    from wlabels_bench import power_limit_w

    assert torch.cuda.is_available(), "sdd_bench needs a GPU"
    dev = torch.device("cuda:0")
    W, ratio, mms, max_step = 64, 0.5, 128, 300
    tmp = tempfile.mkdtemp(prefix="sdd_bench_")
    try:
        videos = make_videos(os.path.join(tmp, "original"), args.tracks)
        t0 = time.perf_counter()
        rng = np.random.RandomState(0)
        plans = [sdd_sample_plan(v, W, ratio, mms, max_step, rng) for v in videos]
        plan_s = time.perf_counter() - t0
        t0 = time.perf_counter()
        scenes = [_sdd_scene(v, dev) for v in videos]
        torch.cuda.synchronize()
        decode_s = time.perf_counter() - t0
        boxes = np.concatenate([p["box"] for p in plans])
        src = np.concatenate([np.full(len(p["name"]), i) for i, p in enumerate(plans)])
        sides = np.maximum(boxes[:, 2] - boxes[:, 0], boxes[:, 3] - boxes[:, 1])
        n0 = _native.launch_count()
        sdd_crops(scenes, boxes, W, src)
        launches = _native.launch_count() - n0
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
        kernel_ms = []
        for _ in range(20):
            ev[0].record()
            sdd_crops(scenes, boxes, W, src)
            ev[1].record()
            torch.cuda.synchronize()
            kernel_ms.append(ev[0].elapsed_time(ev[1]))
        write_s = []
        for r in range(4):
            out = os.path.join(tmp, f"write{r}")
            batch = [(p, s, os.path.join(out, p["scene"], p["video"])) for p, s in zip(plans, scenes)]
            for _, _, d in batch:
                os.makedirs(d)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            _write_sdd_samples(batch, W, dev)
            write_s.append(time.perf_counter() - t0)
            shutil.rmtree(out)
        del scenes, batch
        real_deflate, deflate_ev = _native.deflate, []

        def timed_deflate(*a, **k):
            e = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
            e[0].record()
            r = real_deflate(*a, **k)
            e[1].record()
            deflate_ev.append(e)
            return r

        _native.deflate = timed_deflate
        e2e, deflate_ms = [], []
        for r in range(4):
            out = os.path.join(tmp, f"gpu{r}")
            torch.cuda.synchronize()
            deflate_ev.clear()
            t0 = time.perf_counter()
            n_gpu = save_sdd_samples(videos, out, W, ratio, mms, max_step, rng=np.random.RandomState(0), device=dev)
            e2e.append(time.perf_counter() - t0)
            deflate_ms.append(sum(a.elapsed_time(b) for a, b in deflate_ev))
            if r:
                shutil.rmtree(out)
        _native.deflate = real_deflate
        t0 = time.perf_counter()
        n_host = host_route(videos, os.path.join(tmp, "host"), W, ratio, mms, max_step)
        host_s = time.perf_counter() - t0
        assert n_gpu == n_host == len(boxes), (n_gpu, n_host, len(boxes))
        mismatches, gpu_bytes, host_bytes = 0, 0, 0
        for p in plans:
            for name in p["name"]:
                a = os.path.join(tmp, "gpu0", p["scene"], p["video"], name)
                b = os.path.join(tmp, "host", p["scene"], p["video"], name)
                gpu_bytes, host_bytes = gpu_bytes + os.path.getsize(a), host_bytes + os.path.getsize(b)
                za, zb = np.load(a), np.load(b)
                mismatches += int(za.files != zb.files or any(
                    za[k].dtype != zb[k].dtype or not np.array_equal(za[k], zb[k]) for k in zb.files))
        rec = {
            "device": torch.cuda.get_device_name(dev), "power_limit_w": power_limit_w(0),
            "workload": {"scenes_wh": SCENES, "tracks_per_scene": args.tracks, "samples": int(len(boxes)),
                         "W": W, "min_len_ratio": ratio, "min_max_size": mms, "max_step": max_step,
                         "crop_side_px": {"min": int(sides.min()), "median": float(np.median(sides)),
                                          "max": int(sides.max())}},
            "timing": "kernel: CUDA events around sdd_crops (descriptor upload + one launch), warm-up then median of 20; "
                      "gpu_e2e and write_step: host clock, warm-up then median of 3; deflate: CUDA events around its "
                      "launches in the e2e runs, summed per run; host: one pass, one host core",
            "kernel_launches_per_sdd_crops": launches,
            "kernel_ms": float(np.median(kernel_ms)), "kernel_ms_all": kernel_ms,
            "host_plan_s": plan_s, "host_jpeg_decode_upload_s": decode_s,
            "gpu_e2e_s": float(np.median(e2e[1:])), "gpu_e2e_s_all": e2e,
            "deflate_kernel_ms_per_e2e": float(np.median(deflate_ms[1:])), "deflate_kernel_ms_all": deflate_ms,
            "write_step_s": float(np.median(write_s[1:])), "write_step_s_all": write_s,
            "host_one_core_s": host_s,
            "files_equal": mismatches == 0, "file_mismatches": mismatches,
            "gpu_bytes": gpu_bytes, "host_bytes": host_bytes,
        }
    finally:
        shutil.rmtree(tmp, ignore_errors=True)
    line = json.dumps(rec)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
