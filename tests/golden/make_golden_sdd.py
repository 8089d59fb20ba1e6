#!/usr/bin/env python
"""Fixture for the Stanford Drone (SDD) planning samples (tests/golden/sdd/): synthetic videos and what the
reference's own create_sample_from_dataset (planning-datasets/planning_datasets_utils/SDD.py) writes for them.

  original/<scene>/video<k>/   reference.jpg (seeded smooth scenes with blocks: plaza 720x540, tower 540x960,
                               wide 2100x360) and annotations.txt (tracks built below to cover every rule: the three
                               rejections, several lost runs per id including a one-row run, occluded visible rows,
                               ids whose rows are not contiguous, tracks longer than max_step (some then rejected),
                               ROIs past the right and bottom edges (min_loc branch) and the left and top edges
                               (the other, max_loc clipped in several), crop coordinates ending in .5 below and above
                               zero, all six labels); plaza/video2 keeps no sample
  sdd.npz      videos                  the video directories in sorted glob order
               scene, scene_sha256     each reference.jpg and the SHA-256 of its Pillow-decoded pixels
               <tag>_dirs              every directory the run created under save_dir
               <tag>_files             the files it wrote, "<scene>/<video>/<name>", in write order
               <tag>_roi               the float64 box each sample passed to Image.crop, [K, 4]
               <tag>_image             uint8 [K, W, W, 3]
               <tag>_planes            start_image, goal_image, traj_image as uint8 0/1, [K, 3, W, W]
               <tag>_traj, <tag>_traj_len   every traj, concatenated [sum n, 2], and each one's n
               <tag>_label, <tag>_length_ratio
               <tag>_dtypes            "member dtype ndim" of the members of every file (all files agree)
               with <tag> "default" (W, min_len_ratio, min_max_size, max_step = 64, 0.5, 128, 300: the script's
               defaults) and "small" (32, 0.3, 64, 40), each run after np.random.seed(0) over the videos in order

    python tests/golden/make_golden_sdd.py --reference PATH   # PATH: a checkout of the reference repository
"""
import argparse
import glob as globmod
import hashlib
import importlib.util
import os
import shutil
import sys
import tempfile

import numpy as np
from PIL import Image

HERE = os.path.dirname(os.path.abspath(__file__))
OUT = os.path.join(HERE, "sdd")
PARAMS = {"default": (64, 0.5, 128, 300), "small": (32, 0.3, 64, 40)}
LABELS = ("Pedestrian", "Biker", "Skater", "Car", "Cart", "Bus")
SCENES = {"plaza": (720, 540), "tower": (540, 960), "wide": (2100, 360)}


def scene_image(rng, W, H):
    """Smooth colour fields with a few flat blocks and lines: small as JPEG, with detail the resize must get right."""
    low = rng.randint(0, 256, (max(H // 60, 2), max(W // 60, 2), 3)).astype(np.uint8)
    img = np.asarray(Image.fromarray(low, "RGB").resize((W, H), Image.BILINEAR)).copy()
    for _ in range(12):
        x, y = rng.randint(0, W), rng.randint(0, H)
        img[y:y + rng.randint(10, 80), x:x + rng.randint(10, 80)] = rng.randint(0, 256, 3)
    for _ in range(4):
        y = rng.randint(0, H)
        img[y:y + 3] = 255
    return img


class Track:
    """Rows of one id: box centres along `points` (each row one frame), box size (w, h)."""

    def __init__(self, tid, label, points, w=15, h=21, lost=None, occluded=None):
        self.tid, self.label = tid, label
        self.points = np.asarray(points, np.float64)
        n = len(self.points)
        self.w, self.h = w, h
        self.lost = np.zeros(n, int) if lost is None else np.asarray(lost, int)
        self.occluded = np.zeros(n, int) if occluded is None else np.asarray(occluded, int)

    def rows(self, frame0=0):
        out = []
        for i, (cx, cy) in enumerate(self.points):
            x0, y0 = int(np.floor(cx - self.w / 2)), int(np.floor(cy - self.h / 2))
            out.append(f'{self.tid} {x0} {y0} {x0 + self.w} {y0 + self.h} {frame0 + i} {self.lost[i]} '
                       f'{self.occluded[i]} 0 "{self.label}"')
        return out


def line(p0, p1, n):
    t = np.linspace(0, 1, n)[:, None]
    return np.round(np.asarray(p0) * (1 - t) + np.asarray(p1) * t)


def zigzag(p0, p1, n, amp):
    pts = line(p0, p1, n)
    pts[:, 1] += amp * (np.arange(n) % 20 < 10)
    return pts


def tracks_for(scene, video, rng):
    W, H = SCENES[scene]
    T = []
    lab = lambda k: LABELS[k % len(LABELS)]
    if scene == "plaza" and video == 0:
        # straight tracks inside (kept), near each edge (ROIs past it), .5 coordinates on both sides of zero
        T.append(Track(1, lab(0), line((200, 200), (400, 260), 120)))
        T.append(Track(2, lab(1), line((560, 250), (712, 300), 90), w=16))   # min branch, past the right edge
        T.append(Track(3, lab(2), line((300, 380), (360, 533), 80), h=22))   # min branch, past the bottom edge
        T.append(Track(4, lab(3), line((20, 250), (180, 300), 90), w=16))    # else branch, min_loc x = -29.5
        T.append(Track(5, lab(4), line((300, 29), (460, 70), 90), h=16))     # else branch, min_loc y = -20.5
        T.append(Track(6, lab(5), line((600, 10), (715, 150), 70), w=15, h=15))   # else branch, clipped max_loc
        T.append(Track(7, lab(0), line((61, 120), (240, 150), 70), w=16))    # min branch, min_loc x = 11.5
        T.append(Track(8, lab(1), line((70, 60), (260, 90), 70), w=16, h=16))   # min branch, x0 10.5, y0 -> .5
        # several lost runs, one of one row; occluded visible rows
        n = 160
        lost = np.zeros(n, int)
        lost[50:60] = 1
        lost[61:70] = 1
        lost[150:155] = 1
        occ = (rng.rand(n) < 0.3).astype(int)
        T.append(Track(9, lab(2), line((100, 420), (600, 480), n), lost=lost, occluded=occ))
        # rejections: closed loop (sg_length 0), zigzag (low ratio), small extent
        loop = np.concatenate([line((400, 100), (500, 100), 40), line((500, 100), (400, 100), 40)])
        T.append(Track(10, lab(3), loop))
        T.append(Track(11, lab(4), zigzag((150, 300), (300, 300), 120, 40)))
        T.append(Track(12, lab(5), line((500, 400), (590, 420), 60)))   # extent 90: kept only by "small"
    elif scene == "plaza" and video == 1:
        # long tracks: draws for both parameter sets, one then rejected as a zigzag
        T.append(Track(20, lab(1), line((50, 300), (650, 200), 420), occluded=(rng.rand(420) < 0.1).astype(int)))
        T.append(Track(21, lab(2), zigzag((100, 100), (600, 140), 360, 60)))
        T.append(Track(22, lab(3), line((600, 500), (150, 380), 330)))
        T.append(Track(23, lab(5), line((360, 50), (380, 500), 55)))
    elif scene == "plaza" and video == 2:
        T.append(Track(30, lab(0), np.tile([[300.0, 300.0]], (30, 1))))   # stationary: sg_length 0
        T.append(Track(31, lab(1), line((100, 100), (130, 110), 20)))      # extent 30
    elif scene == "tower":
        T.append(Track(40, lab(4), line((270, 100), (300, 900), 300)))
        T.append(Track(41, lab(5), line((30, 500), (500, 700), 200), w=17))   # else branch, past the left edge
        T.append(Track(42, lab(0), line((100, 930), (400, 955), 150)))        # past the bottom
        lost = np.zeros(100, int)
        lost[::7] = 1
        T.append(Track(43, lab(1), line((200, 300), (450, 420), 100), lost=lost))
        T.append(Track(44, lab(2), line((480, 20), (530, 300), 100), w=19, h=13))
    else:   # wide
        T.append(Track(50, lab(3), line((100, 180), (2000, 200), 500)))
        T.append(Track(51, lab(4), line((1900, 40), (2095, 330), 120)))
        T.append(Track(52, lab(5), line((1000, 300), (1400, 355), 200)))
        T.append(Track(53, lab(0), line((5, 20), (300, 60), 120), w=15, h=17))
    return T


def write_video(path, scene, video, rng):
    os.makedirs(path, exist_ok=True)
    W, H = SCENES[scene]
    Image.fromarray(scene_image(rng, W, H), "RGB").save(os.path.join(path, "reference.jpg"), quality=85)
    tracks = tracks_for(scene, video, rng)
    blocks = [t.rows() for t in tracks]
    lines = []
    if len(blocks) > 2:   # ids whose rows are not contiguous: the first id's second half after the second id
        a = blocks[0]
        lines = a[:len(a) // 2] + blocks[1] + a[len(a) // 2:] + sum(blocks[2:], [])
    else:
        lines = sum(blocks, [])
    with open(os.path.join(path, "annotations.txt"), "w") as f:
        f.write("\n".join(lines) + "\n")


def run_reference(module, videos, W, ratio, mms, max_step):
    rois = []
    real_crop = Image.Image.crop

    def crop(self, box=None):
        rois.append([float(v) for v in box])
        return real_crop(self, box)

    rec = {"files": [], "image": [], "planes": [], "traj": [], "label": [], "length_ratio": [], "dtypes": None}
    with tempfile.TemporaryDirectory() as save:
        Image.Image.crop = crop
        written = []
        real_savez = np.savez_compressed

        def savez(path, **kw):
            written.append(path)
            return real_savez(path, **kw)

        module.np.savez_compressed = savez
        try:
            np.random.seed(0)
            for v in videos:
                module.create_sample_from_dataset(v, save, W, ratio, mms, max_step)
        finally:
            Image.Image.crop = real_crop
            module.np.savez_compressed = real_savez
        rec["dirs"] = sorted(os.path.relpath(d, save) for d, _, _ in os.walk(save) if d != save)
        for p in written:
            z = np.load(p)
            dt = [f"{k} {z[k].dtype.str} {z[k].ndim}" for k in z.files]
            assert rec["dtypes"] in (None, dt), (rec["dtypes"], dt)
            rec["dtypes"] = dt
            rec["files"].append(os.path.relpath(p, save))
            rec["image"].append(z["image"])
            planes = np.stack([z["start_image"], z["goal_image"], z["traj_image"]])
            assert set(np.unique(planes)) <= {0.0, 1.0}
            rec["planes"].append(planes.astype(np.uint8))
            rec["traj"].append(z["traj"])
            rec["label"].append(int(z["label"]))
            rec["length_ratio"].append(float(z["length_ratio"]))
    assert len(rois) == len(rec["files"])
    rec["roi"] = np.array(rois, np.float64).reshape(-1, 4)
    return rec


def check_coverage(rec, W):
    roi = rec["roi"]
    half = roi - np.floor(roi) == 0.5
    assert (half & (roi < 0)).any() and (half & (roi > 0)).any(), "crop coordinates ending in .5 on both sides of 0"
    assert (roi[:, 0] < 0).any() and (roi[:, 1] < 0).any(), "ROIs past the left and top edges"
    assert set(rec["label"]) == set(range(6)), "all six labels"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reference", required=True, help="checkout of the reference repository")
    pd_root = os.path.join(ap.parse_args().reference, "planning-datasets")
    sys.path.insert(0, pd_root)
    spec = importlib.util.spec_from_file_location("sdd_reference", os.path.join(pd_root, "planning_datasets_utils",
                                                                                "SDD.py"))
    module = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(module)
    orig = os.path.join(OUT, "original")
    shutil.rmtree(orig, ignore_errors=True)
    rng = np.random.RandomState(2026)
    for scene, video in (("plaza", 0), ("plaza", 1), ("plaza", 2), ("tower", 0), ("wide", 0)):
        write_video(os.path.join(orig, scene, f"video{video}"), scene, video, rng)
    videos = sorted(globmod.glob(os.path.join(orig, "*", "video*")))
    out = {"videos": np.array([os.path.relpath(v, OUT) for v in videos])}
    scenes = sorted(globmod.glob(os.path.join(orig, "*", "video*", "reference.jpg")))
    out["scene"] = np.array([os.path.relpath(s, OUT) for s in scenes])
    out["scene_sha256"] = np.array([hashlib.sha256(np.asarray(Image.open(s)).tobytes()).hexdigest() for s in scenes])
    for tag, (W, ratio, mms, max_step) in PARAMS.items():
        rec = run_reference(module, videos, W, ratio, mms, max_step)
        if tag == "default":
            check_coverage(rec, W)
        out[f"{tag}_dirs"] = np.array(rec["dirs"])
        out[f"{tag}_files"] = np.array(rec["files"])
        out[f"{tag}_roi"] = rec["roi"]
        out[f"{tag}_image"] = np.stack(rec["image"])
        out[f"{tag}_planes"] = np.stack(rec["planes"])
        out[f"{tag}_traj"] = np.concatenate(rec["traj"])
        out[f"{tag}_traj_len"] = np.array([len(t) for t in rec["traj"]], np.int64)
        out[f"{tag}_label"] = np.array(rec["label"], np.int64)
        out[f"{tag}_length_ratio"] = np.array(rec["length_ratio"], np.float64)
        out[f"{tag}_dtypes"] = np.array(rec["dtypes"])
        print(tag, len(rec["files"]), "samples;", "dirs", rec["dirs"])
    np.savez_compressed(os.path.join(OUT, "sdd.npz"), **out)


if __name__ == "__main__":
    main()
