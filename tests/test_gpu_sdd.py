"""GPU tests of the Stanford Drone (SDD) samples: sdd_crops (nastar_b200_crop_resize_rgb) equals Pillow's
crop(box).resize(size) bit for bit; tools/make_sdd_dataset.py on the fixture videos (tests/golden/sdd/) writes the
tree, names and arrays the reference's create_sample_from_dataset wrote; the many-files .npz writer's archives load
equal to np.savez_compressed's."""
import hashlib
import io
import os
import sys
import zipfile

import numpy as np
import pytest
import torch
from PIL import Image

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SDD = os.path.join(ROOT, "tests", "golden", "sdd")
PARAMS = {"default": (64, 0.5, 128, 300), "small": (32, 0.3, 64, 40)}


@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    return torch.device("cuda:0")


def boxes_for(W, H, Wo, Ho):
    return [
        (10, 20, min(W, 300), min(H, 250)),                       # inside
        (-40, 10, 200, min(H, 200)), (10, -55, 200, 150),          # past the left, top edge
        (W - 100, 10, W + 37, min(H, 200)), (5, H - 50, 180, H + 61),   # past the right, bottom edge
        (-100, -100, W + 100, H + 100),                            # past all four
        (W + 10, 5, W + 200, 190), (-300, -300, -10, -10),         # entirely outside: all zero
        (5, 5, 6, 6), (3, 0, 4, H), (0, 7, W, 8),                  # one pixel, one column, one row
        (7, 9, 7 + Wo, 9 + 101), (-3, 4, 120, 4 + Ho),             # already Wo wide / Ho high: one pass skipped
        (11, 13, 11 + Wo, 13 + Ho),                                # already Wo x Ho: a copy
        (10, 10, 30, 25),                                          # upscaling
        (-50, -400, W + 50, H + 400),                              # sides beyond the source
    ]


def pillow(src, box, Wo, Ho):
    return np.array(Image.fromarray(src, "RGB").crop(box).resize((Wo, Ho)))


@pytest.mark.parametrize("Wo,Ho", [(64, 64), (48, 40), (7, 130)])
def test_crops_equal_pillow(dev, Wo, Ho):
    from neural_astar import _native
    from neural_astar.utils.data import sdd_crops

    rng = np.random.RandomState(Wo * 1000 + Ho)
    shapes = [(540, 720), (333, 517), (300, 2101), (2050, 97)]   # odd sides, sides above 2048
    srcs = [rng.randint(0, 256, (H, W, 3)).astype(np.uint8) for H, W in shapes]
    # smooth regions too, where rounding at the clip edges matters less than the weights' exact values
    srcs[0][:, :360] = np.linspace(0, 255, 360).astype(np.uint8)[None, :, None]
    boxes, src = [], []
    for i, (H, W) in enumerate(shapes):
        b = boxes_for(W, H, Wo, Ho)
        boxes += b
        src += [i] * len(b)
    scenes = [torch.from_numpy(s).to(dev) for s in srcs]
    n0 = _native.launch_count()
    got = sdd_crops(scenes, boxes, (Wo, Ho), src).cpu().numpy()
    assert _native.launch_count() - n0 == 1
    assert got.shape == (len(boxes), Ho, Wo, 3) and got.dtype == np.uint8
    for k, (i, box) in enumerate(zip(src, boxes)):
        want = pillow(srcs[i], box, Wo, Ho)
        assert np.array_equal(got[k], want), (shapes[i], box)
    outside = [k for k, b in enumerate(boxes) if b[0] > shapes[src[k]][1] or b[2] < 0]
    assert outside and not got[outside].any()


def test_crops_of_a_strided_scene(dev):
    """A scene given as a view whose rows are further apart than 3 W bytes."""
    from neural_astar.utils.data import sdd_crops

    rng = np.random.RandomState(5)
    big = rng.randint(0, 256, (400, 700, 3)).astype(np.uint8)
    view = torch.from_numpy(big).to(dev)[:, 100:600]
    boxes = [(-20, 30, 480, 390), (0, 0, 500, 400), (450, 350, 520, 420)]
    got = sdd_crops(view, boxes, 64).cpu().numpy()
    for k, box in enumerate(boxes):
        assert np.array_equal(got[k], pillow(np.ascontiguousarray(big[:, 100:600]), box, 64, 64)), box


def test_crops_reject_bad_arguments(dev):
    from neural_astar.utils.data import sdd_crops

    scene = torch.zeros((10, 10, 3), dtype=torch.uint8, device=dev)
    with pytest.raises(RuntimeError, match="invalid argument"):
        sdd_crops(scene, [(5, 5, 5, 9)], 8)
    with pytest.raises(RuntimeError, match="unsupported"):
        sdd_crops(scene, [(0, 0, 5000, 9)], 8)
    with pytest.raises(RuntimeError):
        sdd_crops(scene.cpu(), [(0, 0, 5, 9)], 8)


@pytest.fixture(scope="module")
def golden():
    return dict(np.load(os.path.join(SDD, "sdd.npz")))


@pytest.fixture(scope="module")
def same_jpeg_decoder(golden):
    """The fixture's images were cropped from the scenes as Pillow decoded them there; another JPEG decoder gives
    other pixels, which is reported as such and not as a mismatch."""
    for rel, sha in zip(golden["scene"], golden["scene_sha256"]):
        with Image.open(os.path.join(SDD, rel)) as im:
            if hashlib.sha256(np.asarray(im).tobytes()).hexdigest() != sha:
                return False
    return True


@pytest.mark.parametrize("tag", sorted(PARAMS))
def test_tool_writes_the_reference_files(dev, golden, same_jpeg_decoder, tag, tmp_path):
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    import make_sdd_dataset

    W, ratio, mms, max_step = PARAMS[tag]
    argv = ["--input-path", os.path.join(SDD, "original"), "--save-dir", str(tmp_path)]
    if tag != "default":
        argv += ["--size", str(W), "--min-len-ratio", str(ratio), "--min-max-size", str(mms),
                 "--max-step", str(max_step)]
    save_dir = make_sdd_dataset.main(argv)
    assert save_dir == "%s/s%03d_%0.1f_%d_%d" % (tmp_path, W, ratio, mms, max_step)
    dirs = sorted(os.path.relpath(d, save_dir) for d, _, _ in os.walk(save_dir) if d != save_dir)
    assert dirs == list(golden[f"{tag}_dirs"])   # plaza/video2 is there, empty
    files = sorted(os.path.relpath(os.path.join(d, f), save_dir) for d, _, fs in os.walk(save_dir) for f in fs)
    want_files = list(golden[f"{tag}_files"])
    assert files == sorted(want_files)
    toff = np.concatenate([[0], np.cumsum(golden[f"{tag}_traj_len"])])
    members = [m.split()[0] for m in golden[f"{tag}_dtypes"]]
    for k, rel in enumerate(want_files):
        z = np.load(os.path.join(save_dir, rel))
        assert z.files == members, rel
        assert [f"{m} {z[m].dtype.str} {z[m].ndim}" for m in z.files] == list(golden[f"{tag}_dtypes"]), rel
        planes = golden[f"{tag}_planes"][k].astype(np.float64)
        for i, m in enumerate(("start_image", "goal_image", "traj_image")):
            assert np.array_equal(z[m], planes[i]), (rel, m)
        assert np.array_equal(z["traj"], golden[f"{tag}_traj"][toff[k]:toff[k + 1]]), rel
        assert z["label"] == golden[f"{tag}_label"][k] and z["length_ratio"] == golden[f"{tag}_length_ratio"][k]
        assert z["image"].shape == (W, W, 3)
        if same_jpeg_decoder:
            assert np.array_equal(z["image"], golden[f"{tag}_image"][k]), rel
    if not same_jpeg_decoder:
        pytest.skip("this Pillow decodes the fixture's JPEG scenes to other pixels; images were not compared")


def test_a_scene_that_is_not_rgb_raises(dev, tmp_path):
    from neural_astar.utils.data import save_sdd_samples

    v = tmp_path / "in" / "grey" / "video0"
    v.mkdir(parents=True)
    Image.fromarray(np.zeros((300, 400), np.uint8)).save(str(v / "reference.jpg"))
    rows = [f'1 {100 + 2 * i} 100 {110 + 2 * i} 110 {i} 0 0 0 "Biker"' for i in range(100)]
    (v / "annotations.txt").write_text("\n".join(rows) + "\n")
    with pytest.raises(ValueError, match="not RGB"):
        save_sdd_samples([str(v)], str(tmp_path / "out"))


def _archives(dev, rng):
    files = []
    for f in range(5):
        files.append(dict(
            image=torch.from_numpy(rng.randint(0, 256, (16 + f, 16, 3)).astype(np.uint8)).to(dev),
            plane=torch.from_numpy((rng.rand(8, 8) < 0.1).astype(np.float64)).to(dev),
            traj=torch.from_numpy(rng.rand(3 + 7 * f, 2)).to(dev),
            label=torch.tensor(f, dtype=torch.int64, device=dev),
            ratio=torch.tensor(rng.rand(), dtype=torch.float64, device=dev),
            empty=torch.zeros((0, 2), dtype=torch.float32, device=dev)))
    files[3] = dict(only=torch.arange(300000, dtype=torch.int32, device=dev))   # more than one deflate chunk
    return files


def test_many_files_writer_equals_savez_compressed(dev, tmp_path):
    from neural_astar import _native
    from neural_astar.utils.data import _savez_compressed_many

    files = _archives(dev, np.random.RandomState(3))
    paths = [str(tmp_path / f"f{i}.npz") for i in range(len(files) - 1)] + [io.BytesIO()]
    n0 = _native.launch_count()
    _savez_compressed_many(list(zip(paths, files)))
    assert _native.launch_count() - n0 == 1
    for path, members in zip(paths, files):
        ref = io.BytesIO()
        np.savez_compressed(ref, **{k: t.cpu().numpy() for k, t in members.items()})
        if isinstance(path, io.BytesIO):
            path.seek(0)
        ref.seek(0)
        assert zipfile.ZipFile(path).testzip() is None
        if isinstance(path, io.BytesIO):
            path.seek(0)
        got, want = np.load(path), np.load(ref)
        assert got.files == want.files
        for k in want.files:
            assert got[k].dtype == want[k].dtype and got[k].shape == want[k].shape, k
            assert np.array_equal(got[k], want[k]), k
