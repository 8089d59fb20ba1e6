"""CPU tests of the Stanford Drone (SDD) sample plan: sdd_sample_plan replays what the reference's own
create_sample_from_dataset wrote for the fixture videos (tests/golden/sdd/, both parameter sets, one RandomState(0)
shared across the videos in sorted order), the annotation parser, and the rejections of nastar_b200_crop_resize_rgb,
which launch nothing."""
import ctypes
import os
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SDD = os.path.join(ROOT, "tests", "golden", "sdd")
PARAMS = {"default": (64, 0.5, 128, 300), "small": (32, 0.3, 64, 40)}
EINVAL, EUNSUPPORTED = 1, 2


@pytest.fixture(scope="module")
def golden():
    return dict(np.load(os.path.join(SDD, "sdd.npz")))


def plans(golden, tag):
    from neural_astar.utils.data import sdd_sample_plan

    W, ratio, mms, max_step = PARAMS[tag]
    rng = np.random.RandomState(0)
    return [sdd_sample_plan(os.path.join(SDD, v), W, ratio, mms, max_step, rng) for v in golden["videos"]]


@pytest.mark.parametrize("tag", sorted(PARAMS))
def test_plan_equals_the_reference(golden, tag):
    W = PARAMS[tag][0]
    ps = plans(golden, tag)
    names = [f"{p['scene']}/{p['video']}/{n}" for p in ps for n in p["name"]]
    assert names == list(golden[f"{tag}_files"])
    roi = golden[f"{tag}_roi"]
    box = np.concatenate([p["box"] for p in ps])
    assert np.array_equal(box, np.array([[round(float(v)) for v in r] for r in roi], np.int64))
    trajs = [t for p in ps for t in p["traj"]]
    assert [len(t) for t in trajs] == list(golden[f"{tag}_traj_len"])
    assert np.array_equal(np.concatenate(trajs), golden[f"{tag}_traj"])   # float64, bit for bit
    assert np.array_equal(np.concatenate([p["label"] for p in ps]), golden[f"{tag}_label"])
    assert np.array_equal(np.concatenate([p["length_ratio"] for p in ps]), golden[f"{tag}_length_ratio"])
    planes = golden[f"{tag}_planes"]
    k = 0
    for p in ps:
        for start, goal, cells in zip(p["start"], p["goal"], p["cells"]):
            want = np.zeros((3, W, W), np.uint8)
            want[0, start[0], start[1]] = want[1, goal[0], goal[1]] = 1
            want[2, cells[:, 0], cells[:, 1]] = 1
            assert np.array_equal(want, planes[k]), names[k]
            k += 1


def test_fixture_covers_the_rules(golden):
    """The fixture exercises both ROI branches past every edge, .5 ties on both sides of zero, every rejection and
    draws for rejected segments; plaza/video2 keeps nothing."""
    from neural_astar.utils.data import read_sdd_annotations

    roi = golden["default_roi"]
    half = roi - np.floor(roi) == 0.5
    assert (half & (roi < 0)).any() and (half & (roi > 0)).any()
    assert any(round(v) != np.floor(v + 0.5) for v in roi[half])   # a tie that rounds to even, not up
    sizes = {}
    for v in golden["videos"]:
        from PIL import Image

        with Image.open(os.path.join(SDD, v, "reference.jpg")) as im:
            sizes[v] = im.size
    files = golden["default_files"]
    Ws = np.array([sizes["original/" + "/".join(f.split("/")[:2])][0] for f in files])
    Hs = np.array([sizes["original/" + "/".join(f.split("/")[:2])][1] for f in files])
    assert (roi[:, 0] < 0).any() and (roi[:, 1] < 0).any() and (roi[:, 2] > Ws).any() and (roi[:, 3] > Hs).any()
    assert max(max(s) for s in sizes.values()) > 2048
    assert set(golden["default_label"]) == set(range(6))
    assert not any(f.startswith("plaza/video2/") for f in files)
    assert "plaza/video2" in set(golden["default_dirs"])
    cols, _ = read_sdd_annotations(os.path.join(SDD, "original", "plaza", "video0", "annotations.txt"))
    assert ((cols[:, 7] == 1) & (cols[:, 6] == 0)).any()   # occluded but visible rows
    assert len(golden["small_files"]) != len(golden["default_files"])


def test_annotation_parser_strips_quotes(tmp_path):
    from neural_astar.utils.data import read_sdd_annotations

    p = tmp_path / "annotations.txt"
    p.write_text('3 10 20 30 40 0 0 1 0 "Biker"\n3 11 21 31 41 1 1 0 1 "Biker"\n\n7 0 0 5 5 0 0 0 0 "Bus"\n')
    cols, labels = read_sdd_annotations(str(p))
    assert cols.dtype == np.int64 and cols.shape == (3, 9)
    assert cols[1].tolist() == [3, 11, 21, 31, 41, 1, 1, 0, 1]
    assert labels == ["Biker", "Biker", "Bus"]
    p.write_text('3 10 20 30 40 0 0 1 "Biker"\n')
    with pytest.raises(ValueError):
        read_sdd_annotations(str(p))


def test_plan_with_global_state_equals_a_shared_random_state(golden):
    """rng=None draws from NumPy's global state, as the reference does after np.random.seed(0)."""
    from neural_astar.utils.data import sdd_sample_plan

    W, ratio, mms, max_step = PARAMS["small"]
    np.random.seed(0)
    got = [sdd_sample_plan(os.path.join(SDD, v), W, ratio, mms, max_step) for v in golden["videos"]]
    want = plans(golden, "small")
    for a, b in zip(got, want):
        assert a["name"] == b["name"] and np.array_equal(a["box"], b["box"])


@pytest.fixture(scope="module")
def built_lib():
    subprocess.check_call(["make", "-C", os.path.join(ROOT, "neural-astar_b200"), "-s", "all"])
    from neural_astar import _native

    return _native


@pytest.fixture
def no_launch(built_lib):
    L = built_lib.lib()
    before = L.nastar_b200_launch_count()
    yield L
    assert L.nastar_b200_launch_count() == before, "a rejected call launched something"


def _crop(native, L, images=None, crops=None, S=None, N=None, Ho=64, Wo=64, out=0x30000, null=()):
    img = np.zeros(2, native.RGB_IMAGE_DTYPE)
    img[0] = (0x10000, 3 * 720, 720, 540)
    img[1] = (0x20000, 3 * 2100 + 4, 2100, 360)
    for k, v in (images or {}).items():
        i, field = k
        img[i][field] = v
    cr = np.zeros(3, native.RGB_CROP_DTYPE)
    cr[0] = (0, 2, -30, -20, 300, 310)
    cr[1] = (1, 0, 2000, 100, 2200, 400)
    cr[2] = (0, 1, 10, 10, 11, 11)
    for k, v in (crops or {}).items():
        i, field = k
        cr[i][field] = v
    args = [img.ctypes.data, 0x40000, len(img) if S is None else S, cr.ctypes.data, 0x50000,
            len(cr) if N is None else N, Ho, Wo, out]
    for i in null:
        args[i] = None
    return L.nastar_b200_crop_resize_rgb(*args, None)


@pytest.mark.parametrize("kw,code", [
    (dict(null=(0,)), EINVAL), (dict(null=(1,)), EINVAL), (dict(null=(3,)), EINVAL), (dict(null=(4,)), EINVAL),
    (dict(out=None), EINVAL), (dict(S=0), EINVAL), (dict(N=0), EINVAL), (dict(Ho=0), EINVAL), (dict(Wo=-1), EINVAL),
    (dict(images={(0, "pixels"): 0}), EINVAL), (dict(images={(1, "W"): 0}), EINVAL),
    (dict(images={(0, "H"): -1}), EINVAL), (dict(images={(0, "pitch"): 3 * 720 - 1}), EINVAL),
    (dict(crops={(0, "src"): 2}), EINVAL), (dict(crops={(0, "src"): -1}), EINVAL),
    (dict(crops={(0, "out"): 3}), EINVAL), (dict(crops={(0, "out"): 0}), EINVAL),
    (dict(crops={(2, "x1"): 10}), EINVAL), (dict(crops={(2, "y1"): 9}), EINVAL),
    (dict(Ho=1025), EUNSUPPORTED), (dict(Wo=1025), EUNSUPPORTED),
    (dict(images={(1, "W"): 4097, (1, "pitch"): 3 * 4097}), EUNSUPPORTED),
    (dict(images={(0, "H"): 4097}), EUNSUPPORTED),
    (dict(crops={(1, "x1"): 2000 + 4097}), EUNSUPPORTED), (dict(crops={(0, "y0"): 310 - 4097}), EUNSUPPORTED),
    # an invalid descriptor takes precedence over an unsupported one before it
    (dict(images={(0, "H"): 4097}, crops={(2, "x1"): 10}), EINVAL),
    (dict(crops={(0, "x1"): -30 + 4097 + 1, (2, "out"): 2}), EINVAL),
])
def test_crop_resize_rejections_launch_nothing(built_lib, no_launch, kw, code):
    assert _crop(built_lib, no_launch, **kw) == code


def test_crop_descriptor_layout_matches_the_header(built_lib):
    assert built_lib.RGB_IMAGE_DTYPE.itemsize == 24 and built_lib.RGB_CROP_DTYPE.itemsize == 24
    assert ctypes.sizeof(ctypes.c_void_p) == 8
