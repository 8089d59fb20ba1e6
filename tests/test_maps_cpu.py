"""CPU checks of the map recipe (DESIGN.md §13): the NumPy oracle against Pillow's resize and np.histogram, against the
shipped planning-datasets maps, the host helpers of utils.data, and the C entry points' rejections."""
import os
import subprocess

import numpy as np
import pytest
import torch

import maps_oracle as mo

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "maps", "sources.npz")
EINVAL, EUNSUPPORTED = 1, 2


def _image(kind, h, w, rng):
    if kind == "random":
        return rng.randint(0, 256, (h, w)).astype(np.uint8)
    if kind == "binary":
        return ((rng.rand(h, w) > 0.5) * 255).astype(np.uint8)
    return (np.add.outer(np.arange(h), np.arange(w)) * 255 // max(1, h + w - 2)).astype(np.uint8)


SHAPES = [(201, 201, 32, 32), (201, 201, 64, 64), (201, 201, 256, 256), (37, 90, 200, 12), (100, 100, 33, 100),
          (5, 7, 3, 64), (1, 1, 5, 5), (7, 1, 1, 9), (1, 40, 3, 1), (64, 64, 64, 64), (300, 5, 3, 700)]


@pytest.mark.parametrize("kind", ["random", "binary", "gradient"])
@pytest.mark.parametrize("shape", SHAPES, ids=lambda s: "{}x{}to{}x{}".format(*s))
def test_oracle_resize_equals_pillow(shape, kind):
    Image = pytest.importorskip("PIL.Image")
    h0, w0, h, w = shape
    img = _image(kind, h0, w0, np.random.RandomState(h0 * 7 + w0))
    ref = np.asarray(Image.fromarray(img, "L").resize((w, h)))
    assert np.array_equal(mo.resize(img, h, w), ref)


def test_level_bins_equal_np_histogram_for_every_range():
    """Levels lo..hi (each level once, plus lo and hi again) land in np.histogram's bins with its float32 centers."""
    for lo in range(256):
        for hi in range(lo + 1, 256):
            a = np.concatenate([[lo, hi], np.arange(lo, hi + 1)]).astype(np.float32)
            counts, edges = np.histogram(a, 256)
            bins, centers = mo.level_bins(lo, hi)
            expect = np.bincount(bins, minlength=256)
            expect[bins[0]] += 1
            expect[bins[-1]] += 1
            assert np.array_equal(counts, expect), (lo, hi)
            assert np.array_equal((edges[:-1] + edges[1:]) / 2, centers), (lo, hi)


def test_otsu_uniform_and_two_level():
    th, uniform = mo.otsu(np.full((5, 7), 37, np.uint8))
    assert uniform and th == 37
    th, uniform = mo.otsu(np.array([[10, 10, 200]], np.uint8))
    assert not uniform and 10 < th < 200


@pytest.fixture(scope="module")
def golden():
    with np.load(GOLDEN) as z:
        return {k: z[k] for k in z.files}


def test_oracle_equals_shipped_mp_maps(golden):
    imgs, ship = golden["mp_images"], np.unpackbits(golden["mp_maps"], axis=1)[:, :1024].reshape(-1, 32, 32)
    got = np.stack([mo.make_map(im, 32, 32)[0] for im in imgs])
    assert np.array_equal(got, ship)


def test_oracle_tiles_replay_shipped_tiled_mp(golden):
    pos, count = golden["tiled_pos"], int(golden["tiled_count"])
    maps = np.stack([mo.make_map(im, 32, 32)[0] for im in golden["tiled_images"]])
    ship = np.unpackbits(golden["tiled_maps"], axis=1).reshape(-1, 64, 64)
    rng = np.random.RandomState(1372)
    for t in range(len(ship)):
        idx = np.searchsorted(pos, rng.choice(count, 4))
        assert np.array_equal(mo.montage(maps[idx], 2), ship[t]), t


def test_tile_maps_equals_montage():
    from neural_astar.utils.data import tile_maps

    rng = np.random.RandomState(3)
    maps = rng.rand(10, 5, 7).astype(np.float32)
    idx = rng.randint(0, 10, (6, 9))
    got = tile_maps(torch.from_numpy(maps), 3, indices=idx)
    assert got.shape == (6, 1, 15, 21)
    for t in range(6):
        assert np.array_equal(got[t, 0].numpy(), mo.montage(maps[idx[t]], 3))
    with pytest.raises(ValueError):
        tile_maps(torch.from_numpy(maps), 3, indices=idx[:, :4])
    with pytest.raises(IndexError):
        tile_maps(torch.from_numpy(maps), 3, indices=idx + 10)


def test_load_map_images_natural_order_and_groups(tmp_path):
    Image = pytest.importorskip("PIL.Image")
    from neural_astar.utils.data import load_map_images

    rng = np.random.RandomState(4)
    made = {}
    for fam in ("b", "a"):
        os.makedirs(tmp_path / fam / "train")
        for i in (10, 2, 1):
            shape = (9, 11) if i == 2 else (6, 6)
            img = rng.randint(0, 256, shape + (3,)).astype(np.uint8)
            Image.fromarray(img, "RGB").save(tmp_path / fam / "train" / f"{i}.png")
            made[(fam, i)] = np.asarray(Image.fromarray(img, "RGB").convert("L"))
    order = [(f, i) for f in ("a", "b") for i in (1, 2, 10)]
    groups = load_map_images(str(tmp_path / "*"), "train")
    seen = {}
    for pos, imgs in groups:
        for p, im in zip(pos, imgs):
            seen[int(p)] = im
    assert sorted(seen) == list(range(6))
    for p, key in enumerate(order):
        assert np.array_equal(seen[p], made[key])
    assert sorted(imgs.shape[1:] for _, imgs in groups) == [(6, 6), (9, 11)]
    with pytest.raises(ValueError):
        load_map_images(str(tmp_path / "a"), "valid")


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


def _maps(L, **kw):
    a = dict(images=0x10000, stride=201 * 201, B=4, H0=201, W0=201, H=32, W=32, maps=0x20000, resized=None,
             thresholds=0x30000, status=0x40000)
    a.update(kw)
    return L.nastar_b200_maps_from_images(a["images"], a["stride"], a["B"], a["H0"], a["W0"], a["H"], a["W"],
                                          a["maps"], a["resized"], a["thresholds"], a["status"], None)


@pytest.mark.parametrize("kw,code", [
    (dict(images=None), EINVAL), (dict(maps=None), EINVAL), (dict(thresholds=None), EINVAL),
    (dict(status=None), EINVAL), (dict(B=0), EINVAL), (dict(H0=0), EINVAL), (dict(W0=-1), EINVAL),
    (dict(H=0), EINVAL), (dict(W=0), EINVAL), (dict(stride=201 * 201 - 1), EINVAL),
    (dict(H=513), EUNSUPPORTED), (dict(W=513), EUNSUPPORTED), (dict(H0=2049, stride=2049 * 201), EUNSUPPORTED),
    (dict(W0=2049, stride=2049 * 201), EUNSUPPORTED),
])
def test_maps_from_images_rejections_launch_nothing(no_launch, kw, code):
    assert _maps(no_launch, **kw) == code


@pytest.mark.parametrize("args", [(None, 0x2000, 2, 16, 0x3000), (0x1000, None, 2, 16, 0x3000),
                                  (0x1000, 0x2000, 0, 16, 0x3000), (0x1000, 0x2000, 2, 0, 0x3000),
                                  (0x1000, 0x2000, 2, 16, None)])
def test_draw_policies_rejections_launch_nothing(no_launch, args):
    m, d, B, N, p = args
    assert no_launch.nastar_b200_draw_policies(m, d, B, N, p, None) == EINVAL
