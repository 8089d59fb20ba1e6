"""CPU tests of the CSM street-crop recipe: street_crop_boxes replays the boxes the reference's crop_images drew on the
fixture sources (tests/golden/street/, both Ns settings, in the glob order it saw), and cropping the sources with
them (through the maps oracle's bicubic resize for the source that is not 256 x 256) gives the crops it saved."""
import os

import numpy as np
import pytest
from PIL import Image

import maps_oracle as mo

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
STREET = os.path.join(ROOT, "tests", "golden", "street")
SPLITS = ("train", "validation", "test")
COUNTS = {"default": (160, 20, 40), "small": (8, 2, 4)}


@pytest.fixture(scope="module")
def golden():
    return dict(np.load(os.path.join(STREET, "street.npz")))


def source_levels(name):
    """A source as crop_images sees it: convert("L"), then the bicubic resize to 256 x 256 (the identity at 256)."""
    with Image.open(os.path.join(STREET, "sources", name)) as im:
        img = np.asarray(im.convert("L"), np.uint8)
    return img if img.shape == (256, 256) else mo.resize(img, 256, 256)


@pytest.mark.parametrize("ns", sorted(COUNTS))
def test_boxes_and_names_equal_the_reference(golden, ns):
    from neural_astar.utils.data import street_crop_boxes

    got = street_crop_boxes(list(golden["glob_train"]), list(golden["glob_test"]), counts=COUNTS[ns])
    for s in SPLITS:
        g = got[s]
        boxes = np.stack([g["left"], g["top"], g["left"] + 128, g["top"] + 128], axis=1)
        assert np.array_equal(boxes, golden[f"{ns}_boxes_{s}"]), s
        assert g["name"] == list(golden[f"{ns}_names_{s}"]), s
        files = golden["glob_test"] if s == "test" else golden["glob_train"]
        assert len(g["source"]) == len(files) * COUNTS[ns][SPLITS.index(s)]
        assert np.array_equal(g["n"], np.tile(np.arange(COUNTS[ns][SPLITS.index(s)]), len(files)))


def test_glob_patterns_split_the_sources(golden):
    """*[0,1]_256.png are the train (and validation) sources, *2_256.png the test sources; one is not 256 x 256."""
    assert all(n[-9] in "01" for n in golden["glob_train"]) and all(n[-9] == "2" for n in golden["glob_test"])
    assert sorted(os.listdir(os.path.join(STREET, "sources"))) == sorted(
        list(golden["glob_train"]) + list(golden["glob_test"]))
    shapes = {}
    for n in os.listdir(os.path.join(STREET, "sources")):
        with Image.open(os.path.join(STREET, "sources", n)) as im:
            shapes[n] = im.size
    assert sum(s != (256, 256) for s in shapes.values()) == 1


def test_crops_equal_the_reference(golden):
    from neural_astar.utils.data import street_crop_boxes

    got = street_crop_boxes(list(golden["glob_train"]), list(golden["glob_test"]), counts=COUNTS["small"])
    for s in SPLITS:
        files = golden["glob_test"] if s == "test" else golden["glob_train"]
        srcs = [source_levels(f) for f in files]
        g = got[s]
        crops = np.stack([srcs[k][t:t + 128, l:l + 128] for k, l, t in zip(g["source"], g["left"], g["top"])])
        assert np.array_equal(crops, golden[f"small_crops_{s}"]), s
