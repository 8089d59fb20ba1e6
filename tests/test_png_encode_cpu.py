"""CPU tests of the PNG encoder's oracle (tests/png_encode_oracle.py) and ABI: the oracle's files decode with Pillow
(CRC checks on) to their inputs, its filter choice follows libpng's heuristic with ties to the lowest type, its
Adler-32 is zlib's, its files are at most 1.10x Pillow's default PNGs of the street fixture's crops (0.997x measured),
and the encode ABI rejects bad arguments without a launch."""
import io
import os
import zlib

import numpy as np
import pytest
from PIL import Image, ImageFile

import png_encode_oracle as P

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
STREET = os.path.join(ROOT, "tests", "golden", "street", "street.npz")


def images(H, W, seed=0):
    """Random, binary, uniform and gradient images of one shape."""
    rng = np.random.RandomState(seed + H * 7 + W)
    yy, xx = np.mgrid[:H, :W]
    return {"random": rng.randint(0, 256, (H, W)).astype(np.uint8),
            "binary": (rng.rand(H, W) > 0.3).astype(np.uint8) * 255,
            "uniform": np.full((H, W), 93, np.uint8),
            "gradient": ((xx * 3 + yy * 5) % 256).astype(np.uint8)}


def pillow_decode(blob: bytes) -> np.ndarray:
    assert not ImageFile.LOAD_TRUNCATED_IMAGES
    with Image.open(io.BytesIO(blob)) as im:
        assert im.mode == "L" and im.format == "PNG"
        im.load()
        return np.asarray(im)


@pytest.mark.parametrize("shape", [(1, 1), (1, 2048), (2048, 1), (7, 13), (128, 128), (256, 256)])
def test_oracle_files_decode_to_input(shape):
    for kind, img in images(*shape).items():
        blob = P.encode(img)
        assert np.array_equal(pillow_decode(blob), img), kind
        z = blob[P.HEAD_BYTES - 2:len(blob) - P.TAIL_BYTES + 4]
        assert zlib.decompress(z) == P.filtered_stream(img), kind


def test_filter_choice_and_ties():
    types, rows = P.filter_rows(np.full((4, 9), 93, np.uint8))
    assert types.tolist() == [1, 2, 2, 2]   # row 0: Sub beats Paeth on a tie; then Up ties with Paeth at 0
    assert not rows[1:].any()
    types, _ = P.filter_rows(np.zeros((3, 5), np.uint8))
    assert types.tolist() == [0, 0, 0]
    # brute force on a random image: the chosen type's cost is the least, and no lower type ties it
    img = np.random.RandomState(5).randint(0, 256, (40, 33)).astype(np.uint8)
    types, rows = P.filter_rows(img)
    x = img.astype(np.int64)
    for y in range(img.shape[0]):
        prev = x[y - 1] if y else np.zeros_like(x[0])
        costs = []
        for f in range(5):
            r = []
            for i in range(img.shape[1]):
                a, b, c = (x[y, i - 1] if i else 0), prev[i], (prev[i - 1] if i else 0)
                p = a + b - c
                pa, pb, pc = abs(p - a), abs(p - b), abs(p - c)
                pr = a if pa <= pb and pa <= pc else (b if pb <= pc else c)
                r.append((x[y, i] - (0, a, b, (a + b) // 2, pr)[f]) & 0xFF)
            costs.append(sum(v if v < 128 else 256 - v for v in r))
            if f == types[y]:
                assert rows[y].tolist() == r
        assert types[y] == int(np.argmin(costs))


@pytest.mark.parametrize("n", [0, 1, 5552, 5553, 100000])
def test_adler_is_zlib(n):
    data = np.random.RandomState(n).randint(0, 256, n).astype(np.uint8).tobytes()
    assert P.adler32(data) == zlib.adler32(data)
    assert P.adler32(b"\xff" * n) == zlib.adler32(b"\xff" * n)


def test_oracle_size_against_pillow_on_street_crops():
    z = np.load(STREET)
    ours = pil = 0
    for s in ("train", "validation", "test"):
        for c in z[f"small_crops_{s}"]:
            ours += len(P.encode(c))
            b = io.BytesIO()
            Image.fromarray(c).save(b, "PNG")
            pil += len(b.getvalue())
    assert ours <= 1.10 * pil, (ours, pil)


def test_abi_rejections_without_launch():
    from neural_astar import _native

    try:
        L = _native.lib()
    except _native.NativeLibraryMissing:
        pytest.skip("engine not built")
    d = np.zeros(2, _native.PNG_ENC_DESC_DTYPE)
    d["pixels"], d["W"], d["H"] = [1 << 40, 1 << 41], [7, 2048], [13, 1]
    d["filt_off"] = [0, 13 * 8]
    filt_bytes = 13 * 8 + 2049
    bound = int(L.nastar_b200_png_encode_bound(d.ctypes.data, 2))
    members = 13 * 8 + 2049
    assert bound >= 43 + 63 + 20 + members
    assert [L.nastar_b200_png_gap(i) for i in range(3)] == [43, 63, 63]
    assert np.array_equal(_native.png_gaps(3), [43, 63, 63])
    filt, adler, dd, out, off, ln = 1 << 42, 1 << 43, 1 << 44, 1 << 45, 1 << 46, 1 << 47
    n0 = L.nastar_b200_launch_count()

    def flt(desc, B=2, ddev=dd, f=filt, fb=filt_bytes, ad=adler):
        return L.nastar_b200_png_filter(desc.ctypes.data if desc is not None else None, ddev, B, f, fb, ad, None)

    def fin(desc, B=2, ddev=dd, of=off, le=ln, ad=adler, o=out, ob=bound):
        return L.nastar_b200_png_finish(desc.ctypes.data if desc is not None else None, ddev, B, of, le, ad, o, ob,
                                        None)

    for call in (flt, fin):
        assert call(None) == 1
        assert call(d, B=0) == 1
        assert call(d, ddev=None) == 1
        for field, value in (("pixels", 0), ("W", 0), ("H", -1)):
            bad = d.copy()
            bad[field][1] = value
            assert call(bad) == 1, (call.__name__, field)
        big = d.copy()
        big["W"][0] = 2049
        assert call(big) == 2
        both = big.copy()
        both["pixels"][1] = 0
        assert call(both) == 1   # an invalid descriptor outranks an unsupported one
    bad = d.copy()
    bad["filt_off"][0] = -1
    assert flt(bad) == 1
    assert flt(d, f=None) == 1 and flt(d, ad=None) == 1
    assert flt(d, fb=filt_bytes - 1) == 4
    assert fin(d, of=None) == 1 and fin(d, le=None) == 1 and fin(d, ad=None) == 1 and fin(d, o=None) == 1
    assert fin(d, ob=bound - 1) == 4
    assert L.nastar_b200_png_encode_bound(big.ctypes.data, 2) == -1
    assert L.nastar_b200_launch_count() == n0
