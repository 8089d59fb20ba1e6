"""NumPy oracle of the planning-datasets generator's map recipe (DESIGN.md §13): Pillow's BICUBIC `Image.resize` of a
uint8 `L` image, skimage's `threshold_otsu` (>= 0.19) of the float32 result, `img > threshold` as 1.0 / 0.0, and
`skimage.util.montage` tiles.  Written from the semantics, with Python's IEEE doubles in Pillow's operation order; it
needs neither Pillow nor skimage.  The GPU kernel (csrc/nastar_maps.cuh) is checked against it bit for bit."""
from __future__ import annotations

import re

import numpy as np

PRECISION_BITS = 22   # Pillow's 8-bit resample: 32 - 8 - 2 fraction bits


def _cubic(x: float) -> float:
    """Keys' cubic convolution kernel with a = -0.5, evaluated in Pillow's operation order."""
    a = -0.5
    if x < 0.0:
        x = -x
    if x < 1.0:
        return ((a + 2.0) * x - (a + 3.0)) * x * x + 1
    if x < 2.0:
        return (((x - 5) * x + 8) * x - 4) * a
    return 0.0


def resize_coeffs(in_size: int, out_size: int):
    """Per output pixel j: (xmin, fixed-point weights int64 [taps]) of one resize axis."""
    scale = float(in_size) / out_size
    fs = max(scale, 1.0)
    support = 2.0 * fs
    ss = 1.0 / fs
    out = []
    for j in range(out_size):
        center = (j + 0.5) * scale
        xmin = max(int(center - support + 0.5), 0)
        n = min(int(center + support + 0.5), in_size) - xmin
        k = [_cubic((x + xmin - center + 0.5) * ss) for x in range(n)]
        ww = 0.0
        for w in k:
            ww += w
        if ww != 0.0:
            k = [w / ww for w in k]
        q = [int(-0.5 + w * (1 << PRECISION_BITS)) if w < 0 else int(0.5 + w * (1 << PRECISION_BITS)) for w in k]
        out.append((xmin, np.array(q, np.int64)))
    return out


def _resample_rows(img: np.ndarray, out_size: int) -> np.ndarray:
    """Resample axis 1 of an int64 [R, in] array to [R, out_size] uint8 levels."""
    res = np.empty((img.shape[0], out_size), np.int64)
    for j, (xmin, k) in enumerate(resize_coeffs(img.shape[1], out_size)):
        res[:, j] = ((1 << (PRECISION_BITS - 1)) + img[:, xmin:xmin + len(k)] @ k) >> PRECISION_BITS
    return np.clip(res, 0, 255)


def resize(img: np.ndarray, H: int, W: int) -> np.ndarray:
    """Image.fromarray(img, "L").resize((W, H)) (BICUBIC, reducing_gap=None) of a uint8 [H0, W0] image: a horizontal
    pass into a uint8 intermediate when the width changes, then a vertical pass when the height changes."""
    out = np.asarray(img, np.uint8).astype(np.int64)
    if out.shape[1] != W:
        out = _resample_rows(out, W)
    if out.shape[0] != H:
        out = _resample_rows(out.T, H).T
    return np.ascontiguousarray(out.astype(np.uint8))


def otsu(img: np.ndarray):
    """(threshold float32, uniform) of skimage.filters.threshold_otsu on np.float32(img): a uniform image returns its
    value; otherwise the center of the first bin that maximises the between-class variance of the 256-bin histogram
    over [min, max], with sequential float64 cumulative sums."""
    f = np.asarray(img, np.float32).reshape(-1)
    if np.all(f == f[0]):
        return f[0], True
    counts, edges = np.histogram(f, 256)
    centers = (edges[:-1] + edges[1:]) / 2
    w1 = np.cumsum(counts)
    w2 = np.cumsum(counts[::-1])[::-1]
    m1 = np.cumsum(counts * centers) / w1
    m2 = (np.cumsum((counts * centers)[::-1]) / w2[::-1])[::-1]
    var = w1[:-1] * w2[1:] * (m1[:-1] - m2[1:]) ** 2
    return centers[np.argmax(var)], False


def level_bins(lo: int, hi: int):
    """The kernel's rule for integer levels lo < hi: (bin int [hi-lo+1] of levels lo..hi, centers float32 [256]).
    np.histogram's edges over [lo, hi] are lo + i*(hi-lo)/256, exact in float32, so level v falls in bin
    min(floor((v-lo)*256/(hi-lo)), 255) and bin i's center is lo + (2i+1)*(hi-lo)/512, also exact."""
    d = hi - lo
    v = np.arange(lo, hi + 1)
    bins = np.minimum((v - lo) * 256 // d, 255)
    centers = (lo + (2 * np.arange(256) + 1) * d / 512).astype(np.float32)
    return bins, centers


def make_map(img: np.ndarray, H: int, W: int):
    """(map float32 [H, W] of 1.0 / 0.0, resized uint8 [H, W], threshold float32, status): the generator's
    load_maze_from_directory for one decoded image; status bit 1 = uniform resized image (all-zero map)."""
    r = resize(img, H, W)
    th, uniform = otsu(r)
    m = (r.astype(np.float32) > th).astype(np.float32)
    return m, r, np.float32(th), int(uniform)


def montage(maps: np.ndarray, t: int) -> np.ndarray:
    """skimage.util.montage of t*t equal-size maps [t*t, h, w] with no fill: map k goes to grid cell (k // t, k % t)."""
    k, h, w = maps.shape
    assert k == t * t
    return maps.reshape(t, t, h, w).transpose(0, 2, 1, 3).reshape(t * h, t * w)


def natural_key(s: str):
    """natsort's default key for these paths: digit runs compare as integers."""
    return [int(p) if p.isdigit() else p for p in re.split(r"(\d+)", s)]
