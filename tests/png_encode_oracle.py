"""NumPy restatement of the PNG encoder (csrc/nastar_png_encode.cuh, DESIGN.md §21): the filter choice and the
Adler-32 here, the raw deflate stream from oracle/deflate.py (the deflate kernel's own oracle) and the CRC-32s from
zlib.  encode() gives the whole file the kernels write: signature, IHDR (8-bit grey, not interlaced), one IDAT chunk
(zlib header 78 DA, the stream, the Adler-32), IEND.

TEST INFRASTRUCTURE ONLY."""
from __future__ import annotations

import struct
import zlib

import numpy as np

SIGNATURE = b"\x89PNG\r\n\x1a\n"
ZLIB_HEADER = b"\x78\xda"
HEAD_BYTES, TAIL_BYTES = 43, 20   # a file's bytes before and after its deflate stream


def filter_rows(img: np.ndarray):
    """(filter types uint8 [H], filtered rows uint8 [H, W]): per row the type 0..4 whose bytes have the least sum of
    |byte as int8|, ties to the lowest type; row 0 sees zeros above it."""
    x = np.asarray(img, np.uint8).astype(np.int32)
    H, W = x.shape
    up = np.vstack([np.zeros((1, W), np.int32), x[:-1]])
    left = np.hstack([np.zeros((H, 1), np.int32), x[:, :-1]])
    upleft = np.hstack([np.zeros((H, 1), np.int32), up[:, :-1]])
    p = left + up - upleft
    pa, pb, pc = np.abs(p - left), np.abs(p - up), np.abs(p - upleft)
    paeth = np.where((pa <= pb) & (pa <= pc), left, np.where(pb <= pc, up, upleft))
    cand = np.stack([x, x - left, x - up, x - ((left + up) >> 1), x - paeth]) & 0xFF   # [5, H, W]
    cost = np.where(cand < 128, cand, 256 - cand).sum(axis=2)                          # [5, H]
    types = np.argmin(cost, axis=0).astype(np.uint8)                                   # the first minimum
    rows = cand[types, np.arange(H)].astype(np.uint8)
    return types, rows


def filtered_stream(img: np.ndarray) -> bytes:
    """The H*(W+1) bytes the filter kernel writes: filter type, then the filtered row, per scanline."""
    types, rows = filter_rows(img)
    return np.hstack([types[:, None], rows]).tobytes()


def adler32(data: bytes) -> int:
    """Adler-32 as the kernel sums it: A = 1 + sum d_j, B = n + sum (n - j) d_j, both mod 65521."""
    d = np.frombuffer(data, np.uint8).astype(np.uint64)
    n = len(d)
    w = (n - np.arange(n, dtype=np.uint64)) % np.uint64(65521)
    a = (1 + int(d.sum())) % 65521
    b = (n + int((d * w % np.uint64(65521)).sum())) % 65521
    return (b << 16) | a


def chunk(ctype: bytes, data: bytes) -> bytes:
    return struct.pack(">I", len(data)) + ctype + data + struct.pack(">I", zlib.crc32(ctype + data) & 0xFFFFFFFF)


def encode(img: np.ndarray) -> bytes:
    """The PNG file the kernels write for one uint8 [H, W] image."""
    from oracle import deflate as D

    img = np.asarray(img, np.uint8)
    H, W = img.shape
    raw = filtered_stream(img)
    z = ZLIB_HEADER + D.member(b"", raw) + struct.pack(">I", adler32(raw))
    return (SIGNATURE + chunk(b"IHDR", struct.pack(">IIBBBBB", W, H, 8, 0, 0, 0, 0)) + chunk(b"IDAT", z)
            + chunk(b"IEND", b""))
