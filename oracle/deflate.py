"""ctypes front-end of the CPU oracle of the chunked deflate (oracle/deflate_oracle.c), plus the CRC-32 shift the
kernel uses to join chunk CRCs, restated in Python.

TEST / BASELINE INFRASTRUCTURE ONLY: imported by tests/ and tools/; the product package never imports this module.
"""
from __future__ import annotations

import ctypes
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_SRC = os.path.join(_HERE, "deflate_oracle.c")
_LIB_PATH = os.path.join(_HERE, "libdeflate_oracle.so")
_CC = ["/usr/bin/gcc", "-O2", "-fPIC", "-Wall", "-Wextra", "-std=c11"]
_lib = None


def build(force: bool = False) -> str:
    """Compile the oracle with gcc (well under a second)."""
    if force or not os.path.exists(_LIB_PATH) or os.path.getmtime(_LIB_PATH) < os.path.getmtime(_SRC):
        subprocess.check_call(_CC + ["-shared", "-o", _LIB_PATH, _SRC])
    return _LIB_PATH


def _load():
    global _lib
    if _lib is None:
        build()
        lib = ctypes.CDLL(_LIB_PATH)
        lib.nastar_oracle_deflate.argtypes = [ctypes.c_void_p, ctypes.c_int64, ctypes.c_void_p]
        lib.nastar_oracle_deflate.restype = ctypes.c_int64
        lib.nastar_oracle_deflate_chunk_bound.argtypes = [ctypes.c_int64]
        lib.nastar_oracle_deflate_chunk_bound.restype = ctypes.c_int64
        lib.nastar_oracle_deflate_chunk_size.restype = ctypes.c_int64
        _lib = lib
    return _lib


def chunk_size() -> int:
    return int(_load().nastar_oracle_deflate_chunk_size())


def bound(n: int) -> int:
    """Worst-case size of deflate(n bytes)."""
    lib, c = _load(), chunk_size()
    full, rest = divmod(n, c)
    return full * int(lib.nastar_oracle_deflate_chunk_bound(c)) + int(lib.nastar_oracle_deflate_chunk_bound(rest))


def deflate(data) -> bytes:
    """The raw deflate stream of `data` (bytes or an array's bytes) cut into chunks, as the kernel writes it."""
    src = np.frombuffer(bytes(data) if not isinstance(data, np.ndarray) else np.ascontiguousarray(data).tobytes(),
                        np.uint8)
    out = np.zeros(bound(len(src)), np.uint8)
    n = _load().nastar_oracle_deflate(src.ctypes.data if len(src) else None, len(src), out.ctypes.data)
    return out[:n].tobytes()


def member(header: bytes, data) -> bytes:
    """One .npz member's stream: the .npy header as its own chunk, then the data's chunks (final only when the data
    is empty)."""
    raw = np.ascontiguousarray(data).tobytes() if isinstance(data, np.ndarray) else bytes(data)
    if not raw:
        return deflate(header)
    head = deflate_nonfinal(header)
    return head + deflate(raw)


def deflate_nonfinal(data: bytes) -> bytes:
    """One chunk (len(data) <= chunk_size()) that is not its stream's last."""
    lib = _load()
    lib.nastar_oracle_deflate_chunk.argtypes = [ctypes.c_void_p, ctypes.c_int64, ctypes.c_int, ctypes.c_void_p]
    lib.nastar_oracle_deflate_chunk.restype = ctypes.c_int64
    src = np.frombuffer(bytes(data), np.uint8)
    if len(src) > chunk_size():
        raise ValueError("one chunk at most")
    out = np.zeros(int(lib.nastar_oracle_deflate_chunk_bound(len(src))), np.uint8)
    n = lib.nastar_oracle_deflate_chunk(src.ctypes.data if len(src) else None, len(src), 0, out.ctypes.data)
    return out[:n].tobytes()


# ---- CRC-32 shift: crc(A || B) = shift(crc(A), |B|) ^ crc(B), over GF(2) modulo the reflected polynomial ---------
_POLY = 0xEDB88320


def _multmodp(a: int, b: int) -> int:
    """a * b modulo the CRC polynomial (reflected bit order: bit 31 is x^0)."""
    m, p = 1 << 31, 0
    while True:
        if a & m:
            p ^= b
            if (a & (m - 1)) == 0:
                break
        m >>= 1
        b = (b >> 1) ^ _POLY if b & 1 else b >> 1
    return p


def _x2nmodp(n: int) -> int:
    """x^(8 n) modulo the polynomial, by squaring: x^(2^k) for k = 3.. over the bits of n."""
    p, sq = 1 << 31, 1 << 30   # p = x^0; sq = x^1, squared three times to x^8 (one byte)
    for _ in range(3):
        sq = _multmodp(sq, sq)
    while n:
        if n & 1:
            p = _multmodp(sq, p)
        n >>= 1
        sq = _multmodp(sq, sq)
    return p


def crc32_shift(crc_a: int, len_b: int) -> int:
    """The CRC-32 of A || zeros(len_b) XOR the CRC-32 of zeros(len_b), so crc32_shift(crc(A), |B|) ^ crc(B) is
    crc(A || B)."""
    return _multmodp(_x2nmodp(len_b), crc_a)
