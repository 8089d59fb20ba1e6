"""CPU tests of the chunked deflate (oracle/deflate_oracle.c) and the host side of savez_compressed_device: the
oracle's streams inflate to their input on a seeded corpus, its archive of the golden maps' labels stays within 1.10x
np.savez_compressed, the host zip writer gives archives zipfile and np.load read (ZIP64 and > 65 535 members too),
the CRC-32 shift joins CRCs as zlib does, and the deflate ABI rejects bad arguments without a launch."""
import ctypes
import io
import os
import zipfile
import zlib

import numpy as np
import pytest

from oracle import deflate as D

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "inputs_mazes032_all1000.npz")


def corpus():
    rng = np.random.RandomState(1234)
    C = D.chunk_size()
    cases = {"empty": b"", "one": b"a", "chunk-1": bytes(rng.randint(0, 4, C - 1, dtype=np.uint8)),
             "chunk+1": bytes(rng.randint(0, 4, C + 1, dtype=np.uint8)),
             "65535": bytes(rng.randint(0, 2, 65535, np.uint8)),
             "65536": rng.bytes(65536), "zeros": bytes(600000), "random": rng.bytes(300000),
             "single": b"\x07" * 5000}
    for per in (1, 2, 3, 4, 8, 257, 32767, 32768, 32769):
        base = rng.bytes(per)
        cases[f"period{per}"] = (base * (120000 // per + 2))[:120000]
    fib = [1, 1]
    while len(fib) < 25:
        fib.append(fib[-1] + fib[-2])
    f = np.repeat(np.arange(25, dtype=np.uint8), fib)
    rng.shuffle(f)
    cases["fibonacci"] = f.tobytes()
    pol = np.zeros((40, 8, 1, 32, 32), np.float32)
    act = rng.randint(0, 8, (40, 32, 32))
    for k in range(8):
        pol[:, k, 0] = act == k
    cases["onehot32"] = pol.tobytes()
    cases["onehot64"] = pol.astype(np.float64).tobytes()
    return cases


CORPUS = corpus()


@pytest.mark.parametrize("name", sorted(CORPUS))
def test_oracle_round_trip(name):
    x = CORPUS[name]
    s = D.deflate(x)
    assert zlib.decompress(s, -15) == x
    assert len(s) <= D.bound(len(x))


def test_oracle_member_is_header_then_data():
    head, data = b"\x93NUMPY header", bytes(range(256)) * 3000
    assert zlib.decompress(D.member(head, data), -15) == head + data
    assert zlib.decompress(D.member(head, b""), -15) == head


def _golden_labels():
    from oracle import labels as LO

    z = np.load(GOLDEN)
    maps = np.unpackbits(z["obst_bits"], axis=1)[:, :1024].reshape(1000, 32, 32).astype(np.float32)
    goal = z["goal_idx"]
    if maps.reshape(1000, -1)[np.arange(1000), goal].min() == 0:
        maps = 1 - maps
    dists, _, action = LO.opt_labels(maps, goal)
    pol = np.zeros((1000, 8, 1, 32, 32), np.float32)
    for k in range(8):
        pol[:, k, 0] = action[:, 0] == k
    goals = np.zeros((1000, 1, 32, 32), np.float32)
    goals.reshape(1000, -1)[np.arange(1000), goal] = 1
    arrays = []
    for s in (slice(0, 800), slice(800, 900), slice(900, 1000)):
        arrays += [maps[s], goals[s], pol[s], dists[s]]
    return arrays


def test_oracle_ratio_on_golden_labels():
    arrays = _golden_labels()
    b = io.BytesIO()
    np.savez_compressed(b, *arrays)
    ours = 0
    for a in arrays:
        raw = io.BytesIO()
        np.save(raw, a)
        raw = raw.getvalue()
        head = raw[:len(raw) - a.nbytes]
        ours += len(D.member(head, raw[len(head):])) + 2 * (30 + len("arr_0.npy") + 20) + 46
    assert ours <= 1.10 * len(b.getvalue()), (ours, len(b.getvalue()))


def _zlib_chunks(raw: bytes) -> bytes:
    C = D.chunk_size()
    out = []
    for off in range(0, max(len(raw), 1), C):
        c = zlib.compressobj(6, zlib.DEFLATED, -15)
        out.append(c.compress(raw[off:off + C]))
        out.append(c.flush(zlib.Z_FULL_FLUSH if off + C < len(raw) else zlib.Z_FINISH))
    return b"".join(out)


def _archive(arrays, force_zip64=False):
    from neural_astar.utils import data as ud

    names = [f"arr_{i}.npy".encode() for i in range(len(arrays))]
    parts, offs, cs, us, crcs, pos = [], [], [], [], [], 0
    for name, a in zip(names, arrays):
        b = io.BytesIO()
        np.save(b, a)
        raw = b.getvalue()
        s = _zlib_chunks(raw)
        gap = ud._zip_local_header_bytes(name)
        parts += [bytes(gap), s]
        offs.append(pos + gap)
        pos += gap + len(s)
        cs.append(len(s))
        us.append(len(raw))
        crcs.append(zlib.crc32(raw))
    image = np.frombuffer(b"".join(parts), np.uint8).copy()
    tail = ud._zip_finish(image, names, offs, cs, us, crcs, force_zip64=force_zip64)
    return image.tobytes() + tail


@pytest.mark.parametrize("force_zip64", [False, True])
def test_zip_container_loads(force_zip64):
    rng = np.random.RandomState(0)
    arrays = [rng.rand(300, 300).astype(np.float32), np.zeros((0, 3), np.int64), np.array(7, np.int32),
              rng.rand(5) > 0.5, np.arange(600000, dtype=np.uint8)]
    f = io.BytesIO(_archive(arrays, force_zip64))
    assert zipfile.ZipFile(f).testzip() is None
    f.seek(0)
    z = np.load(f)
    for i, a in enumerate(arrays):
        got = z[f"arr_{i}"]
        assert got.dtype == a.dtype and got.shape == a.shape and np.array_equal(got, a)


def test_zip_container_many_members():
    arrays = [np.array([i], np.int32) for i in range(65537)]
    f = io.BytesIO(_archive(arrays))
    zf = zipfile.ZipFile(f)
    assert len(zf.namelist()) == 65537 and zf.testzip() is None
    f.seek(0)
    z = np.load(f)
    assert int(z["arr_65536"][0]) == 65536 and int(z["arr_0"][0]) == 0


def test_npy_header_matches_np_save():
    from neural_astar.utils import data as ud

    for a in (np.zeros((3, 4), np.float32), np.zeros((), np.float64), np.zeros((0,), bool),
              np.zeros((2, 1, 5), np.int64),
              np.zeros((7,), np.uint8), np.zeros((1, 2), np.int32)):
        b = io.BytesIO()
        np.save(b, a)
        assert ud._npy_header(a.dtype, a.shape) == b.getvalue()[:len(b.getvalue()) - a.nbytes]


@pytest.mark.parametrize("lb", [0, 1, 5, 65536, 262144, 10 ** 7 + 3])
def test_crc_shift_combines(lb):
    rng = np.random.RandomState(lb % 1000)
    a, b = rng.bytes(1000), (rng.bytes(lb) if lb < 10 ** 6 else bytes(lb))
    assert D.crc32_shift(zlib.crc32(a), len(b)) ^ zlib.crc32(b) == zlib.crc32(a + b)


def test_abi_rejections_without_launch():
    from neural_astar import _native

    try:
        L = _native.lib()
    except _native.NativeLibraryMissing:
        pytest.skip("engine not built")
    d = np.zeros(2, _native.DEFLATE_DESC_DTYPE)
    d["head"], d["head_len"], d["data"], d["data_len"], d["gap"] = 1 << 40, 100, 1 << 41, 1000, 60
    d["chunk0"] = [0, 2]
    ok_bound = int(L.nastar_b200_deflate_bound(d.ctypes.data, 2))
    assert ok_bound > 2 * 1100
    ws = int(L.nastar_b200_deflate_workspace_bytes(d.ctypes.data, 2))
    assert ws > 0
    out, offs, lens, crc, wsp, dd = 1 << 42, 1 << 43, (1 << 43) + 4096, (1 << 43) + 8192, 1 << 44, 1 << 45
    n0 = L.nastar_b200_launch_count()

    def call(desc, M=2, o=out, ob=ok_bound, of=offs, ln=lens, cr=crc, w=wsp, wb=ws, ddev=dd):
        return L.nastar_b200_deflate(desc.ctypes.data if desc is not None else None, ddev, M, o, ob, of, ln, cr, w,
                                     wb, None)

    bad = d.copy()
    bad["chunk0"] = [0, 1]
    assert call(bad) == 1
    bad = d.copy()
    bad["data_len"][1] = -1
    assert call(bad) == 1
    bad = d.copy()
    bad["gap"][0] = -5
    assert call(bad) == 1
    bad = d.copy()
    bad["data"][0] = 0
    assert call(bad) == 1
    assert call(None) == 1
    assert call(d, M=0) == 1
    assert call(d, o=None) == 1
    assert call(d, of=None) == 1
    assert call(d, ddev=None) == 1
    assert call(d, ln=offs + 8) == 1             # out_len overlaps out_off
    assert call(d, o=(1 << 41) + 10) == 1       # out overlaps member 0's data
    assert call(d, ob=-1) == 1
    assert call(d, ob=ok_bound - 1) == 4
    assert call(d, wb=ws - 1) == 4
    assert call(d, w=None) == 4
    assert call(d, w=out + 256) == 1            # the workspace overlaps out
    assert call(d, w=1 << 41) == 1              # the workspace overlaps member 0's data
    bad = d.copy()
    bad["head_len"][0] = D.chunk_size() + 1     # a head is one chunk
    assert call(bad) == 1
    edge = d.copy()
    edge["head_len"][0] = D.chunk_size()
    assert L.nastar_b200_deflate_bound(edge.ctypes.data, 2) > D.chunk_size()
    assert L.nastar_b200_deflate_bound(bad.ctypes.data, 2) == -1
    assert L.nastar_b200_deflate_workspace_bytes(bad.ctypes.data, 2) == 0
    assert L.nastar_b200_launch_count() == n0
