"""GPU tests of the .npz reader (utils.data.load_npz_device, nastar_b200_inflate; DESIGN.md §23): every member equals
np.load's (torch.equal, same dtype and shape) for random arrays of every supported dtype, stored and deflated, for the
files savez_compressed_device, save_planning_dataset and tools/make_sdd_dataset.py write, and for all of them in one
call; a corrupt member raises the error that names it while the other files of the call are still exact."""
import io
import os
import sys
import zipfile
import zlib

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SDD = os.path.join(ROOT, "tests", "golden", "sdd", "original")
DTYPES = ["|b1", "|u1", "|i1", "<i2", "<i4", "<i8", "<f2", "<f4", "<f8"]


@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    return torch.device("cuda:0")


def random_members(seed):
    rng = np.random.RandomState(seed)
    out = {}
    for i, dt in enumerate(DTYPES):
        shape = [(3, 5), (17,), (2, 3, 4), (64, 64, 3)][(i + seed) % 4]
        out[f"a{i}"] = rng.rand(*shape) < 0.5 if dt == "|b1" else (rng.rand(*shape) * 250 - 120).astype(dt)
        out[f"z{i}"] = np.zeros((0, 3), dt)          # zero-size
        out[f"s{i}"] = np.array(out[f"a{i}"].flat[0])  # 0-d
    out["big"] = rng.randint(0, 1000, 100000).astype(np.int64)     # 800 KB, more than one 256 KiB deflate chunk
    out["smooth"] = np.repeat(np.arange(300), 1000).astype(np.float32)   # long matches
    return out


def npz_bytes(members, compressed):
    f = io.BytesIO()
    (np.savez_compressed if compressed else np.savez)(f, **members)
    return f.getvalue()


def assert_equal_np_load(got, blob_or_path):
    want = np.load(io.BytesIO(blob_or_path) if isinstance(blob_or_path, bytes) else blob_or_path)
    assert list(got) == want.files
    for k in want.files:
        w = want[k]
        t = got[k]
        assert t.is_cuda and tuple(t.shape) == w.shape, k
        assert torch.equal(t.cpu(), torch.from_numpy(np.array(w))), k   # np.array keeps a 0-d array 0-d


@pytest.mark.parametrize("compressed", [False, True])
def test_random_members_equal_np_load(dev, compressed):
    from neural_astar import _native
    from neural_astar.utils.data import load_npz_device

    blobs = [npz_bytes(random_members(s), compressed) for s in range(3)]
    n0 = _native.launch_count()
    got = load_npz_device(blobs, dev)
    assert _native.launch_count() - n0 == 1
    for g, b in zip(got, blobs):
        assert_equal_np_load(g, b)
    base = got[0]["a0"].untyped_storage().data_ptr()
    for g in got:   # one buffer, each array 64-byte aligned
        for t in g.values():
            assert t.untyped_storage().data_ptr() == base and (t.data_ptr() - base) % 64 == 0


def device_files(dev, tmp):
    """Files of the repository's own writers: savez_compressed_device (chunked streams) and save_planning_dataset."""
    from neural_astar.utils.data import save_planning_dataset, savez_compressed_device

    rng = np.random.RandomState(7)
    a = str(tmp / "dev.npz")
    savez_compressed_device(a, torch.from_numpy(rng.rand(300, 300)).to(dev),
                            lab=torch.arange(5, device=dev), flag=torch.tensor(True, device=dev),
                            half=torch.from_numpy(rng.rand(40, 7).astype(np.float16)).to(dev))
    b = str(tmp / "planning.npz")
    splits = []
    for n in (6, 2, 3):
        maps = torch.from_numpy((rng.rand(n, 16, 16) > 0.3).astype(np.float32)).to(dev)
        goals = torch.zeros((n, 1, 16, 16), device=dev)
        pol = torch.from_numpy(rng.rand(n, 8, 1, 16, 16).astype(np.float32)).to(dev)
        dists = torch.from_numpy(-rng.randint(0, 50, (n, 1, 16, 16)).astype(np.float32)).to(dev)
        splits.append((maps, goals, pol, dists))
    save_planning_dataset(b, *splits)
    return [a, b]


def sdd_files(tmp):
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    import make_sdd_dataset

    save_dir = make_sdd_dataset.main(["--input-path", SDD, "--save-dir", str(tmp)])
    files = sorted(os.path.join(d, f) for d, _, fs in os.walk(save_dir) for f in fs if f.endswith(".npz"))
    assert len(files) == 21
    return files


def test_repository_writers_and_sdd_samples_in_one_call(dev, tmp_path):
    from neural_astar import _native
    from neural_astar.utils.data import load_npz_device

    files = device_files(dev, tmp_path) + sdd_files(tmp_path / "sdd")
    blobs = [npz_bytes(random_members(9), True), npz_bytes(random_members(10), False)]
    n0 = _native.launch_count()
    got = load_npz_device(files + blobs, dev)
    assert _native.launch_count() - n0 == 1
    for g, f in zip(got, files + blobs):
        assert_equal_np_load(g, f)
    sample = got[2]
    assert sample["image"].dtype == torch.uint8 and sample["label"].ndim == 0 and sample["length_ratio"].ndim == 0


def truncated_member_zip(members, cut):
    """A zip whose member `cut` has its deflate stream cut in half, with the central directory's sizes and CRC of the
    whole member (the host reads its header from the stream's start)."""
    from neural_astar.utils.data import _zip_finish, _zip_local_header_bytes

    names, streams, usizes, crcs = [], [], [], []
    for k, a in members.items():
        f = io.BytesIO()
        np.lib.format.write_array(f, a)
        raw = f.getvalue()
        c = zlib.compressobj(6, zlib.DEFLATED, -15)
        s = c.compress(raw) + c.flush()
        names.append((k + ".npy").encode())
        streams.append(s[:len(s) // 2] if k == cut else s)
        usizes.append(len(raw))
        crcs.append(zlib.crc32(raw))
    offs, pos = [], 0
    for n, s in zip(names, streams):
        pos += _zip_local_header_bytes(n)
        offs.append(pos)
        pos += len(s)
    image = np.zeros(pos, np.uint8)
    for o, s in zip(offs, streams):
        image[o:o + len(s)] = np.frombuffer(s, np.uint8)
    tail = _zip_finish(image, names, offs, [len(s) for s in streams], usizes, crcs)   # writes the local headers
    return image.tobytes() + tail


def test_corrupt_members_are_named_and_the_rest_is_exact(dev):
    from neural_astar.utils.data import load_npz_device

    rng = np.random.RandomState(11)
    good = [npz_bytes(random_members(1), True), npz_bytes(random_members(2), False)]
    # a flipped byte in the data of a stored member: its CRC-32 differs
    flipped = bytearray(npz_bytes(dict(x=rng.rand(50), y=rng.rand(40)), False))
    z = zipfile.ZipFile(io.BytesIO(bytes(flipped)))
    lh = z.getinfo("y.npy").header_offset
    nlen, elen = np.frombuffer(bytes(flipped[lh + 26:lh + 30]), "<u2")
    at = lh + 30 + int(nlen) + int(elen) + 200   # past the 128-byte .npy header, inside the 320 data bytes
    flipped[at] ^= 0x40
    cut = truncated_member_zip(dict(p=rng.rand(20), q=np.repeat(rng.rand(100), 50)), "q")
    with pytest.raises(ValueError) as e:
        load_npz_device([good[0], bytes(flipped), cut, good[1]], dev)
    msg = str(e.value)
    assert "<npz 1>: Bad CRC-32 for file 'y.npy'" in msg, msg
    assert "<npz 2>: member 'q.npy': corrupt deflate stream (stream ends early" in msg, msg
    assert "'x.npy'" not in msg and "'p.npy'" not in msg
    arrays = e.value.arrays
    assert_equal_np_load(arrays[0], good[0])
    assert_equal_np_load(arrays[3], good[1])
    assert torch.equal(arrays[1]["x"].cpu(), torch.from_numpy(np.load(io.BytesIO(bytes(flipped)))["x"]))
    assert torch.equal(arrays[2]["p"].cpu(), torch.from_numpy(np.load(io.BytesIO(cut))["p"]))


def test_refusals_happen_before_any_launch(dev):
    from neural_astar import _native
    from neural_astar.utils.data import load_npz_device

    f = io.BytesIO()
    np.savez(f, big_endian=np.arange(3, dtype=">i8"))
    n0 = _native.launch_count()
    with pytest.raises(ValueError, match=r"<npz 1>: member 'big_endian.npy': dtype '>i8' is not supported"):
        load_npz_device([npz_bytes(dict(a=np.zeros(3)), True), f.getvalue()], dev)
    assert _native.launch_count() == n0
    assert load_npz_device([], dev) == []
