"""GPU tests of the chunked deflate (csrc/nastar_deflate.cuh) and savez_compressed_device: kernel streams equal the
oracle's byte for byte (the whole corpus in one launch, and the MP-sized labels dataset), archives round-trip through
zipfile and np.load, both dataset loaders read a device-written dataset as the host-written one, two calls give the
same bytes in one launch each, every argument form works, a member above 4 GiB is ZIP64, and a batch with more chunks
than CTAs reuses the workspace slots."""
import io
import zipfile
import zlib

import numpy as np
import pytest
import torch

from oracle import deflate as D
from test_npz_cpu import CORPUS, _golden_labels

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    return torch.device("cuda:0")


def _kernel_streams(blobs, dev):
    """Every blob as one member with an empty head, in one launch: the kernel's raw streams and CRCs."""
    from neural_astar import _native

    data = [torch.tensor(np.frombuffer(b, np.uint8), device=dev) if b else None for b in blobs]
    head = torch.tensor(np.frombuffer(b"\x00", np.uint8), device=dev)
    d = np.zeros(len(blobs), _native.DEFLATE_DESC_DTYPE)
    d["head"] = head.data_ptr()
    d["head_len"] = 0
    d["data"] = [t.data_ptr() if t is not None else 0 for t in data]
    d["data_len"] = [len(b) for b in blobs]
    d["chunk0"] = np.concatenate([[0], np.cumsum(_native.deflate_chunk_counts(d["data_len"]))[:-1]])
    dd = torch.tensor(d.view(np.uint8), device=dev)
    n0 = _native.launch_count()
    out, off, ln, crc = _native.deflate(d, dd)
    torch.cuda.synchronize()
    assert _native.launch_count() - n0 == 1
    o = out.cpu().numpy()
    off, ln, crc = off.cpu().numpy(), ln.cpu().numpy(), crc.cpu().numpy().astype(np.uint32)
    return [o[a:a + n].tobytes() for a, n in zip(off, ln)], crc


def test_kernel_equals_oracle_on_corpus(dev):
    names = sorted(CORPUS)
    streams, crcs = _kernel_streams([CORPUS[k] for k in names], dev)
    for k, s, c in zip(names, streams, crcs):
        assert s == D.member(b"", CORPUS[k]), k
        assert zlib.decompress(s, -15) == CORPUS[k], k
        assert int(c) == zlib.crc32(CORPUS[k]), k


def test_kernel_equals_oracle_on_labels(dev):
    blobs = []
    for a in _golden_labels():
        b = io.BytesIO()
        np.save(b, a)
        blobs.append(b.getvalue())
    streams, _ = _kernel_streams(blobs, dev)
    for s, b in zip(streams, blobs):
        assert s == D.member(b"", b)


def _arrays(dev):
    rng = np.random.RandomState(3)
    base = torch.tensor(rng.rand(40, 70), dtype=torch.float32, device=dev)
    return dict(
        a=base, b=base.t(), c=torch.tensor(7.5, dtype=torch.float64, device=dev),
        d=torch.zeros((0, 4), dtype=torch.int64, device=dev), e=torch.tensor(rng.rand(1000) > 0.5, device=dev),
        f=torch.arange(300000, dtype=torch.int32, device=dev),
        g=torch.tensor(rng.randint(0, 255, 12345), dtype=torch.uint8, device=dev))


def test_round_trip_and_argument_forms(dev, tmp_path):
    from neural_astar import _native
    from neural_astar.utils.data import savez_compressed_device

    arrs = _arrays(dev)
    pos = list(arrs.values())[:2]
    kw = dict(list(arrs.items())[2:])
    p1, p2 = tmp_path / "x.npz", tmp_path / "y"
    n0 = _native.launch_count()
    savez_compressed_device(str(p1), *pos, **kw)
    assert _native.launch_count() - n0 == 1
    savez_compressed_device(str(p2), *pos, **kw)
    assert p1.read_bytes() == (tmp_path / "y.npz").read_bytes()
    assert zipfile.ZipFile(str(p1)).testzip() is None
    zf = zipfile.ZipFile(str(p1))
    z = np.load(str(p1))
    for k, t in list(zip(["arr_0", "arr_1"], pos)) + list(kw.items()):
        ref = t.cpu().numpy()
        b = io.BytesIO()
        np.save(b, ref.copy(order="C"))   # members hold C-order data, whatever the tensor's strides
        assert zf.read(k + ".npy") == b.getvalue(), k
        assert z[k].dtype == ref.dtype and np.array_equal(z[k], ref), k


def test_one_launch_and_two_explicit_waits(dev, tmp_path, monkeypatch):
    """One launch; the host waits twice, both explicitly: once for the sizes and CRCs, once for exactly the compressed
    bytes.  Sync debug mode "warn" reports synchronising operations; it may report the same one once only, so it must
    report no more than the two explicit waits."""
    from neural_astar import _native
    from neural_astar.utils.data import savez_compressed_device

    arrs = _arrays(dev)
    savez_compressed_device(str(tmp_path / "warm.npz"), **arrs)
    waits = []
    real = torch.cuda.Stream.synchronize
    monkeypatch.setattr(torch.cuda.Stream, "synchronize", lambda self: (waits.append(self), real(self))[1])
    n0 = _native.launch_count()
    import warnings

    with warnings.catch_warnings(record=True) as seen:
        warnings.simplefilter("always")
        torch.cuda.set_sync_debug_mode("warn")
        try:
            savez_compressed_device(str(tmp_path / "x.npz"), **arrs)
        finally:
            torch.cuda.set_sync_debug_mode("default")
    syncs = [w for w in seen if str(w.message).startswith("called a synchronizing CUDA operation")]
    assert _native.launch_count() - n0 == 1
    assert len(waits) == 2 and 1 <= len(syncs) <= len(waits), (len(waits), [str(w.message) for w in syncs])
    z = np.load(str(tmp_path / "x.npz"))
    assert all(np.array_equal(z[k], t.cpu().numpy()) for k, t in arrs.items())


def test_non_cuda_raises(dev):
    from neural_astar.utils.data import savez_compressed_device

    with pytest.raises(RuntimeError):
        savez_compressed_device(io.BytesIO(), np.zeros(3))


def test_slot_reuse_many_chunks(dev, tmp_path):
    from neural_astar.utils.data import savez_compressed_device

    n_sm = torch.cuda.get_device_properties(dev).multi_processor_count
    x = torch.arange(2 * n_sm * D.chunk_size() // 4 + 17, dtype=torch.int32, device=dev) % 251
    p = tmp_path / "big.npz"
    savez_compressed_device(str(p), x=x)
    got = np.load(str(p))["x"]
    assert np.array_equal(got, x.cpu().numpy())
    raw = io.BytesIO()
    np.save(raw, x.cpu().numpy())
    raw = raw.getvalue()
    head = raw[:len(raw) - x.numel() * 4]
    with zipfile.ZipFile(str(p)) as zf:
        info = zf.getinfo("x.npy")
        with open(p, "rb") as f:
            f.seek(info.header_offset + 30 + len("x.npy") + 20)
            assert f.read(info.compress_size) == D.member(head, raw[len(head):])


def test_dataset_loaders_read_device_file(dev, tmp_path):
    from neural_astar.utils.data import DeviceMazeDataset, MazeDataset, save_planning_dataset

    arrays = _golden_labels()
    host, devp = str(tmp_path / "h.npz"), str(tmp_path / "d.npz")
    splits_np = [arrays[0:4], arrays[4:8], arrays[8:12]]
    save_planning_dataset(host, *splits_np)
    save_planning_dataset(devp, *[[torch.tensor(a, device=dev) for a in s] for s in splits_np])
    zh, zd = np.load(host), np.load(devp)
    assert zh.files == zd.files
    for k in zh.files:
        assert np.array_equal(zh[k], zd[k]) and zh[k].dtype == zd[k].dtype
    import os

    assert os.path.getsize(devp) <= 1.10 * os.path.getsize(host)
    for split in ("train", "valid", "test"):
        a, b = MazeDataset(host, split), MazeDataset(devp, split)
        assert len(a) == len(b)
        for name in ("map_designs", "goal_maps", "opt_policies", "opt_dists"):
            u, v = getattr(a, name), getattr(b, name)
            assert u.dtype == v.dtype and np.array_equal(u, v), name
        for i in range(0, len(a), max(1, len(a) // 8)):
            np.random.seed(i)   # MazeDataset draws start maps with np.random
            ua = a[i]
            np.random.seed(i)
            for u, v in zip(ua, b[i]):
                assert np.array_equal(np.asarray(u), np.asarray(v))
        da, db = DeviceMazeDataset(host, split, device=dev), DeviceMazeDataset(devp, split, device=dev)
        assert len(da) == len(db)
        assert torch.equal(da.map_designs, db.map_designs) and torch.equal(da.goal_maps, db.goal_maps)
        for u, v in zip(da._tables, db._tables):   # the sampler's tables, built from the policies and distances
            assert torch.equal(u, v)


def test_zip64_member_over_4gib(dev, tmp_path):
    from neural_astar.utils.data import savez_compressed_device

    free, _ = torch.cuda.mem_get_info(dev)
    n = (1 << 32) + 4096
    if free < 3 * n:
        pytest.skip("needs ~13 GB of free device memory")
    x = torch.zeros((n,), dtype=torch.uint8, device=dev)
    p = tmp_path / "z.npz"
    savez_compressed_device(str(p), x)
    del x
    torch.cuda.empty_cache()
    with zipfile.ZipFile(str(p)) as zf:
        info = zf.getinfo("arr_0.npy")
        assert info.file_size > 1 << 32
        with zf.open("arr_0.npy") as f:
            head = f.read(128)
            assert head.startswith(b"\x93NUMPY")
            total, crc = len(head), zlib.crc32(head)
            while True:
                piece = f.read(1 << 26)
                if not piece:
                    break
                assert not any(piece)
                total += len(piece)
        assert total == info.file_size


def test_kernel_equals_oracle_on_bench_workloads(dev):
    """tools/npz_bench.py's workloads (MP, tiled 64x64 in float32 and float64, Config-5): in every array the first, a
    middle and the last chunk of its bytes, each as a member of one launch, equal the oracle's stream."""
    import os
    import sys

    sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tools"))
    from npz_bench import workloads

    C = D.chunk_size()
    for name, splits in workloads(dev):
        windows = []
        for t in (x for s in splits for x in s):
            raw = t.contiguous().reshape(-1).view(torch.uint8)
            n = raw.numel()
            last = (n - 1) // C * C
            for a in sorted({0, (n // C // 2) * C, last}):
                windows.append(raw[a:a + C].cpu().numpy().tobytes())
        streams, crcs = _kernel_streams(windows, dev)
        for w, s, c in zip(windows, streams, crcs):
            assert s == D.member(b"", w), name
            assert int(c) == zlib.crc32(w), name
