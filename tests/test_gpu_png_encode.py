"""GPU tests of the PNG encoder (csrc/nastar_png_encode.cuh + the deflate kernel, utils.data.encode_pngs): every file
equals the oracle's (tests/png_encode_oracle.py) byte for byte on random, binary, uniform and gradient images from
1 x 1 to 2048 x 2048 (multi-chunk), as [B,H,W] batches and as one batch of mixed sizes; Pillow (CRC checks on) and
the repository's own decode_pngs read every file back to its input; a call makes 3 launches and 2 host waits;
save_pngs writes the same files; CPU tensors are refused."""
import functools
import warnings

import numpy as np
import pytest
import torch
from PIL import Image

import png_encode_oracle as P
from test_png_encode_cpu import images, pillow_decode

pytestmark = pytest.mark.gpu

SHAPES = [(1, 1), (1, 2048), (2048, 1), (7, 13), (128, 128), (256, 256), (1024, 1024), (2048, 2048)]
KINDS = ("random", "binary", "uniform", "gradient")


@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    return torch.device("cuda:0")


@functools.lru_cache(maxsize=None)
def oracle_file(H, W, kind):
    return P.encode(images(H, W)[kind])


@pytest.mark.parametrize("shape", SHAPES)
def test_batch_equals_oracle_and_decodes(dev, shape):
    from neural_astar.utils.data import decode_pngs, encode_pngs

    imgs = images(*shape)
    batch = torch.from_numpy(np.stack([imgs[k] for k in KINDS])).to(dev)
    files = encode_pngs(batch)
    assert len(files) == len(KINDS)
    for k, f in zip(KINDS, files):
        assert f == oracle_file(*shape, k), k
        assert np.array_equal(pillow_decode(f), imgs[k]), k
    groups, status = decode_pngs(files, device=dev)
    assert not status.any() and len(groups) == 1
    assert np.array_equal(groups[0][0], np.arange(len(KINDS)))
    assert torch.equal(groups[0][1], batch)


def test_mixed_sizes_in_one_call(dev):
    from neural_astar import _native
    from neural_astar.utils.data import encode_pngs

    order = [(s, k) for s in SHAPES for k in KINDS]
    np.random.RandomState(0).shuffle(order)
    planes = [torch.from_numpy(images(*s)[k]).to(dev) for s, k in order]
    n0 = _native.launch_count()
    files = encode_pngs(planes)
    assert _native.launch_count() - n0 == 3
    for (s, k), f, p in zip(order, files, planes):
        assert f == oracle_file(*s, k), (s, k)
    # the files were back to back on the device: every one is a whole PNG from signature to IEND
    assert all(f.startswith(P.SIGNATURE) and f.endswith(P.chunk(b"IEND", b"")) for f in files)


def test_three_launches_and_two_explicit_waits(dev, monkeypatch):
    from neural_astar import _native
    from neural_astar.utils.data import encode_pngs

    x = torch.from_numpy(np.stack([images(128, 128, seed=s)["binary"] for s in range(50)])).to(dev)
    encode_pngs(x)
    waits = []
    real = torch.cuda.Stream.synchronize
    monkeypatch.setattr(torch.cuda.Stream, "synchronize", lambda self: (waits.append(self), real(self))[1])
    n0 = _native.launch_count()
    with warnings.catch_warnings(record=True) as seen:
        warnings.simplefilter("always")
        torch.cuda.set_sync_debug_mode("warn")
        try:
            files = encode_pngs(x)
        finally:
            torch.cuda.set_sync_debug_mode("default")
    syncs = [w for w in seen if str(w.message).startswith("called a synchronizing CUDA operation")]
    assert _native.launch_count() - n0 == 3
    assert len(waits) == 2 and 1 <= len(syncs) <= len(waits), (len(waits), [str(w.message) for w in syncs])
    assert all(np.array_equal(pillow_decode(f), x[i].cpu().numpy()) for i, f in enumerate(files))


def test_save_pngs_and_argument_checks(dev, tmp_path):
    from neural_astar.utils.data import encode_pngs, save_pngs

    x = torch.from_numpy(np.stack([images(7, 13)[k] for k in KINDS])).to(dev)
    paths = [str(tmp_path / f"{k}.png") for k in KINDS]
    save_pngs(paths, x)
    for p, f in zip(paths, encode_pngs(x)):
        with open(p, "rb") as fh:
            assert fh.read() == f
    with Image.open(paths[0]) as im:
        im.verify()
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        encode_pngs(x.cpu())
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        encode_pngs([x[0], x[1].cpu()])
    with pytest.raises(ValueError):
        encode_pngs(torch.zeros((1, 2049, 4), dtype=torch.uint8, device=dev))
    with pytest.raises(TypeError):
        encode_pngs(torch.zeros((1, 4, 4), dtype=torch.float32, device=dev))
    with pytest.raises(ValueError):
        save_pngs(paths[:2], x)
    assert encode_pngs([]) == []
    # a non-contiguous batch encodes its values
    t = x.transpose(1, 2)
    assert [pillow_decode(f).tolist() for f in encode_pngs(t)] == [a.tolist() for a in t.cpu().numpy()]
