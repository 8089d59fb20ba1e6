"""CPU checks of the .npz reader (utils.data.load_npz_device, DESIGN.md §23): the host zip / .npy planner
(utils.data._npz_plan) reports what zipfile and np.lib.format report for files of np.savez, np.savez_compressed,
zipfile with data descriptors and the repository's own ZIP64 writer, refuses what the reader does not read, naming the
file and member; nastar_b200_inflate and nastar_b200_chamfer reject bad arguments before any launch; and the Chamfer
oracle (tests/chamfer_oracle.py) agrees with brute force."""
import io
import os
import struct
import subprocess
import zipfile
import zlib

import numpy as np
import pytest

import chamfer_oracle as co

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EINVAL, EUNSUPPORTED, EWORKSPACE = 1, 2, 4
DTYPES = ["|b1", "|u1", "|i1", "<i2", "<i4", "<i8", "<f2", "<f4", "<f8"]


def arrays(rng):
    out = {}
    for i, dt in enumerate(DTYPES):
        shape = [(3, 5), (7,), (2, 3, 4)][i % 3]
        out[f"a{i}"] = (rng.rand(*shape) * 200 - 100).astype(dt) if dt != "|b1" else rng.rand(*shape) < 0.5
    out["scalar"] = np.array(2.5)
    out["label"] = np.array(3, np.int64)
    out["empty"] = np.zeros((0, 2), np.float32)
    out["big"] = rng.randint(0, 7, 70000).astype(np.int32)   # > 256 KiB
    return out


def savez(kind, members):
    f = io.BytesIO()
    if kind == "savez":
        np.savez(f, **members)
    elif kind == "savez_compressed":
        np.savez_compressed(f, **members)
    elif kind == "descriptors":
        # a stream that cannot seek: zipfile writes each member's sizes in a data descriptor after it
        class Unseekable(io.RawIOBase):
            def __init__(self):
                self.buf = bytearray()

            def writable(self):
                return True

            def write(self, b):
                self.buf += b
                return len(b)

        u = Unseekable()
        with zipfile.ZipFile(u, "w", zipfile.ZIP_DEFLATED) as z:
            for k, a in members.items():
                with z.open(k + ".npy", "w", force_zip64=True) as m:
                    np.lib.format.write_array(m, a)
        return bytes(u.buf)
    elif kind == "zip64":
        return zip64_archive(members)
    return f.getvalue()


def zip64_archive(members):
    """The repository's own writer (_zip_finish with force_zip64=True) around zlib's raw deflate streams."""
    from neural_astar.utils.data import _zip_finish, _zip_local_header_bytes

    names, streams, usizes, crcs = [], [], [], []
    for k, a in members.items():
        f = io.BytesIO()
        np.lib.format.write_array(f, a)
        raw = f.getvalue()
        c = zlib.compressobj(6, zlib.DEFLATED, -15)
        names.append((k + ".npy").encode())
        streams.append(c.compress(raw) + c.flush())
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
    tail = _zip_finish(image, names, offs, [len(s) for s in streams], usizes, crcs, force_zip64=True)
    return image.tobytes() + tail


@pytest.mark.parametrize("kind", ["savez", "savez_compressed", "descriptors", "zip64"])
def test_planner_reports_what_zipfile_and_numpy_report(kind):
    from neural_astar.utils.data import _npz_plan

    members = arrays(np.random.RandomState(len(kind)))
    blob = savez(kind, members)
    plan = _npz_plan(blob, "f.npz")
    z = zipfile.ZipFile(io.BytesIO(blob))
    infos = z.infolist()
    assert [m[0] for m in plan] == [i.filename[:-4] for i in infos] == list(members)
    want_method = 0 if kind == "savez" else 8
    for m, info in zip(plan, infos):
        key, method, off, csize, usize, crc, descr, shape, hl = m
        assert (method, csize, usize, crc) == (want_method, info.compress_size, info.file_size, info.CRC)
        raw = z.read(info)
        comp = blob[off:off + csize]
        assert (comp if method == 0 else zlib.decompress(comp, -15)) == raw, key
        f = io.BytesIO(raw)
        version = np.lib.format.read_magic(f)
        read = np.lib.format.read_array_header_1_0 if version == (1, 0) else np.lib.format.read_array_header_2_0
        shp, fortran, dt = read(f)
        assert (shape, descr, hl) == (shp, dt.str, f.tell()), key
        a = np.frombuffer(raw[hl:], dtype=descr).reshape(shape)
        assert np.array_equal(a, members[key]), key


def test_planner_reads_npy_format_versions_2_and_3():
    from neural_astar.utils.data import _npz_plan

    a = np.arange(12, dtype=np.int16).reshape(3, 4)
    f = io.BytesIO()
    hls = []
    with zipfile.ZipFile(f, "w", zipfile.ZIP_DEFLATED) as z:
        for v in ((2, 0), (3, 0)):
            g = io.BytesIO()
            np.lib.format.write_array(g, a, version=v)
            z.writestr(f"v{v[0]}.npy", g.getvalue())
            hls.append(len(g.getvalue()) - a.nbytes)
    plan = _npz_plan(f.getvalue())
    assert [(m[0], m[6], m[7], m[8]) for m in plan] == [("v2", "<i2", (3, 4), hls[0]), ("v3", "<i2", (3, 4), hls[1])]


def raw_npy(a):
    f = io.BytesIO()
    np.lib.format.write_array(f, a, allow_pickle=True)
    return f.getvalue()


def one_member_zip(name, raw, method=zipfile.ZIP_DEFLATED):
    f = io.BytesIO()
    with zipfile.ZipFile(f, "w", method) as z:
        z.writestr(name, raw)
    return f.getvalue()


def with_npy_header(text: bytes, body=b""):
    text = text + b" " * (-(len(text) + 11) % 64) + b"\n"
    return b"\x93NUMPY\x01\x00" + struct.pack("<H", len(text)) + text + body


def encrypted():
    blob = bytearray(one_member_zip("x.npy", raw_npy(np.zeros(3))))
    cd = blob.rfind(b"PK\x01\x02")
    blob[cd + 8] |= 1   # the central directory's "encrypted" flag
    return bytes(blob)


@pytest.mark.parametrize("blob,member,why", [
    (lambda: one_member_zip("x.npy", raw_npy(np.zeros(3)), zipfile.ZIP_BZIP2), "x.npy", "compression method 12"),
    (lambda: one_member_zip("x.npy", raw_npy(np.zeros(3)), zipfile.ZIP_LZMA), "x.npy", "compression method 14"),
    (encrypted, "x.npy", "encrypted"),
    (lambda: one_member_zip("o.npy", raw_npy(np.array([1, "a"], dtype=object))), "o.npy", "dtype '|O'"),
    (lambda: one_member_zip("b.npy", raw_npy(np.arange(4, dtype=">i4"))), "b.npy", "dtype '>i4'"),
    (lambda: one_member_zip("s.npy", raw_npy(np.zeros(2, dtype=[("a", "<i4")]))), "s.npy", "dtype"),
    (lambda: one_member_zip("u.npy", raw_npy(np.zeros(2, dtype="<u4"))), "u.npy", "dtype '<u4'"),
    (lambda: one_member_zip("f.npy", raw_npy(np.asfortranarray(np.zeros((2, 3))))), "f.npy", "Fortran"),
    (lambda: one_member_zip("t.txt", b"hello"), "t.txt", "not a .npy member"),
    (lambda: one_member_zip("n.npy", b"\x93NUMPY\x04\x00" + b"\x00" * 60), "n.npy", "format 1, 2 or 3"),
    (lambda: one_member_zip("h.npy", with_npy_header(b"{'descr': '<f8', 'fortran_order': False, 'shape': (3,), }")),
     "h.npy", "does not match"),
])
def test_planner_refusals_name_file_and_member(blob, member, why):
    from neural_astar.utils.data import _npz_plan

    with pytest.raises(ValueError) as e:
        _npz_plan(blob(), "dir/sample.npz")
    msg = str(e.value)
    assert msg.startswith("dir/sample.npz: ") and repr(member) in msg and why in msg, msg


def test_planner_refuses_files_that_are_not_zips():
    from neural_astar.utils.data import _npz_plan

    with pytest.raises(ValueError, match="^x.npz: not a zip file"):
        _npz_plan(b"PK\x03\x04" + b"\x00" * 40, "x.npz")
    blob = one_member_zip("x.npy", raw_npy(np.zeros(300)))
    with pytest.raises(ValueError, match="^x.npz: "):
        _npz_plan(blob[:40] + blob[-60:], "x.npz")


# ---- the C ABI ----------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def native():
    subprocess.check_call(["make", "-C", os.path.join(ROOT, "neural-astar_b200"), "-s", "all"])
    from neural_astar import _native

    return _native


def _desc(native, n=3, **kw):
    d = np.zeros(n, native.INFLATE_DESC_DTYPE)
    d["in_off"], d["in_len"] = np.arange(n) * 100, 100
    d["out_off"], d["out_len"], d["method"] = np.arange(n) * 128, 128, 8
    for k, v in kw.items():
        d[k] = v
    return d


def _inflate(native, d, data_bytes=300, out_bytes=384, ws_bytes=256, **ptrs):
    args = dict(data=0x10000, desc_dev=0x20000, out=0x30000, status=0x40000, crc=0x50000, ws=0x60000)
    args.update(ptrs)
    return native.lib().nastar_b200_inflate(args["data"], data_bytes, d.ctypes.data if d is not None else None,
                                            args["desc_dev"], len(d) if d is not None else 1, args["out"], out_bytes,
                                            args["status"], args["crc"], args["ws"], ws_bytes, None)


@pytest.mark.parametrize("case,status", [
    (dict(data=None), EINVAL), (dict(desc_dev=None), EINVAL), (dict(out=None), EINVAL), (dict(status=None), EINVAL),
    (dict(crc=None), EINVAL), (dict(kw=dict(method=9)), EINVAL), (dict(kw=dict(method=12)), EINVAL),
    (dict(kw=dict(in_len=-1)), EINVAL), (dict(kw=dict(out_len=-1)), EINVAL), (dict(data_bytes=299), EINVAL),
    (dict(out_bytes=383), EINVAL), (dict(kw=dict(in_off=-1)), EINVAL), (dict(kw=dict(method=0)), EINVAL),
    (dict(kw=dict(out_off=[0, 100, 256])), EINVAL), (dict(kw=dict(out_off=[256, 128, 0])), EINVAL),
    (dict(ws=None), EWORKSPACE), (dict(ws_bytes=255), EWORKSPACE),
])
def test_inflate_rejects_without_launch(native, case, status):
    L = native.lib()
    before = L.nastar_b200_launch_count()
    d = _desc(native, **case.pop("kw", {}))
    assert _inflate(native, d, **case) == status
    assert L.nastar_b200_launch_count() == before, "a rejected call launched something"


def test_inflate_rejects_null_descriptors_and_empty_batches(native):
    L = native.lib()
    before = L.nastar_b200_launch_count()
    assert _inflate(native, None) == EINVAL
    d = _desc(native)
    assert L.nastar_b200_inflate(0x10000, 300, d.ctypes.data, 0x20000, 0, 0x30000, 384, 0x40000, 0x50000, 0x60000,
                                 256, None) == EINVAL
    assert L.nastar_b200_launch_count() == before


@pytest.mark.parametrize("args,status", [
    ((0, 2, 8, 8, 0x20000), EINVAL), ((0x10000, 2, 8, 8, 0), EINVAL), ((0x10000, 0, 8, 8, 0x20000), EINVAL),
    ((0x10000, 2, 0, 8, 0x20000), EINVAL), ((0x10000, 2, 8, -1, 0x20000), EINVAL),
    ((0x10000, 2, 1025, 8, 0x20000), EUNSUPPORTED), ((0x10000, 2, 8, 1025, 0x20000), EUNSUPPORTED),
])
def test_chamfer_rejects_without_launch(native, args, status):
    L = native.lib()
    before = L.nastar_b200_launch_count()
    assert L.nastar_b200_chamfer(*args, None, 0, None) == status
    assert L.nastar_b200_launch_count() == before


def test_chamfer_workspace_only_for_maps_beyond_shared_memory(native):
    L = native.lib()
    assert L.nastar_b200_chamfer_workspace_bytes(4096, 64, 64) == 0
    assert L.nastar_b200_chamfer_workspace_bytes(100, 200, 37) == 0
    big = L.nastar_b200_chamfer_workspace_bytes(2, 1024, 1024)
    assert big >= 2 * 1024 * 1024 * 2
    assert L.nastar_b200_chamfer_workspace_bytes(0, 64, 64) == 0
    assert L.nastar_b200_chamfer_workspace_bytes(1, 2048, 64) == 0
    before = L.nastar_b200_launch_count()
    assert L.nastar_b200_chamfer(0x10000, 2, 1024, 1024, 0x20000, None, 0, None) == EWORKSPACE
    assert L.nastar_b200_chamfer(0x10000, 2, 1024, 1024, 0x20000, 0x30000, big - 1, None) == EWORKSPACE
    assert L.nastar_b200_launch_count() == before


# ---- the Chamfer oracle -------------------------------------------------------------------------------------------
def test_chamfer_oracle_equals_brute_force():
    rng = np.random.RandomState(0)
    for H, W in ((1, 1), (1, 9), (7, 13), (16, 16), (23, 5)):
        a = rng.rand(6, H, W) < 0.3
        b = rng.rand(6, H, W) < 0.2
        a[0], b[1] = False, False   # empty sets
        np.testing.assert_allclose(co.chamfer(a, b), co.chamfer_brute(a, b), rtol=1e-13, equal_nan=True)


def test_chamfer_oracle_swaps_directions_and_is_zero_on_equal_masks():
    rng = np.random.RandomState(1)
    a = (rng.rand(5, 1, 12, 9) < 0.3).astype(np.float32)
    b = (rng.rand(5, 1, 12, 9) < 0.3).astype(np.float32)
    a[:, :, 0, 0] = b[:, :, -1, -1] = 1
    assert np.array_equal(co.chamfer(a, b), co.chamfer(b, a)[:, ::-1])
    assert np.array_equal(co.chamfer(a, a), np.zeros((5, 2)))
    e = co.chamfer(np.zeros((2, 4, 4)), np.ones((2, 4, 4)))
    assert np.isnan(e).all()
    one = np.zeros((1, 5, 5)); one[0, 0, 0] = 1
    other = np.zeros((1, 5, 5)); other[0, 3, 4] = 1
    assert np.array_equal(co.chamfer(one, other), [[5.0, 5.0]])
