"""The encoder's hand-written kernels checked bit for bit (helpers in tests/encoder_exact_oracle.py).

  exact     conv3x3_head_taps on dyadic operands whose every product and partial sum is exact in fp32, so the fp64
            taps are the only correct output: every tile width, ragged maps, every kind of schedule round, B = 1 and
            the flagship batch; then the same convolution with random fp32 bias and head weights, within the bound of
            the bias add and the fp32 head sum alone;
  tf32      which conversion the tensor cores apply to fp32 operands of a TF32 wgmma, probed one product at a time;
  placement conv3x3_head_taps on random fp32 data gives a map the same bits wherever it lands in a batch, and a map
            the same bits as its zero extension to a wider tile class or more rows;
  replays   head_taps<C> and conv1_marks bit-equal to a CPU replay of their fp32 operation sequence.

Batch sizes for the fused kernel's schedule assume what its occupancy query gives on an H100 (one CTA per SM, so
SMs / 2 clusters of 2); the tile-count sweep in test_gpu_engine_schedules.py covers every other cluster count.
"""
import functools

import numpy as np
import pytest
import torch

import encoder_exact_oracle as eo

pytestmark = pytest.mark.gpu
WIDTH_CLASSES = (8, 16, 32, 64)
RAGGED_W = {8: 5, 16: 12, 32: 27, 64: 50}


@pytest.fixture(scope="module")
def native():
    from neural_astar import _native

    _native.lib()
    return _native


@pytest.fixture(scope="module")
def sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


# ------------------------------------------------------------------------------------------------ schedule helpers
def _round_kind(T, nC):
    """conv3x3_head_kernel's schedule for T tiles on nC clusters (ch_tile): whole rounds of 2 nC tiles, then a tail of
    at most nC tiles split into half tiles, or a longer tail run as one more full round."""
    tail = T % (2 * nC)
    return "full" if tail == 0 else "half" if tail <= nC else "extra"


def _batches(sms, tiles_per_map):
    """{kind: B}: two full rounds, plus nothing, a half-tile tail, or a tail run as an extra full round."""
    nC = sms // 2
    out = {}
    for kind, tail in (("full", 0), ("half", nC // 2), ("extra", nC + nC // 2)):
        B = -(-(4 * nC + tail) // tiles_per_map)
        assert _round_kind(B * tiles_per_map, nC) == kind
        out[kind] = B
    return out


def _tiles_per_map(H, W):
    R = 128 // next(wp for wp in WIDTH_CLASSES if W <= wp)
    return -(-H // R)


def _first_mismatch(got, want, what="tap"):
    """None if got == want element for element, else the first wrong (map, y, x, tap) with got and want."""
    bad = (got.double() != want.double()) | torch.isnan(got)
    if not bool(bad.any()):
        return None
    b, y, x, k = bad.nonzero()[0].tolist()
    return (f"{int(bad.sum())} wrong; first at map {b}, y {y}, x {x}, {what} {k}: got {float(got[b, y, x, k])!r}, "
            f"want {float(want[b, y, x, k])!r}")


def _run(native, x, w, b, hw):
    """conv3x3_head_taps into a NaN-filled buffer with a guard after it: unwritten taps stay NaN, stray writes show."""
    B, _, H, W = x.shape
    n = B * H * W * 9
    buf = torch.full((n + 64,), float("nan"), device="cuda")
    out = native.conv3x3_head_taps(x, w, b, hw, out=buf[:n].view(B, H, W, 9))
    assert bool(torch.isnan(buf[n:]).all()), "conv3x3_head_taps wrote past its output"
    return out


@functools.lru_cache(maxsize=4)
def _exact(B, H, W, seed):
    return eo.exact_operands(B, H, W, seed)


# ------------------------------------------------------------------------------------ a. exact operands, bit for bit
def _exact_cases():
    cases = []
    for wp in WIDTH_CLASSES:
        R = 128 // wp
        cases += [(wp, (R, wp)), (wp, (R + 1, RAGGED_W[wp]))]
    return cases


@pytest.mark.parametrize("wp,shape", _exact_cases(), ids=lambda v: "x".join(map(str, v)) if isinstance(v, tuple) else f"wp{v}")
def test_fused_taps_exact_operands_every_schedule(native, sms, wp, shape):
    """R x Wp maps (one tile each) and R + 1 rows of a ragged width (two tiles per map, the second with one valid row,
    so half tiles and partial columns land past the edge), at B = 1 and at batches that end in full rounds only, in a
    half-tile tail and in a tail run as an extra full round.  Every tap must equal the exact fp64 result."""
    H, W = shape
    batches = _batches(sms, _tiles_per_map(H, W))
    Bmax = max(batches.values())
    x, w, b, hw, want, _ = _exact(Bmax, H, W, seed=wp * 100 + W)
    for kind, B in [("single map", 1)] + sorted(batches.items()):
        got = _run(native, x[:B], w, b, hw)
        bad = _first_mismatch(got, want[:B])
        assert bad is None, f"{H}x{W}, B = {B} ({kind}): {bad}"


def test_fused_taps_exact_operands_flagship(native):
    """The flagship batch, 100 maps of 32x32: 800 tiles, whole rounds and a half-tile tail on an H100."""
    x, w, b, hw, want, _ = _exact(100, 32, 32, seed=1)
    bad = _first_mismatch(_run(native, x, w, b, hw), want)
    assert bad is None, bad


@pytest.mark.parametrize("B,H,W", [(100, 32, 32), (3, 20, 27), (2, 64, 64)])
def test_fused_taps_exact_conv_random_fp32_epilogue(native, B, H, W):
    """x and w exact as above, so the tensor cores' pre-activations d are exact; bias and head weights random fp32.
    What remains is the kernel's epilogue: fl(d + bias) loses at most 2^-24 relu(d + bias) (a negative sum stays
    negative and ReLU gives 0 either way), and the 256-channel head sum is 66 fp32 roundings (64 FMAs per lane, two
    cross-lane adds): |tap - want| <= sum_c |hw| relu(d + bias) (2^-24 + gamma_66 (1 + 2^-24))."""
    x, w, _, _, _, _ = _exact(B, H, W, seed=B + H + W)
    g = torch.Generator(device="cpu").manual_seed(B * H)
    b = (torch.randn(256, generator=g) * 0.5).cuda()
    hw = (torch.randn(256, 9, generator=g) * 0.05).numpy().astype(np.float32)
    hwd = torch.from_numpy(hw).double().cuda()
    d = torch.nn.functional.conv2d(x.double(), w.double(), padding=1)
    a = torch.relu(d + b.double().view(1, -1, 1, 1))
    want = torch.einsum("bchw,ck->bhwk", a, hwd)
    g66 = eo.HEAD_ROUNDINGS * 2.0 ** -24 / (1 - eo.HEAD_ROUNDINGS * 2.0 ** -24)
    bound = torch.einsum("bchw,ck->bhwk", a, hwd.abs()) * (2.0 ** -24 + g66 * (1 + 2.0 ** -24)) + 1e-30
    got = _run(native, x, w, b, hw)
    ratio = float(((got.double() - want).abs() / bound).max())
    print(f"B={B} {H}x{W}: max error / epilogue bound = {ratio:.3f}")
    assert ratio <= 1.0


# ---------------------------------------------------------------------------------------- b. TF32 conversion probe
def _full_mantissas(rng, n):
    """Positive fp32 values in [1/8, 8) with all 23 mantissa bits random."""
    bits = (rng.randint(124, 130, n).astype(np.uint32) << np.uint32(23)) | rng.randint(0, 1 << 23, n).astype(np.uint32)
    return bits.view(np.float32)


def _mode_of(got, val):
    """Which conversions explain got == |tf32(val)| for every probe; and whether any probe tells them apart."""
    val = np.abs(val)
    match = {m: got == eo.tf32(val, m) for m in ("trunc", "rne")}
    fits = [m for m in match if match[m].all()]
    counts = {m: int(match[m].sum()) for m in match}
    return fits, counts, int((eo.tf32(val, "trunc") != eo.tf32(val, "rne")).sum())


def test_tf32_operand_conversion_mode(native):
    """Single-product outputs: bias 0, and one-hot head columns, so tap k of a pixel is relu(one product) exactly.
      A operand: 9 input channels carry full-mantissa values, each read by one output channel through a unit centre
      weight (-1 for the channels whose values are negative), so tap k = |tf32(x[p][ci_k])|: 8 maps x 32 x 32 x 9.
      B operand: impulses of +-1 at every third pixel, each in its own input channel; the 9 read-out channels' weights
      have full mantissas (negative for the channels hit by -1), so the 3x3 pixels around an impulse read
      |tf32(w[c_k][ky][kx][ci])| in their 9 taps: 2 maps x 100 impulses x 81.
    Every probe of both operands must follow one conversion, the same for both, and it must be eo.TF32_MODE."""
    rng = np.random.RandomState(19)
    cout = np.arange(9) * 28 + 5                       # read-out channels in both halves of N
    hw = np.zeros((256, 9), np.float32)
    hw[cout, np.arange(9)] = 1.0
    b = torch.zeros(256, device="cuda")

    # A operand
    B, H, W = 8, 32, 32
    cin = np.arange(9) * 14 + 3                        # input channels in every 32-channel chunk
    sign = np.where(np.arange(9) % 2 == 0, 1.0, -1.0).astype(np.float32)
    xa = np.zeros((B, H, W, 128), np.float32)
    vals = _full_mantissas(rng, B * H * W * 9).reshape(B, H, W, 9) * sign
    xa[..., cin] = vals
    wa = np.zeros((256, 128, 3, 3), np.float32)
    wa[cout, cin, 1, 1] = sign
    x = torch.from_numpy(xa).cuda().permute(0, 3, 1, 2).contiguous(memory_format=torch.channels_last)
    w = torch.from_numpy(wa).cuda().contiguous(memory_format=torch.channels_last)
    got_a = native.conv3x3_head_taps(x, w, b, hw).cpu().numpy()
    fits_a, counts_a, split_a = _mode_of(got_a, vals)

    # B operand
    B, H, W = 2, 32, 32
    pos = np.arange(10) * 3 + 1
    xb = np.zeros((B, H, W, 128), np.float32)
    ci = (np.arange(B * 100).reshape(B, 10, 10)) % 128
    imp = np.where(ci < 64, 1.0, -1.0).astype(np.float32)
    bi, iy, ix = np.meshgrid(np.arange(B), np.arange(10), np.arange(10), indexing="ij")
    xb[bi, pos[iy], pos[ix], ci] = imp
    wb = np.zeros((256, 128, 3, 3), np.float32)
    wv = _full_mantissas(rng, 9 * 128 * 9).reshape(9, 128, 3, 3)
    wv[:, 64:] *= -1
    wb[cout] = wv
    x = torch.from_numpy(xb).cuda().permute(0, 3, 1, 2).contiguous(memory_format=torch.channels_last)
    w = torch.from_numpy(wb).cuda().contiguous(memory_format=torch.channels_last)
    got_b = native.conv3x3_head_taps(x, w, b, hw).cpu().numpy()
    # pixel (y, x) < 30 lies next to the impulse at (3 (y // 3) + 1, 3 (x // 3) + 1) and reads w[.][ky][kx] with
    # ky - 1 = impulse y - y; rows and columns 30, 31 see no impulse
    yy, xx = np.meshgrid(np.arange(30), np.arange(30), indexing="ij")
    ky, kx = (yy // 3) * 3 + 1 - yy + 1, (xx // 3) * 3 + 1 - xx + 1
    c_at = ci[:, yy // 3, xx // 3]                                       # [B, 30, 30]
    want_w = wv[np.arange(9)[None, None, None, :], c_at[..., None], ky[None, ..., None], kx[None, ..., None]]
    assert not got_b[:, 30:].any() and not got_b[:, :, 30:].any()
    fits_b, counts_b, split_b = _mode_of(got_b[:, :30, :30], want_w)

    print(f"TF32 operand conversion: A operand fits {fits_a} ({counts_a} of {got_a.size}, {split_a} probes tell the "
          f"modes apart), B operand fits {fits_b} ({counts_b} of {want_w.size}, {split_b} tell them apart)")
    assert split_a > 0 and split_b > 0
    assert len(fits_a) == 1 and fits_a == fits_b, "the two operands are not converted by one rule"
    assert fits_a[0] == eo.TF32_MODE, f"observed {fits_a[0]!r}, eo.TF32_MODE says {eo.TF32_MODE!r}"


# -------------------------------------------------------------------------------- d. placement and zero extension
def _random_problem(B, H, W, seed):
    g = torch.Generator(device="cpu").manual_seed(seed)
    x = torch.randn(B, 128, H, W, generator=g) * (torch.rand(B, 128, H, W, generator=g) > 0.3)
    w = torch.randn(256, 128, 3, 3, generator=g) * 0.03
    b = torch.randn(256, generator=g) * 0.1
    hw = (torch.randn(256, 9, generator=g) * 0.05).numpy().astype(np.float32)
    return (x.cuda().contiguous(memory_format=torch.channels_last), w.cuda().contiguous(memory_format=torch.channels_last),
            b.cuda(), hw)


@pytest.mark.parametrize("H,W", [(4, 32), (9, 12), (32, 32), (3, 50)])
def test_fused_taps_same_bits_at_every_batch_index(native, sms, H, W):
    """Random fp32 data, no tolerance: one map's taps computed alone equal its taps at every index of batches made of
    copies of it, for every round and tail kind (and the flagship B = 100), so full tiles, half tiles of either CTA
    of a cluster, and every CTA and round give a map the same bits."""
    x, w, b, hw = _random_problem(1, H, W, seed=H * 64 + W)
    alone = _run(native, x, w, b, hw)
    assert bool(torch.isfinite(alone).all())
    for kind, B in sorted(_batches(sms, _tiles_per_map(H, W)).items()) + [("flagship batch", 100)]:
        got = _run(native, x.repeat(B, 1, 1, 1).contiguous(memory_format=torch.channels_last), w, b, hw)
        same = (got == alone).flatten(1).all(1)
        assert bool(same.all()), (f"{H}x{W}, B = {B} ({kind}): maps {same.logical_not().nonzero().flatten().tolist()[:10]}"
                                  f" differ from the map computed alone: {_first_mismatch(got, alone.expand_as(got))}")


@pytest.mark.parametrize("H,W,bigger", [
    (5, 7, [(5, 8), (5, 12), (5, 27), (5, 64), (6, 7), (21, 7), (64, 64)]),
    (9, 12, [(9, 16), (9, 32), (9, 50), (17, 12), (40, 33)]),
    (20, 27, [(20, 32), (20, 64), (21, 27), (64, 27)]),
    (3, 50, [(3, 64), (4, 50), (64, 64)]),
])
def test_fused_taps_same_bits_as_zero_extension(native, H, W, bigger):
    """Random fp32 data, no tolerance: a map and its zero extension to a wider tile class or to more rows give the same
    taps on the original map, so the convolution's padding (TMA's out-of-bounds fill) and explicit zeros agree and
    the tile geometry (Wp, R) does not enter the arithmetic."""
    x, w, b, hw = _random_problem(3, H, W, seed=H * 64 + W + 1)
    base = _run(native, x, w, b, hw)
    for H2, W2 in bigger:
        xz = torch.nn.functional.pad(x, (0, W2 - W, 0, H2 - H)).contiguous(memory_format=torch.channels_last)
        got = _run(native, xz, w, b, hw)[:, :H, :W]
        bad = _first_mismatch(got, base)
        assert bad is None, f"{H}x{W} zero-extended to {H2}x{W2}: {bad}"


# ---------------------------------------------------------------------------------- e, f. replays of the glue kernels
def _replay_mismatch(got, want, idx, what):
    bad = ~((got == want) | (np.isnan(got) & np.isnan(want)))
    if not bad.any():
        return None
    i, c = np.argwhere(bad)[0]
    return (f"{int(bad.sum())} wrong; first at pixel {int(idx[i])}, {what} {c}: got {got[i, c]!r} "
            f"(0x{got[i, c:c + 1].view(np.uint32)[0]:08x}), want {want[i, c]!r} (0x{want[i, c:c + 1].view(np.uint32)[0]:08x})")


def _sample(P, n, rng):
    """n pixel indices out of P: random ones, the first and the last 40 (the ragged last 32-pixel group)."""
    return np.unique(np.concatenate([rng.randint(0, P, n), np.arange(40), np.arange(P - 40, P)]))


@pytest.mark.parametrize("C", [16, 32, 64, 128, 256])
def test_head_taps_bit_equal_to_replay(native, sms, C):
    """head_taps<C> against head_taps_replay: every pixel of a ragged P (3 x 37 x 31 = 3441, not a multiple of 32), and
    4 096 sampled pixels (plus the first and last 40) of a P past the capped grid (16 CTAs per SM of 4 warps of 32
    pixels), where warps take further 32-pixel groups and prefetch across them."""
    rng = np.random.RandomState(C)
    wgt = (rng.randn(C, 9) / C ** 0.5).astype(np.float32)
    cap = sms * 16 * 4 * 32
    n_big = cap // (61 * 61) + 2
    n_big += 1 - n_big % 2
    for B, H, W, n in ((3, 37, 31, None), (n_big, 61, 61, 4096)):
        P = B * H * W
        assert P % 32
        torch.manual_seed(C + B)
        x = torch.randn(B, C, H, W, device="cuda").contiguous(memory_format=torch.channels_last)
        got = native.head_taps(x, wgt).view(P, 9)
        idx = np.arange(P) if n is None else _sample(P, n, rng)
        it = torch.from_numpy(idx).cuda()
        xs = x.permute(0, 2, 3, 1).reshape(P, C)[it].cpu().numpy()
        want = eo.head_taps_replay(xs, wgt)
        bad = _replay_mismatch(got[it].cpu().numpy(), want, idx, "tap")
        assert bad is None, f"C = {C}, P = {P}: {bad}"


def _conv1_problem(B, H, W, seed, device="cuda"):
    """Non-binary maps, and start / goal planes with a few non-binary marks (start + goal is rounded once)."""
    g = torch.Generator(device="cpu").manual_seed(seed)
    maps = torch.rand(B, 1, H, W, generator=g) * 2 - 0.5
    start = torch.rand(B, 1, H, W, generator=g) * (torch.rand(B, 1, H, W, generator=g) > 0.9)
    goal = torch.rand(B, 1, H, W, generator=g) * (torch.rand(B, 1, H, W, generator=g) > 0.9)
    w = (torch.randn(9, 2, 32, generator=g) * 0.3).numpy()
    bias = (torch.randn(32, generator=g) * 0.1).numpy()
    return maps.to(device), start.to(device), goal.to(device), w, bias


@pytest.mark.parametrize("B,H,W", [(1, 5, 3), (4, 3, 5), (3, 20, 27), (2, 33, 64), (2, 64, 64)])
def test_conv1_marks_bit_equal_to_replay(native, B, H, W):
    """conv1_marks against conv1_marks_replay on every pixel, with contiguous planes and with start / goal given as
    strided views into one stacked buffer."""
    maps, start, goal, w, bias = _conv1_problem(B, H, W, seed=B * 1000 + H * 10 + W)
    want = eo.conv1_marks_replay(maps.cpu().numpy(), start.cpu().numpy(), goal.cpu().numpy(), w, bias).reshape(-1, 32)
    idx = np.arange(B * H * W)
    got = native.conv1_marks(maps, start, goal, w, bias).permute(0, 2, 3, 1).reshape(-1, 32).cpu().numpy()
    bad = _replay_mismatch(got, want, idx, "channel")
    assert bad is None, f"{B}x{H}x{W}: {bad}"
    stacked = torch.stack((start, maps, goal), 2)            # [B, 1, 3, H, W]: start and goal are strided views
    s, gl = stacked[:, :, 0], stacked[:, :, 2]
    assert s.stride(0) == 3 * H * W
    got = native.conv1_marks(maps, s, gl, w, bias).permute(0, 2, 3, 1).reshape(-1, 32).cpu().numpy()
    bad = _replay_mismatch(got, want, idx, "channel")
    assert bad is None, f"{B}x{H}x{W}, strided start / goal: {bad}"


def test_conv1_marks_bit_equal_to_replay_beyond_the_grid(native, sms):
    """More pixels than the capped grid covers (8 CTAs per SM of 8 warps of 32 pixels): 4 096 sampled pixels, plus the
    first and last 40, against the replay."""
    cap = sms * 8 * 8 * 32
    H, W = 37, 53
    B = cap // (H * W) + 2
    P = B * H * W
    assert P > cap
    maps, start, goal, w, bias = _conv1_problem(B, H, W, seed=5)
    got = native.conv1_marks(maps, start, goal, w, bias).permute(0, 2, 3, 1).reshape(P, 32)
    idx = _sample(P, 4096, np.random.RandomState(5))
    want = eo.conv1_marks_replay(maps.cpu().numpy(), start.cpu().numpy(), goal.cpu().numpy(), w, bias, pix=idx)
    bad = _replay_mismatch(got[torch.from_numpy(idx).cuda()].cpu().numpy(), want, idx, "channel")
    assert bad is None, bad
