"""CPU helpers for checking the encoder's hand-written kernels bit for bit (tests/test_gpu_encoder_exact.py):

  tf32, fma32           fp32 -> TF32 conversion (truncation or round to nearest even; tf32_torch on a device) and an
                        exact, vectorised fp32 FMA;
  head_taps_replay      head_taps_kernel<C>'s operation sequence (nastar_glue.cuh): ascending channel, one fmaf per
                        product;
  conv1_marks_replay    conv1_marks_kernel's: bias, then the 9 taps in (ky, kx) order, fmaf(k, w1, fmaf(m, w0, acc)),
                        fmaxf with 0;
  exact_operands        operands for conv3x3_head_kernel whose fp64 result is the only correct fp32 output;
  tf32_taps_and_bound   fp64 taps of TF32-converted operands and a bound that covers only fp32 accumulation and the head.

Conventions follow the kernels: the fused kernel's x is [B,128,H,W] (channels-last in memory), its weights
[256,128,3,3], bias [256] and head weights [256,9]; taps come out as [B,H,W,9].
"""
import numpy as np
import torch

# Mode in which the tensor cores read fp32 operands of a TF32 wgmma: observed on an H100 SXM by
# test_gpu_encoder_exact.py::test_tf32_operand_conversion_mode (every probe of both operands agrees).
TF32_MODE = "trunc"
# a sum is exact in fp32 in any order and with any rounding when every term is a multiple of u and the sum of the
# terms' magnitudes stays below BUDGET * u (fp32 keeps 24 bits; 2 spare bits cover the tensor cores' alignment)
BUDGET = 2 ** 22
K_CONV = 9 * 128          # products per pre-activation of the fused kernel
HEAD_ROUNDINGS = 66       # fp32 roundings of one fused-kernel tap: 64 channel FMAs per lane, then 2 cross-lane adds


# ---------------------------------------------------------------------------------------------- fp32 primitives
def tf32(a, mode):
    """fp32 array -> TF32 values (10 explicit mantissa bits) as fp32.  "trunc" clears the low 13 bits, "rne" rounds
    to nearest, ties to even (a carry may reach the exponent, as IEEE rounding does)."""
    bits = np.ascontiguousarray(a, dtype=np.float32).view(np.uint32)
    if mode == "rne":
        bits = bits + np.uint32(0x0FFF) + ((bits >> np.uint32(13)) & np.uint32(1))
    elif mode != "trunc":
        raise ValueError(f"unknown TF32 mode {mode!r}")
    return (bits & np.uint32(0xFFFFE000)).view(np.float32)


def tf32_torch(t, mode):
    """tf32 on an fp32 torch tensor, on its device (int32 arithmetic wraps like the uint32 one of tf32)."""
    bits = t.contiguous().view(torch.int32)
    if mode == "rne":
        bits = bits + 0x0FFF + ((bits >> 13) & 1)
    elif mode != "trunc":
        raise ValueError(f"unknown TF32 mode {mode!r}")
    return (bits & -0x2000).view(torch.float32).view(t.shape)


def fma32(a, b, c):
    """fp32 fmaf(a, b, c) for finite operands, element-wise: a*b is exact in fp64, TwoSum gives s + e = a*b + c
    exactly, s is rounded to fp32 and, where s lies exactly halfway between two fp32 neighbours, the sign of e picks
    the neighbour (the fp64 sum hid which side of the midpoint the exact value lies on).  Subnormal results included."""
    a, b, c = (np.asarray(v, dtype=np.float32) for v in (a, b, c))
    p = a.astype(np.float64) * b.astype(np.float64)
    c64 = c.astype(np.float64)
    s = p + c64
    bb = s - p
    e = (p - (s - bb)) + (c64 - bb)
    r = s.astype(np.float32)
    r64 = r.astype(np.float64)
    d = s - r64
    other = np.nextafter(r, np.where(d > 0, np.float32(np.inf), np.float32(-np.inf)).astype(np.float32))
    mid = (d != 0) & (r64 + other.astype(np.float64) == 2 * s)
    away = mid & (e != 0) & ((e > 0) == (d > 0))       # the exact value lies past the midpoint, on other's side
    return np.where(away, other, r)


# --------------------------------------------------------------------------------------------------- replays
def head_taps_replay(x, w):
    """head_taps_kernel<C>: out[p][k] = sum_c x[p][c] * w[c][k], accumulated from 0 in ascending c with one fmaf per
    product.  x: fp32 [P, C] (pixels, channels-last); w: fp32 [C, 9].  Returns fp32 [P, 9]."""
    x = np.asarray(x, dtype=np.float32)
    w = np.asarray(w, dtype=np.float32)
    acc = np.zeros((x.shape[0], 9), np.float32)
    for c in range(x.shape[1]):
        acc = fma32(x[:, c:c + 1], w[c][None, :], acc)
    return acc


def conv1_marks_replay(maps, start, goal, w, b, pix=None):
    """conv1_marks_kernel: acc = b; for ky, kx: m = map, k = start + goal (one fp32 add), acc = fmaf(k, w[t][1],
    fmaf(m, w[t][0], acc)), with m = k = 0 outside the map; then fmaxf(acc, 0).  maps/start/goal: fp32 [B,H,W] (or
    [B,1,H,W]); w: fp32 [9,2,32] = [tap][cin][cout]; b: fp32 [32].  pix: flat pixel indices b*H*W + y*W + x to evaluate
    (default: all).  Returns fp32 [n, 32] for pix, else [B,H,W,32]."""
    maps, start, goal = (np.asarray(v, dtype=np.float32) for v in (maps, start, goal))
    if maps.ndim == 4:
        maps, start, goal = maps[:, 0], start[:, 0], goal[:, 0]
    B, H, W = maps.shape
    w = np.asarray(w, dtype=np.float32)
    b = np.asarray(b, dtype=np.float32)
    idx = np.arange(B * H * W) if pix is None else np.asarray(pix, dtype=np.int64)
    bi, rc = idx // (H * W), idx % (H * W)
    y, x = rc // W, rc % W
    acc = np.broadcast_to(b, (idx.size, 32)).copy()
    for ky in range(3):
        for kx in range(3):
            yy, xx = y + ky - 1, x + kx - 1
            inside = (yy >= 0) & (yy < H) & (xx >= 0) & (xx < W)
            yc, xc = np.clip(yy, 0, H - 1), np.clip(xx, 0, W - 1)
            m = np.where(inside, maps[bi, yc, xc], np.float32(0))[:, None]
            k = np.where(inside, start[bi, yc, xc] + goal[bi, yc, xc], np.float32(0))[:, None]
            t = ky * 3 + kx
            acc = fma32(k, w[t, 1][None, :], fma32(m, w[t, 0][None, :], acc))
    out = np.maximum(acc, np.float32(0))
    return out if pix is not None else out.reshape(B, H, W, 32)


# ------------------------------------------------------------------------------------ fused conv + head operands
def _conv64(x, w, b=None):
    return torch.nn.functional.conv2d(x.double(), w.double(), None if b is None else b.double(), padding=1)


def exact_budget(x, w, b, hw, ux, uw):
    """Refuse (ValueError) operands for which an fp32 evaluation of the fused kernel in some order could round:
    x must be a multiple of ux and w of uw, both exact in TF32, the bias a multiple of u = ux * uw and the head weights
    integers; then every conv product and every head product a[c] * hw[c][k] is a multiple of u, and both sums of
    magnitudes (sum|x||w| + |b| per pre-activation, sum_c relu(pre[c]) |hw[c][k]| per tap) must stay below BUDGET * u.
    Returns the exact fp64 taps [B,H,W,9] and pre-activations [B,256,H,W]."""
    u = ux * uw
    hwt = torch.as_tensor(np.asarray(hw), device=x.device).double()
    for name, v, q in (("x", x.double(), ux), ("w", w.double(), uw), ("bias", b.double(), u), ("head", hwt, 1.0)):
        if not bool(torch.equal(torch.round(v / q), v / q)):
            raise ValueError(f"{name} is not a multiple of {q}")
        f = v.float().cpu().numpy()
        if name in ("x", "w") and not (np.array_equal(tf32(f, "trunc"), f) and np.array_equal(tf32(f, "rne"), f)):
            raise ValueError(f"{name} is not exact in TF32")       # the tensor cores' operands; bias and head are fp32
    s_conv = _conv64(x.abs(), w.abs()) + b.double().abs().view(1, -1, 1, 1)
    if float(s_conv.max()) >= BUDGET * u:
        raise ValueError(f"conv budget: max sum|x||w| + |b| = {float(s_conv.max()) / u:.0f} u >= 2^22 u")
    pre = _conv64(x, w, b)
    a = torch.relu(pre)
    s_head = torch.einsum("bchw,ck->bhwk", a, hwt.abs())
    if float(s_head.max()) >= BUDGET * u:
        raise ValueError(f"head budget: max sum relu(pre)|hw| = {float(s_head.max()) / u:.0f} u >= 2^22 u")
    return torch.einsum("bchw,ck->bhwk", a, hwt), pre


def exact_operands(B, H, W, seed, device="cuda"):
    """Dyadic operands for conv3x3_head_taps whose every product and partial sum is exact in fp32 in any order
    (exact_budget), so the fp64 taps are the only correct output, bit for bit, whatever the tensor cores' accumulation
    order or rounding.  x in (1/32) {-31..31} (40 % zeros, both signs: the kernel does not assume ReLU inputs), w in
    (1/256) {-31..31}, u = 2^-13, bias in u {-4096..4096}, head weights in {-3..3}, all drawn independently, so a
    channel, tap or k step read in place of another changes the result.  Returns (x channels-last, w channels-last, b, hw numpy
    [256,9], exact taps fp64 [B,H,W,9], pre-activations fp64 [B,256,H,W])."""
    g = torch.Generator(device="cpu").manual_seed(seed)
    ux, uw = 2.0 ** -5, 2.0 ** -8
    ix = torch.randint(-31, 32, (B, 128, H, W), generator=g) * (torch.rand(B, 128, H, W, generator=g) > 0.4)
    iw = torch.randint(-31, 32, (256, 128, 3, 3), generator=g)
    ib = torch.randint(-4096, 4097, (256,), generator=g)
    hw = torch.randint(-3, 4, (256, 9), generator=g).numpy().astype(np.float32)
    x = (ix.float() * ux).to(device).contiguous(memory_format=torch.channels_last)
    w = (iw.float() * uw).to(device).contiguous(memory_format=torch.channels_last)
    b = (ib.float() * (ux * uw)).to(device)
    taps, pre = exact_budget(x, w, b, hw, ux, uw)
    return x, w, b, hw, taps, pre


def tf32_taps_and_bound(x, w, b, hw, mode=TF32_MODE):
    """fp64 taps of the operands the tensor cores read (tf32(x), tf32(w) in `mode`; bias and head weights are fp32
    operands of fp32 FFMA), and a per-tap bound on what the kernel's fp32 arithmetic may add to them.

    Pre-activation.  With S = sum |tf32(x)||tf32(w)| over the K = 1152 products: the tensor cores add the products to
    the fp32 accumulator n >= 4 at a time (a k8 instruction in groups of 4 or 8).  In each group every addend but the
    largest is aligned to the largest one keeping at least 24 significant bits, which loses less than 2^-23 of the
    largest addend, and the sum is then rounded or truncated to fp32 once, losing less than 2^-23 of it.  Every addend
    and every partial sum is at most S (1 + small), so a group costs at most (n + 1) 2^-23 S and all K / n groups at
    most E = (1 + 1/n) K 2^-23 S <= 1.25 K 2^-23 S (times 1.001 for the partial sums' own error).

    Epilogue.  The kernel forms relu(fl(pre~ + b)) with pre~ within E of pre: when pre + b + E <= 0 the channel is 0
    either way, otherwise the activation is off by at most min(E, R) + 2^-24 R with R = relu(pre + b + E).  The head
    sum over 256 channels is 64 FMAs per lane and two cross-lane adds, 66 fp32 roundings: at most gamma_66 (1 + 2^-24)
    sum_c R_c |hw[c][k]|.  So

        |tap_k - want_k| <= sum_c |hw[c][k]| (min(E_c, R_c) + 2^-24 R_c) + gamma_66 (1 + 2^-24) sum_c R_c |hw[c][k]|.

    Returns (want fp64 [B,H,W,9], bound fp64 [B,H,W,9])."""
    xt, wt = tf32_torch(x.float(), mode), tf32_torch(w.float(), mode)
    hwd = torch.as_tensor(np.asarray(hw), device=x.device).double()
    z = _conv64(xt, wt, b)
    E = 1.001 * 1.25 * K_CONV * 2.0 ** -23 * _conv64(xt.abs(), wt.abs())
    R = torch.relu(z + E)
    want = torch.einsum("bchw,ck->bhwk", torch.relu(z), hwd)
    g66 = HEAD_ROUNDINGS * 2.0 ** -24 / (1 - HEAD_ROUNDINGS * 2.0 ** -24)
    act = torch.minimum(E, R) + 2.0 ** -24 * R + g66 * (1 + 2.0 ** -24) * R
    bound = torch.einsum("bchw,ck->bhwk", act, hwd.abs())
    return want, bound + 1e-12
