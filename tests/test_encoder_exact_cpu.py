"""The CPU helpers of tests/encoder_exact_oracle.py against exact rational arithmetic (fractions.Fraction), without a
GPU: fma32 and tf32 rounding, the fused-kernel operand generator's budget, and the two kernel replays."""
from fractions import Fraction

import numpy as np
import pytest
import torch

import encoder_exact_oracle as eo


def _round(q, p, mode="rne", emin=-126):
    """Fraction q rounded to p significant bits (exponent at least emin: the subnormal grid below 2^emin)."""
    if q == 0:
        return Fraction(0)
    a = abs(q)
    e = a.numerator.bit_length() - a.denominator.bit_length()
    if Fraction(2) ** e > a:
        e -= 1
    ulp = Fraction(2) ** (max(e, emin) - p + 1)
    n = a / ulp
    m = n.numerator // n.denominator
    rem = n - m
    if mode == "rne" and (rem > Fraction(1, 2) or (rem == Fraction(1, 2) and m % 2)):
        m += 1
    return (m * ulp) * (1 if q > 0 else -1)


def _f32(v):
    return np.float32(v)


def _fma_cases(rng):
    """(a, b, c) fp32 triples: random exponents, exact fp32 midpoints missed by a tiny product tail (fp64 rounds the
    tail away), subnormal results, cancellation and mixed signs."""
    n = 4000
    a = (rng.randn(n) * 2.0 ** rng.randint(-30, 30, n)).astype(np.float32)
    b = (rng.randn(n) * 2.0 ** rng.randint(-30, 30, n)).astype(np.float32)
    c = (rng.randn(n) * 2.0 ** rng.randint(-60, 60, n)).astype(np.float32)
    cases = [(a, b, c)]
    # c + half an ulp of c, missed by -+ 2^-40 relatively: (h (1 + 2^-20)) (1 - 2^-20) = h (1 - 2^-40)
    cm = (rng.rand(n) + 1).astype(np.float32) * np.float32(2.0) ** rng.randint(-100, 100, n).astype(np.float32)
    cm *= np.where(rng.rand(n) < 0.5, 1, -1).astype(np.float32)
    half = (np.spacing(np.abs(cm)) / 2).astype(np.float32)
    sgn = np.where(rng.rand(n) < 0.5, 1, -1).astype(np.float32)
    am = (half * np.float32(1 + 2.0 ** -20) * sgn).astype(np.float32)
    bm = np.where(rng.rand(n) < 0.5, 1 - 2.0 ** -20, 1 + 2.0 ** -20).astype(np.float32)
    cases.append((am, bm, cm))
    # the same at the bottom of the subnormal range: products of 2^-150 (1 -+ 2^-40) onto multiples of 2^-149
    k = rng.randint(0, 1 << 22, n).astype(np.float64)
    cs = (k * 2.0 ** -149).astype(np.float32) * sgn
    as_ = np.float32(2.0 ** -75 * (1 + 2.0 ** -20)) * np.where(rng.rand(n) < 0.5, 1, -1).astype(np.float32)
    bs = np.where(rng.rand(n) < 0.5, 2.0 ** -75 * (1 - 2.0 ** -20), 2.0 ** -75).astype(np.float32)
    cases.append((as_.astype(np.float32), bs, cs))
    # subnormal results from small products and small addends
    a2 = (rng.randn(n) * 2.0 ** rng.randint(-80, -60, n)).astype(np.float32)
    b2 = (rng.randn(n) * 2.0 ** rng.randint(-80, -60, n)).astype(np.float32)
    c2 = (rng.randn(n) * 2.0 ** rng.randint(-150, -126, n)).astype(np.float32)
    cases.append((a2, b2, c2))
    # cancellation: c = -fl(a b), the result is the product's rounding error
    cases.append((a, b, -(a * b).astype(np.float32)))
    return cases


def test_fma32_matches_exact_rounding():
    rng = np.random.RandomState(0)
    naive_differs = 0
    for a, b, c in _fma_cases(rng):
        got = eo.fma32(a, b, c)
        naive = (a.astype(np.float64) * b.astype(np.float64) + c.astype(np.float64)).astype(np.float32)
        for i in range(a.size):
            want = _round(Fraction(float(a[i])) * Fraction(float(b[i])) + Fraction(float(c[i])), 24)
            assert Fraction(float(got[i])) == want, (a[i], b[i], c[i], got[i], float(want))
        naive_differs += int((naive != got).sum())
    assert naive_differs > 0     # the midpoint cases are really decided by the TwoSum tail, not by fp64 rounding


def test_fma32_signs_of_zero_and_exact_cases():
    z = np.float32(0)
    assert np.signbit(eo.fma32(np.float32(-0.0), np.float32(1), np.float32(-0.0)))     # -0 + -0 = -0
    assert not np.signbit(eo.fma32(np.float32(1), np.float32(-0.0), z))                # -0 + +0 = +0
    assert not np.signbit(eo.fma32(np.float32(3), np.float32(2), np.float32(-6)))      # exact cancellation: +0
    assert eo.fma32(np.float32(1 + 2.0 ** -12), np.float32(1 - 2.0 ** -12), np.float32(-1)) == np.float32(-2.0 ** -24)
    # 2^24 + 2 + (1 - 2^-40): just below the midpoint 2^24 + 3, so 2^24 + 2; fp64 would see the tie and round to even
    a, b, c = np.float32(1 + 2.0 ** -20), np.float32(1 - 2.0 ** -20), np.float32(2.0 ** 24 + 2)
    assert eo.fma32(a, b, c) == np.float32(2.0 ** 24 + 2)
    assert np.float32(np.float64(a) * np.float64(b) + np.float64(c)) == np.float32(2.0 ** 24 + 4)
    # broadcasting
    assert eo.fma32(np.ones((3, 1), np.float32), np.ones((1, 4), np.float32), np.zeros((3, 4), np.float32)).shape == (3, 4)


@pytest.mark.parametrize("mode", ["trunc", "rne"])
def test_tf32_matches_exact_rounding(mode):
    rng = np.random.RandomState(1)
    bits = rng.randint(0, 2 ** 32, 20000, dtype=np.uint64).astype(np.uint32)
    bits = bits[((bits >> 23) & 0xFF) != 0xFF]                                    # finite
    bits = np.concatenate([bits, rng.randint(0, 1 << 23, 2000).astype(np.uint32),   # subnormals
                           np.array([0x00000000, 0x80000000, 0x3F801000, 0x3F803000, 0x3F800FFF, 0x3F801001,
                                     0x00001000, 0x00003000, 0x807FF000, 0x7F7FFFFF, 0x3FFFF000], np.uint32)])
    x = bits.view(np.float32)
    got = eo.tf32(x, mode)
    for v, g in zip(x, got):
        want = _round(Fraction(float(v)), 11, mode)
        if want >= Fraction(2) ** 128:
            assert np.isinf(g)                     # rounding the largest fp32 values up overflows, as IEEE does
        else:
            assert Fraction(float(g)) == want, (v, g, float(want))
        assert np.signbit(g) == np.signbit(v)
    # ties go to even: 1 + 2^-11 to 1, 1 + 3 * 2^-11 to 1 + 2^-9; and the two modes differ somewhere
    assert eo.tf32(np.float32(1 + 2.0 ** -11), "rne") == np.float32(1)
    assert eo.tf32(np.float32(1 + 3 * 2.0 ** -11), "rne") == np.float32(1 + 2.0 ** -9)
    assert (eo.tf32(x, "trunc") != eo.tf32(x, "rne")).any()
    assert np.array_equal(eo.tf32_torch(torch.from_numpy(x), mode).numpy().view(np.uint32), got.view(np.uint32))


# -------------------------------------------------------------------------------------------- operand generator
def test_exact_operands_are_exact_in_fp32_in_another_order():
    """The generator accepts its own draws, and an fp32 evaluation in PyTorch's CPU order gives the fp64 taps."""
    x, w, b, hw, taps, pre = eo.exact_operands(2, 5, 7, seed=3, device="cpu")
    assert x.min() < 0 < x.max() and (x == 0).any()
    a32 = torch.relu(torch.nn.functional.conv2d(x, w, b, padding=1))
    assert torch.equal(a32.double(), torch.relu(pre))
    t32 = torch.einsum("bchw,ck->bhwk", a32, torch.from_numpy(hw))
    assert torch.equal(t32.double(), taps)
    assert (taps != 0).float().mean() > 0.9


def _budget_problem(conv_units, head_second_channel):
    """1x1 map; u = 2^-13.  Channel 0 sums 128 products of 31 x 1023 units plus a bias that brings the conv budget to
    conv_units; with head_second_channel the head reads channel 0 (pre = 2^22 - 1 - the bias) and a channel 1 of pre 1."""
    ux, uw = 2.0 ** -5, 2.0 ** -8
    x = torch.zeros(1, 128, 1, 1)
    w = torch.zeros(256, 128, 3, 3)
    b = torch.zeros(256)
    hw = np.zeros((256, 9), np.float32)
    if not head_second_channel:
        x[0, :, 0, 0] = 31 * ux
        w[0, :, 1, 1] = 1023 * uw
        b[0] = -(conv_units - 128 * 31 * 1023) * ux * uw
    else:
        x[0, 0, 0, 0] = ux
        w[0, 0, 1, 1] = uw
        w[1, 0, 1, 1] = uw
        b[0] = (2 ** 22 - 2) * ux * uw                # channel 0: pre = 2^22 - 1 units, conv budget 2^22 - 1
        hw[0, 0] = hw[1, 0] = 1.0
    return x, w, b, hw, ux, uw


def test_exact_budget_refuses_one_unit_over():
    eo.exact_budget(*_budget_problem(2 ** 22 - 1, False))
    with pytest.raises(ValueError, match="conv budget"):
        eo.exact_budget(*_budget_problem(2 ** 22, False))
    x, w, b, hw, ux, uw = _budget_problem(None, True)
    hw1 = hw.copy()
    hw1[1, 0] = 0.0
    eo.exact_budget(x, w, b, hw1, ux, uw)             # head sum 2^22 - 1 units
    with pytest.raises(ValueError, match="head budget"):
        eo.exact_budget(x, w, b, hw, ux, uw)          # plus channel 1: 2^22
    with pytest.raises(ValueError, match="not exact in TF32"):
        eo.exact_budget(x.mul(2047), w * 2049, b, hw1, ux, uw)
    with pytest.raises(ValueError, match="multiple"):
        eo.exact_budget(x * 0.5, w, b, hw1, ux, uw)


# --------------------------------------------------------------------------------------------------- replays
def _wide_randn(rng, *shape):
    return (rng.randn(*shape) * 2.0 ** rng.randint(-12, 12, shape)).astype(np.float32)


def test_head_taps_replay_matches_fraction_evaluation():
    rng = np.random.RandomState(4)
    P, C = 6, 16
    x, w = _wide_randn(rng, P, C), _wide_randn(rng, C, 9)
    got = eo.head_taps_replay(x, w)
    for p in range(P):
        for k in range(9):
            acc = Fraction(0)
            for c in range(C):
                acc = _round(Fraction(float(x[p, c])) * Fraction(float(w[c, k])) + acc, 24)
            assert Fraction(float(got[p, k])) == acc, (p, k)


def test_conv1_marks_replay_matches_fraction_evaluation():
    rng = np.random.RandomState(5)
    B, H, W = 2, 3, 4
    maps, start, goal = (_wide_randn(rng, B, 1, H, W) for _ in range(3))
    w, b = _wide_randn(rng, 9, 2, 32), _wide_randn(rng, 32)
    got = eo.conv1_marks_replay(maps, start, goal, w, b)
    assert got.shape == (B, H, W, 32)
    pix = np.array([0, 5, B * H * W - 1])
    assert np.array_equal(eo.conv1_marks_replay(maps, start, goal, w, b, pix=pix), got.reshape(-1, 32)[pix])
    F = lambda v: Fraction(float(v))   # noqa: E731
    for bi in range(B):
        for y in range(H):
            for x in range(W):
                for c in range(32):
                    acc = F(b[c])
                    for ky in range(3):
                        for kx in range(3):
                            yy, xx = y + ky - 1, x + kx - 1
                            m = k = Fraction(0)
                            if 0 <= yy < H and 0 <= xx < W:
                                m = F(maps[bi, 0, yy, xx])
                                k = _round(F(start[bi, 0, yy, xx]) + F(goal[bi, 0, yy, xx]), 24)
                            acc = _round(m * F(w[ky * 3 + kx, 0, c]) + acc, 24)
                            acc = _round(k * F(w[ky * 3 + kx, 1, c]) + acc, 24)
                    assert F(got[bi, y, x, c]) == max(acc, Fraction(0)), (bi, y, x, c)
