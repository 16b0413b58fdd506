"""CPU: the e4m3 cross K|V quantizer oracle (oracle/kv_fp8_oracle.py) on hand-worked blocks.  e4m3fn: 1 sign, 4 exponent
(bias 7), 3 mantissa bits; 0x7E = 448 (the largest finite), 0x7F = NaN, 0x01 = 2^-9 (the smallest subnormal)."""
import math

import torch

import kv_fp8_oracle as ko


def _block(vals, dtype=torch.float32):
    x = torch.zeros(64, dtype=torch.float32)
    x[: len(vals)] = torch.tensor(vals, dtype=torch.float32)
    return x.to(dtype)[None]


def _codes(vals, dtype=torch.float32):
    c, s = ko.quantize_e4m3(_block(vals, dtype))
    return c[0].tolist(), float(s[0, 0])


def test_exact_round_trip():
    """amax = 448 -> inv = 1, scale = 1: values that are e4m3 numbers keep their bits and dequantize exactly."""
    vals = [448.0, -448.0, 1.0, -1.5, 0.5, 240.0, 2.0 ** -6, 2.0 ** -9, 3.25]
    c, s = _codes(vals)
    assert s == 1.0
    assert c[:5] == [0x7E, 0xFE, 0x38, 0xBC, 0x30]
    back = ko.dequantize_e4m3(torch.tensor([c], dtype=torch.uint8), torch.tensor([[s]]))[0, : len(vals)]
    assert back.tolist() == vals


def test_row_maximum_maps_to_448():
    """The block's largest magnitude (either sign) becomes +-448 (0x7E / 0xFE) whatever the scale."""
    for amax in (1.0, 3.0, 0.1, 1e-3, 6e4):
        for sign in (1.0, -1.0):
            c, s = _codes([0.25 * amax, sign * amax, -0.5 * amax])
            assert c[1] == (0x7E if sign > 0 else 0xFE), (amax, sign)
            assert s == float(torch.tensor(amax, dtype=torch.float32) / torch.tensor(448.0))


def test_ties_round_to_even():
    """With scale 1: 1.0625 lies halfway between 1.0 (0x38) and 1.125 (0x39) -> 0x38 (even); 1.1875 halfway between 1.125
    and 1.25 (0x3A) -> 0x3A; 17 between 16 (0x58) and 18 (0x59) -> 0x58; 0.5 * 2^-9 (half the smallest subnormal) -> 0."""
    c, _ = _codes([448.0, 1.0625, 1.1875, 17.0, 19.0, 2.0 ** -10, 3 * 2.0 ** -10])
    assert c[1:7] == [0x38, 0x3A, 0x58, 0x5A, 0x00, 0x02]


def test_saturation():
    """x * inv can round above 448 only by float error; the clamp keeps it at 448, never NaN (torch's cast would give NaN
    past 464)."""
    x = _block([448.0, 470.0])
    x[0, 0] = 300.0                      # amax = 470: 470 * (448 / 470) rounds to 448 or a hair above
    c, s = ko.quantize_e4m3(x)
    assert c[0, 1] == 0x7E
    y = (x.float() * (torch.tensor(448.0) / torch.tensor(470.0))).clamp(-1e9, 1e9)
    assert float(y[0, 1]) >= 447.99
    big = (torch.tensor([[500.0]]) * 1.0).clamp(-448, 448).to(torch.float8_e4m3fn).view(torch.uint8)
    assert int(big) == 0x7E


def test_subnormal_codes():
    """Small members of a block land on e4m3 subnormals: k * 2^-9 -> code k for k = 1..7 (scale 1)."""
    vals = [448.0] + [k * 2.0 ** -9 for k in range(1, 8)] + [-(2.0 ** -9)]
    c, _ = _codes(vals)
    assert c[1:8] == list(range(1, 8))
    assert c[8] == 0x81


def test_zero_and_nan_blocks():
    """amax == 0 -> scale 0 and codes 0; a NaN or an inf anywhere in a block -> scale NaN and codes 0; other blocks of the
    same row are unaffected.  fp16 and bf16 inputs."""
    for dtype in (torch.float16, torch.bfloat16):
        x = torch.randn(3, 4 * 64).to(dtype)
        x[0, :64] = 0.0
        x[1, 64 + 5] = float("nan")
        x[2, 128 + 63] = float("inf")
        x[2, 192] = -float("inf")
        c, s = ko.quantize_e4m3(x)
        assert s[0, 0] == 0.0 and bool((c[0, :64] == 0).all())
        assert math.isnan(s[1, 1]) and bool((c[1, 64:128] == 0).all())
        assert math.isnan(s[2, 2]) and math.isnan(s[2, 3]) and bool((c[2, 128:] == 0).all())
        ok = torch.isfinite(s) & (s > 0)
        assert int(ok.sum()) == 12 - 4
        deq = ko.dequantize_e4m3(c, s).view(3, 4, 64)
        ref = x.double().view(3, 4, 64)
        err = (deq - ref).abs()[ok]
        assert float(err.max()) <= float((ref.abs().amax(-1)[ok] / 448.0 * 16).max())    # half an e4m3 step at 448 = 16


def test_dequantized_error_is_half_a_step():
    """|dequant - x| <= half an e4m3 spacing at |x| (relative 2^-4 for normals, 2^-10 * scale for subnormals) + the fp32
    rounding of x * inv."""
    g = torch.Generator().manual_seed(3)
    x = (torch.randn(64, 12 * 64, generator=g) * torch.rand(64, 1, generator=g) * 8).to(torch.bfloat16)
    c, s = ko.quantize_e4m3(x)
    deq = ko.dequantize_e4m3(c, s).view(64, 12, 64)
    ref = x.double().view(64, 12, 64)
    y = ref / s.double()[..., None]                    # in code units
    step = torch.exp2(torch.floor(torch.log2(y.abs().clamp_min(2.0 ** -6))) - 3)
    assert bool(((deq - ref).abs() <= (0.5 * step * (1 + 2.0 ** -20) + 1e-6 * y.abs()) * s.double()[..., None]).all())
