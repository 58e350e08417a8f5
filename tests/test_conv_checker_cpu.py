"""The conv-engine checker (conv_check.py) rejects the small edge errors it exists to catch, and accepts noise.

A kernel that drops one tap at a row end, loses one row's bias in a partial row tile or shifts its last column moves the
whole-tensor relative RMS by less than the layer tolerance.  These tests build exactly such results from a float64
reference on CPU tensors, at sweep shapes of test_conv_engine_edges_gpu.py, and assert that the checker rejects each one;
so a later loosening of its bounds shows up here.
"""
import pytest
import torch
import torch.nn.functional as F

import conv_check as CC
from test_bench_scale_gpu import LAYER_REL_TOL

# (cin, cout, k, dil, pad, b, t): a partial row tile (150, 80, 192 rows), a Cin tail (13, 150), K = 1 with 513 inputs,
# "valid" and over-padded convs, one output row (conv_post)
SHAPES = [
    (150, 150, 3, 1, 1, 2, 129),
    (13, 80, 5, 3, 0, 2, 131),
    (513, 192, 1, 1, 0, 1, 124),
    (64, 300, 11, 6, 33, 1, 257),
    (32, 1, 7, 1, 3, 2, 255),
    (200, 192, 3, 1, 2, 2, 64),
]
PARTIAL_ROW_TILE = [s for s in SHAPES if s[1] > 1 and s[1] % 128]
SLOPE = 0.1


def _id(s):
    return f"cin{s[0]}_cout{s[1]}_k{s[2]}_d{s[3]}_p{s[4]}"


def _layer(cin, cout, k, dil, pad, b, t, seed=0):
    g = torch.Generator().manual_seed(seed + cin * 7 + cout)
    x = torch.randn(b, cin, t, generator=g)
    w = torch.randn(cout, cin, k, generator=g) / (cin * k) ** 0.5
    bias = torch.randn(cout, generator=g) * 0.1
    want = CC.conv(x, w, bias, dilation=dil, padding=pad, in_slope=SLOPE)
    return x, w, bias, want


def _drop_product(x, w, want, dil, pad, col):
    """want with one tap x channel product removed from output column `col` (batch 0, middle row): the product of
    median magnitude among the ones inside the input, as a kernel that skips one channel or tap there would."""
    xs = F.leaky_relu(x.double(), SLOPE)
    r = w.shape[0] // 2
    t_in = col + dil * torch.arange(w.shape[2]) - pad
    ok = (t_in >= 0) & (t_in < x.shape[2])
    prods = w[r].double()[:, ok] * xs[0][:, t_in[ok]]          # [Cin, taps inside]
    flat = prods.flatten()
    nz = flat[flat != 0]
    med = nz.abs().median()
    i = int((flat.abs() - med).abs().argmin())
    got = want.clone()
    got[0, r, col] -= flat[i]
    return got


def _rejected(got, want):
    fails, _ = CC.failures(got, want, LAYER_REL_TOL)
    return fails


@pytest.mark.parametrize("shape", SHAPES, ids=_id)
def test_checker_accepts_1e6_noise(shape):
    cin, cout, k, dil, pad, b, t = shape
    _, _, _, want = _layer(*shape)
    g = torch.Generator().manual_seed(1)
    got = want * (1 + 1e-6 * torch.randn(want.shape, generator=g, dtype=torch.float64))
    fails, m = CC.failures(got, want, LAYER_REL_TOL)
    assert not fails, (fails, m)


@pytest.mark.parametrize("where", ["first", "last"])
@pytest.mark.parametrize("shape", SHAPES, ids=_id)
def test_checker_rejects_one_dropped_product(shape, where):
    cin, cout, k, dil, pad, b, t = shape
    x, w, _, want = _layer(*shape)
    col = 0 if where == "first" else want.shape[2] - 1
    assert _rejected(_drop_product(x, w, want, dil, pad, col), want)


@pytest.mark.parametrize("shape", PARTIAL_ROW_TILE, ids=_id)
def test_checker_rejects_one_row_without_bias_in_a_partial_row_tile(shape):
    x, w, bias, want = _layer(*shape)
    r = want.shape[1] - 1                       # last row of the last (partial) 128-row tile
    got = want.clone()
    got[0, r, :] -= bias[r].double()
    fails = _rejected(got, want)
    assert any("per-row" in f for f in fails), fails


@pytest.mark.parametrize("shape", SHAPES, ids=_id)
def test_checker_rejects_a_shifted_last_column(shape):
    _, _, _, want = _layer(*shape)
    got = want.clone()
    got[..., -1] = want[..., -2]
    assert _rejected(got, want)


@pytest.mark.parametrize("shape", SHAPES, ids=_id)
def test_checker_rejects_1e3_perturbation_of_one_column(shape):
    _, _, _, want = _layer(*shape)
    got = want.clone()
    c = want.shape[2] // 2
    got[-1, :, c] *= 1 + 1e-3
    fails = _rejected(got, want)
    assert any("per-column" in f for f in fails), fails


@pytest.mark.parametrize("shape", SHAPES, ids=_id)
def test_fp32_calibrated_check(shape):
    """The FMA-kernel criterion: another fp32 summation order (unfold + matmul) passes; the edge errors above, made on
    top of torch's fp32 conv, do not."""
    cin, cout, k, dil, pad, b, t = shape
    x, w, bias, want = _layer(*shape)
    cpu32 = CC.conv(x, w, bias, dilation=dil, padding=pad, in_slope=SLOPE, dtype=torch.float32)
    cols = F.unfold(F.leaky_relu(x, SLOPE)[:, :, None, :], (1, k), dilation=(1, dil), padding=(0, pad))
    alt = (w.reshape(cout, -1).flip(1) @ cols.flip(1)) + bias[None, :, None]    # [B, Cout, Tout], reversed order
    assert not CC.fp32_calibrated_failures(alt, want, cpu32)
    col = want.shape[2] - 1
    bad = [_drop_product(x, w, cpu32.double(), dil, pad, 0), _drop_product(x, w, cpu32.double(), dil, pad, col)]
    shifted = cpu32.clone()
    shifted[..., -1] = cpu32[..., -2]
    bumped = cpu32.clone()
    bumped[-1, :, col // 2] *= 1 + 1e-3
    for got in bad + [shifted, bumped]:
        assert CC.fp32_calibrated_failures(got, want, cpu32)
