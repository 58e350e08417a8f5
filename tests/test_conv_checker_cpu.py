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


# ----------------------------------------------------------------------------- the engine-option reference
# engine_epilogue / engine_layer (conv_check.py) restate launch_conv's documented order; test_conv_engine_epilogues_gpu.py
# holds the kernels to them.  Here they are pinned to plain restatements of the model code they stand for, and the
# checker is shown to reject each option applied wrongly.
H_WN, T_WN = 96, 131


def _wn_inputs(seed=3):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(2, H_WN, T_WN, generator=g, dtype=torch.float64)
    w_in = torch.randn(2 * H_WN, H_WN, 5, generator=g, dtype=torch.float64) / (5 * H_WN) ** 0.5
    b_in = torch.randn(2 * H_WN, generator=g, dtype=torch.float64) * 0.1
    w_rs = torch.randn(2 * H_WN, H_WN, 1, generator=g, dtype=torch.float64) / H_WN ** 0.5
    b_rs = torch.randn(2 * H_WN, generator=g, dtype=torch.float64) * 0.1
    cond = torch.randn(2, 2 * H_WN, generator=g, dtype=torch.float64)
    out_old = torch.randn(2, H_WN, T_WN, generator=g, dtype=torch.float64)
    mask = torch.ones(2, T_WN, dtype=torch.float64)
    mask[0, 100:] = 0
    mask[1, 7:11] = 0            # zeros inside the row too
    return x, w_in, b_in, w_rs, b_rs, cond, out_old, mask


def _wn_layer_plain(x, w_in, b_in, w_rs, b_rs, cond, out_old, mask, dil):
    """one WaveNet layer as wavenet.py writes it (:6-13, :98-113), not the last one"""
    x_in = F.conv1d(x, w_in, b_in, dilation=dil, padding=2 * dil)
    in_act = x_in + cond[:, :, None]
    acts = torch.tanh(in_act[:, :H_WN]) * torch.sigmoid(in_act[:, H_WN:])
    rs = F.conv1d(acts, w_rs, b_rs)
    return acts, (x + rs[:, :H_WN]) * mask[:, None], out_old + rs[:, H_WN:]


def _wn_layer_engine(x, w_in, b_in, w_rs, b_rs, cond, out_old, mask, dil, **mutate):
    acts, _ = CC.engine_layer(x, w_in, b_in, dilation=dil, padding=2 * dil, cond=mutate.get("cond_override", cond),
                              flags=CC.EPI_GATE)
    if mutate.get("swap_gate"):
        c = F.conv1d(x, w_in, b_in, dilation=dil, padding=2 * dil) + cond[:, :, None]
        acts = torch.sigmoid(c[:, :H_WN]) * torch.tanh(c[:, H_WN:])
    h, out = CC.engine_layer(acts, w_rs, b_rs, ymask=mask, flags=CC.EPI_SPLIT | CC.EPI_ACCUM2, split=H_WN,
                             y_old=x, y2_old=out_old)
    if mutate.get("mask_y2"):
        out = out * mask[:, None]
    return acts, h, out


@pytest.mark.parametrize("dil", [1, 2])
def test_engine_reference_is_one_wavenet_layer(dil):
    args = _wn_inputs()
    want = _wn_layer_plain(*args, dil)
    got = _wn_layer_engine(*args, dil)
    for g, w in zip(got, want):
        torch.testing.assert_close(g, w, rtol=1e-12, atol=1e-12)


def test_engine_reference_is_the_last_wavenet_layer_and_the_coupling_post():
    x, w_in, b_in, w_rs, b_rs, cond, out_old, mask = _wn_inputs()
    w_last, b_last = w_rs[:H_WN], b_rs[:H_WN]
    # last layer: output = (output + res_skip(acts)) * x_mask
    y, _ = CC.engine_layer(x, w_last, b_last, ymask=mask, flags=CC.EPI_MASK_POST | CC.EPI_ACCUM, y_old=out_old)
    torch.testing.assert_close(y, (out_old + F.conv1d(x, w_last, b_last)) * mask[:, None], rtol=1e-12, atol=1e-12)
    # coupling post (networks.py:151-164, mean_only): m = post(h) * mask; reverse x1 = (x1 - m) * mask, forward
    # x1 = m + x1 * mask
    x1 = out_old[:, : H_WN // 2]
    w_post, b_post = w_rs[: H_WN // 2], b_rs[: H_WN // 2]
    m = F.conv1d(x, w_post, b_post) * mask[:, None]
    for scale, want in ((-1.0, (x1 - m) * mask[:, None]), (1.0, m + x1 * mask[:, None])):
        y, _ = CC.engine_layer(x, w_post, b_post, ymask=mask, scale=scale, y_old=x1,
                               flags=CC.EPI_MASK_PRE | CC.EPI_ACCUM | CC.EPI_MASK_POST)
        torch.testing.assert_close(y, want, rtol=1e-12, atol=1e-12)


def test_checker_rejects_swapped_gate_halves():
    args = _wn_inputs()
    want, got = _wn_layer_engine(*args, 1), _wn_layer_engine(*args, 1, swap_gate=True)
    assert _rejected(got[0], want[0])


def test_checker_rejects_a_dropped_cond_on_one_row():
    args = _wn_inputs()
    cond = args[5].clone()
    r = H_WN + 17                                  # one row of the sigmoid half
    cond[1, r] = 0
    want, got = _wn_layer_engine(*args, 1), _wn_layer_engine(*args, 1, cond_override=cond)
    fails = _rejected(got[0], want[0])
    assert any("per-row" in f for f in fails), fails


def test_checker_rejects_the_mask_on_y2_rows():
    args = _wn_inputs()
    want, got = _wn_layer_engine(*args, 1), _wn_layer_engine(*args, 1, mask_y2=True)
    assert torch.equal(got[1], want[1])
    assert _rejected(got[2], want[2])


def test_checker_rejects_mask_pre_after_the_residual():
    x, _, _, w_rs, b_rs, _, out_old, mask = _wn_inputs()
    w, b = w_rs[: H_WN // 2], b_rs[: H_WN // 2]
    res = out_old[:, H_WN // 2:]
    want, _ = CC.engine_layer(x, w, b, ymask=mask, residual=res, flags=CC.EPI_MASK_PRE)
    got = (F.conv1d(x, w, b) + res) * mask[:, None]
    assert _rejected(got, want)


def test_checker_rejects_a_ragged_row_one_column_short():
    x, w_in, b_in, _, _, _, _, _ = _wn_inputs()
    lens, rate, need = torch.tensor([T_WN, 57]), 2, 3
    want, _ = CC.engine_layer(x, w_in[:H_WN], b_in[:H_WN], padding=2)
    ext = CC.ragged_extent(lens, rate, need, T_WN)
    valid = CC.columns_below(ext, T_WN)
    got = want.clone()
    got[1, :, int(ext[1]) - 1] = 0                 # the row's last column not computed (a zeroed buffer)
    assert int(ext[1]) == 117
    assert not CC.failures(torch.where(valid[:, None], want, want), want, LAYER_REL_TOL)[0]
    assert _rejected(torch.where(valid[:, None], got, want), want)
