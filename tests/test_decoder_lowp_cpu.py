"""16-bit decoder precision without a GPU: the precision setting is validated, and the 16-bit layer reference rounds
exactly as a hand-written round-to-nearest-even does."""
import numpy as np
import pytest
import torch

import lowp_reference as R


def _decoder():
    from tts_b200.hifigan import HifiganGenerator
    return HifiganGenerator(in_channels=20, out_channels=1, resblock_type="1", resblock_dilation_sizes=[[1, 3]],
                            resblock_kernel_sizes=[3], upsample_kernel_sizes=[4], upsample_initial_channel=32,
                            upsample_factors=[2])


def test_precision_default_and_validation():
    m = _decoder()
    assert m.precision == "fp32"
    for p in ("bf16", "fp16", "fp32"):
        m.precision = p
        assert m.precision == p
    for bad in ("int8", "BF16", "float16", None, 1, torch.bfloat16):
        with pytest.raises(ValueError, match="precision"):
            m.precision = bad
    assert m.precision == "fp32"                     # a rejected value leaves the setting alone


def test_precision_is_not_part_of_the_state_dict():
    m = _decoder()
    keys = set(m.state_dict())
    m.precision = "bf16"
    assert set(m.state_dict()) == keys


def test_fused_conv_precision_validation():
    from tts_b200.conv import FusedConv1d
    w = torch.randn(32, 16, 3)
    assert FusedConv1d(w).precision == "fp32"
    assert FusedConv1d(w, precision="bf16").precision == "bf16"
    with pytest.raises(ValueError, match="precision"):
        FusedConv1d(w, precision="tf32")
    with pytest.raises(ValueError, match="tensor_cores"):
        FusedConv1d(w, precision="fp16", tensor_cores=False)


def _round_bf16(a):
    """bf16 round to nearest even by hand on the fp32 bit pattern (finite inputs)."""
    u = np.asarray(a, dtype=np.float32).view(np.uint32).astype(np.uint64)
    r = ((u + 0x7FFF + ((u >> 16) & 1)) >> 16) << 16
    return r.astype(np.uint32).view(np.float32).astype(np.float64)


def _round_fp16(a):
    return np.asarray(a, dtype=np.float32).astype(np.float16).astype(np.float64)


def _conv_loop(x, w, b, dil, pad):
    bsz, cin, t = x.shape
    cout, _, k = w.shape
    tout = t + 2 * pad - dil * (k - 1)
    y = np.zeros((bsz, cout, tout))
    for n in range(bsz):
        for co in range(cout):
            for q in range(tout):
                s = b[co]
                for ci in range(cin):
                    for kk in range(k):
                        ti = q + kk * dil - pad
                        if 0 <= ti < t:
                            s += w[co, ci, kk] * x[n, ci, ti]
                y[n, co, q] = s
    return y


@pytest.mark.parametrize("precision,rnd", [("bf16", _round_bf16), ("fp16", _round_fp16)])
def test_reference_matches_hand_rounding(precision, rnd):
    # values that land between 16-bit neighbours (ties included) so that every rounding decision matters
    assert float(R.round_to(torch.tensor([1 + 2 ** -8]), "bf16")) == 1.0                  # tie -> even
    assert float(R.round_to(torch.tensor([1 + 3 * 2 ** -8]), "bf16")) == 1 + 2 ** -6      # tie -> even (up)
    assert float(R.round_to(torch.tensor([1 + 3 * 2 ** -9]), "bf16")) == 1 + 2 ** -7
    assert float(R.round_to(torch.tensor([1 + 2 ** -11]), "fp16")) == 1.0
    assert float(R.round_to(torch.tensor([70000.0]), "fp16")) == float("inf")             # fp16 overflow
    gen = torch.Generator().manual_seed(5)
    x = torch.randn(2, 3, 17, generator=gen) * 3
    w = torch.randn(4, 3, 3, generator=gen)
    b = torch.randn(4, generator=gen)
    got = R.lowp_conv1d(x, w, b, precision=precision, in_slope=0.1, dilation=2, padding=2)
    xs = x.numpy()
    xl = np.maximum(xs, xs * np.float32(0.1))
    want = _conv_loop(rnd(xl), rnd(w.numpy()), b.double().numpy(), 2, 2)
    np.testing.assert_allclose(got.numpy(), want, rtol=1e-12, atol=1e-12)
    # the rounding is real: the fp32 conv differs by far more than float64 noise
    full = _conv_loop(xl.astype(np.float64), w.double().numpy(), b.double().numpy(), 2, 2)
    assert np.abs(full - want).max() > 1e-4


def test_reference_transposed_is_the_rounded_transposed_conv():
    gen = torch.Generator().manual_seed(6)
    x = torch.randn(1, 4, 9, generator=gen)
    w = torch.randn(4, 2, 4, generator=gen)
    got = R.lowp_conv1d(x, w, None, precision="bf16", in_slope=0.1, transposed=True, stride=2, padding=1)
    xl = torch.maximum(x, x * 0.1)
    xr = torch.from_numpy(_round_bf16(xl.numpy()))
    wr = torch.from_numpy(_round_bf16(w.numpy()))
    want = torch.nn.functional.conv_transpose1d(xr, wr, None, stride=2, padding=1)
    assert torch.allclose(got, want, rtol=1e-12, atol=1e-12)
