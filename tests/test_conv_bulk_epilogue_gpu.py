"""The tensor-core conv's bulk epilogue (conv_tc3.cuh): whole interior tiles of plain layers without an accumulate
operand are finished per consumer warp, with the residual prefetched into shared memory during the MMAs and the output
written with bulk stores; edge tiles and accumulate layers keep the shared-tile epilogue.

Each layer runs at Tout = 256 m + 100 with enough batch rows that every CTA of the persistent grid runs several tiles,
interior and edge ones interleaved (m + 1 tiles per row, coprime with the SM count), so both epilogues follow each other
inside one CTA.  Results are held to float64 with conv_check's bounds, and two launches into NaN-poisoned output buffers
must agree bit for bit (a race between the paths, or a row / column a bulk copy misses, shows up as a NaN or a
difference).  The in-place residual case (residual == output, as the decoder's ResBlocks run) must equal the
out-of-place one exactly."""
import ctypes
import math

import pytest
import torch

import conv_check as CC
from test_bench_scale_gpu import LAYER_REL_TOL

pytestmark = pytest.mark.gpu

NAN = float("nan")


def _tiles_per_row(sms):
    """m + 1 tiles per row (m interior, one edge tile), coprime with the SM count: every CTA meets both kinds."""
    return next(n for n in (5, 7, 3, 11) if math.gcd(n, sms) == 1)


def _launch(conv, x, y, residual, slope):
    """One b200tts_conv1d_forward into the caller's output buffer `y` (residual may be `y` itself)."""
    from tts_b200 import _lib
    h = conv._handle(x.device)
    L = _lib.lib()
    b, _, t = x.shape
    with torch.cuda.device(x.device), _lib.dispatch_log() as log:
        rc = L.b200tts_conv1d_forward(h, _lib.ptr(x), b, t, ctypes.c_float(slope), _lib.ptr(residual),
                                      ctypes.c_float(1.0), 0, ctypes.c_float(1.0), _lib.ptr(y), _lib.stream_ptr(x.device))
    _lib.check(rc, "conv1d_forward")
    return log.names


@pytest.mark.parametrize("precision", ["f16x3", "tf32x3"])
@pytest.mark.parametrize("res", [False, True])
@pytest.mark.parametrize("k", [3, 11])
@pytest.mark.parametrize("c", [128, 256])
def test_bulk_epilogue_against_float64(c, k, res, precision):
    from tts_b200.conv import FusedConv1d
    dev = torch.device("cuda", 0)
    sms = torch.cuda.get_device_properties(dev).multi_processor_count
    nt = _tiles_per_row(sms)
    t = 256 * (nt - 1) + 100
    b = -(-2 * sms // (c // 128))                      # at least two tiles of every residue per CTA
    torch.manual_seed(c * 100 + k * 10 + res)
    dil = 3 if k == 3 else 1
    w = torch.randn(c, c, k, dtype=torch.float64) / math.sqrt(c * k)
    bias = torch.randn(c, dtype=torch.float64) * 0.1
    x = torch.randn(b, c, t, device=dev)
    r = torch.randn(b, c, t, device=dev) if res else None
    conv = FusedConv1d(w, bias, dilation=dil, padding=dil * (k - 1) // 2, precision=precision)
    ys = []
    for _ in range(2):
        y = torch.full((b, c, t), NAN, device=dev)
        names = _launch(conv, x, y, r, 0.1)
        assert names == ["tc3"], names
        ys.append(y)
    torch.cuda.synchronize()
    assert torch.equal(ys[0], ys[1])
    want = CC.epilogue(CC.conv(x, w.to(dev), bias.to(dev), dilation=dil, padding=dil * (k - 1) // 2, in_slope=0.1),
                       residual=r)
    fails, m = CC.failures(ys[0], want, LAYER_REL_TOL)
    assert not fails, (fails, m)
    if res:                                            # the decoder's in-place residual: y = conv(x) + y
        y = r.clone()
        _launch(conv, x, y, y, 0.1)
        torch.cuda.synchronize()
        assert torch.equal(y, ys[0])


@pytest.mark.parametrize("precision", ["f16x3", "tf32x3"])
def test_accumulate_layer_keeps_shared_tile_epilogue(precision):
    """A layer with an accumulate operand takes the shared-tile epilogue on every tile: ((conv + res) + y_old)."""
    from tts_b200.conv import FusedConv1d
    dev = torch.device("cuda", 0)
    sms = torch.cuda.get_device_properties(dev).multi_processor_count
    c, k, t = 128, 3, 256 * (_tiles_per_row(sms) - 1) + 100
    b = 2 * sms
    torch.manual_seed(7)
    w = torch.randn(c, c, k, dtype=torch.float64) / math.sqrt(c * k)
    bias = torch.randn(c, dtype=torch.float64) * 0.1
    x, r, old = (torch.randn(b, c, t, device=dev) for _ in range(3))
    conv = FusedConv1d(w, bias, dilation=1, padding=1, precision=precision)
    outs = []
    for _ in range(2):
        y = old.clone()
        outs.append(conv(x, in_slope=0.1, residual=r, accumulate_into=y))
    torch.cuda.synchronize()
    assert torch.equal(outs[0], outs[1])
    want = CC.epilogue(CC.conv(x, w.to(dev), bias.to(dev), padding=1, in_slope=0.1), residual=r, y_old=old)
    fails, m = CC.failures(outs[0], want, LAYER_REL_TOL)
    assert not fails, (fails, m)


def test_ragged_decoder_bulk_tiles_match_dense():
    """A ragged decoder call (per-row tile schedules, rows ending mid-tile) equals the dense call on valid samples and
    is repeatable bit for bit."""
    from tts_b200.hifigan import HifiganGenerator
    torch.manual_seed(3)
    m = HifiganGenerator(in_channels=192, out_channels=1, resblock_type="1", resblock_dilation_sizes=[[1, 3, 5]] * 3,
                         resblock_kernel_sizes=[3, 7, 11], upsample_kernel_sizes=[16, 16, 4, 4],
                         upsample_initial_channel=512, upsample_factors=[8, 8, 2, 2], inference_padding=0,
                         cond_channels=0, conv_pre_weight_norm=False, conv_post_weight_norm=False,
                         conv_post_bias=False).eval().cuda()
    lens = [48, 37, 9, 21]
    lens_t = torch.tensor(lens)
    t = max(lens)
    mask = (torch.arange(t)[None, :] < lens_t[:, None]).float().unsqueeze(1)
    z = (torch.randn(len(lens), 192, t) * mask).cuda()
    dense = m(z)
    ragged = m(z, lengths=lens_t.cuda())
    again = m(z, lengths=lens_t.cuda())
    torch.cuda.synchronize()
    assert torch.equal(ragged, again)
    for i, n in enumerate(lens):
        assert torch.equal(ragged[i, :, : n * 256], dense[i, :, : n * 256]), (i, n)
    assert torch.isfinite(dense).all()
