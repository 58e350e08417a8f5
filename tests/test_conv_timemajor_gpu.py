"""The time-major split-fp16 kernel (conv_tc3.cuh tm_consumers) behind the `tc3_grouped` dispatch at f16x3: layers with
exactly 32 or 64 output rows run as M = time, N = channels, every tap summed in the accumulator.

The longest-reach layers the grouped predicate admits take 128-column tiles (a 256-column window would not fit the
staging rows); they are checked against float64 with a residual, an accumulate operand and a final divide, at a length
that leaves an edge tile.  A decoder whose 64- and 32-channel stages hold such layers must give the same samples, bit
for bit, in a ragged call as in the dense one, and in column windows as in the one-shot call: each column's sum does not
depend on where its tile starts."""
import math

import pytest
import torch

import conv_check as CC
from test_bench_scale_gpu import LAYER_REL_TOL
from test_stream_gpu import _stream

pytestmark = pytest.mark.gpu


# (rows, K, dil): the grouped predicate's window round8(256 + (ceil(K / G) - 1) * G * dil) <= 320 with G = 128 / rows,
# and (G - 1) * dil <= 15.  Reach (K - 1) * dil = 75 and 76 are the longest it admits for 64 / 32 rows (beyond the 64
# of a 256-column tile); at 64 rows a reach of 60 also takes 128-column tiles (shared memory).  K = 6 at dilation 15
# gives Tout = T - 1, rows that are not 16-byte aligned: every tile takes the bounds-checked epilogue.
LONG_REACH = [(64, 6, 15), (64, 7, 10), (32, 20, 4)]


@pytest.mark.parametrize("rows,k,dil", LONG_REACH)
@pytest.mark.parametrize("form", ["plain", "residual", "accumulate"])
def test_long_reach_layer_against_float64(rows, k, dil, form):
    from tts_b200.conv import FusedConv1d
    from tts_b200 import _lib
    dev = torch.device("cuda", 0)
    torch.manual_seed(rows * 1000 + k * 10 + len(form))
    cin, b, t = 64, 5, 128 * 9 + 36                    # nine whole tiles and an edge tile per row
    w = torch.randn(rows, cin, k, dtype=torch.float64) / math.sqrt(cin * k)
    bias = torch.randn(rows, dtype=torch.float64) * 0.1
    pad = dil * (k - 1) // 2
    tout = t + 2 * pad - dil * (k - 1)
    conv = FusedConv1d(w, bias, dilation=dil, padding=pad, precision="f16x3")
    x = torch.randn(b, cin, t, device=dev)
    r = torch.randn(b, rows, tout, device=dev) if form != "plain" else None
    old = torch.randn(b, rows, tout, device=dev) if form == "accumulate" else None
    post_div = 3.0 if form == "accumulate" else 1.0
    with _lib.dispatch_log() as log:
        y = conv(x, in_slope=0.1, residual=r, accumulate_into=None if old is None else old.clone(), post_div=post_div)
    torch.cuda.synchronize()
    assert log.names == ["tc3_grouped"], log.names
    assert _lib.lib().b200tts_debug_tc_error() == 0
    want = CC.epilogue(CC.conv(x, w.to(dev), bias.to(dev), dilation=dil, padding=pad, in_slope=0.1),
                       residual=r, y_old=old, post_div=post_div)
    fails, m = CC.failures(y, want, LAYER_REL_TOL)
    assert not fails, (fails, m)


def _long_reach_decoder():
    """Stages of 64 and 32 channels; kernel size 6 at dilation 15 (64 channels) is a 128-column time-major layer, the
    dilations 1 and 5 take 256-column tiles."""
    from tts_b200.hifigan import HifiganGenerator
    return HifiganGenerator(in_channels=32, out_channels=1, resblock_type="1", resblock_dilation_sizes=[[1, 15, 5]],
                            resblock_kernel_sizes=[6], upsample_kernel_sizes=[4, 4], upsample_initial_channel=128,
                            upsample_factors=[2, 2], inference_padding=0, cond_channels=0, conv_pre_weight_norm=False,
                            conv_post_weight_norm=False, conv_post_bias=False).eval()   # default precision: split fp16


def test_long_reach_decoder_ragged_and_windows_match_dense():
    from tts_b200 import _lib
    torch.manual_seed(11)
    m = _long_reach_decoder().cuda()
    lens = [700, 433, 96, 250]
    t = max(lens)
    mask = (torch.arange(t)[None, :] < torch.tensor(lens)[:, None]).float().unsqueeze(1)
    z = (torch.randn(len(lens), 32, t) * mask).cuda()
    with _lib.dispatch_log() as log:
        dense = m(z)
    assert log.names.count("tc3_grouped") >= 3, log.names
    lt = torch.tensor(lens).cuda()
    ragged = m(z, lengths=lt)
    torch.cuda.synchronize()
    assert torch.isfinite(dense).all()
    for i, n in enumerate(lens):
        assert torch.equal(ragged[i, :, : n * m.hop], dense[i, :, : n * m.hop]), (i, n)
    assert torch.equal(_stream(m, z, 97), dense)
    assert torch.equal(_stream(m, z, 97, lengths=lt), ragged)
    assert _lib.lib().b200tts_debug_tc_error() == 0
