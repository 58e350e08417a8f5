"""Split-fp16 ("f16x3") layers whose weight rows span more than fp16's normal range: the third product's weight,
W_hi * 2^-11, is made by the kernel from W_hi, and for elements more than 2^17 below their row's max it is subnormal
or zero in fp16.  Such rows must keep the layer tolerance against float64, in the plain and in both grouped kernels."""
import pytest
import torch
import torch.nn.functional as F

from test_bench_scale_gpu import LAYER_REL_TOL
from test_decoder_lowp_gpu import _rel_rms

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("rows,family", [(128, "tc3"), (64, "tc3_grouped"), (32, "tc3_grouped")])
def test_rows_spanning_beyond_fp16_normal_range(rows, family):
    from tts_b200 import _lib
    from tts_b200.conv import FusedConv1d
    torch.manual_seed(7 + rows)
    cin, k = 64, 7
    w = torch.randn(rows, cin, k) / (cin * k) ** 0.5
    # every element scaled by 2^-u, u uniform in [0, 40): most of a row lies far below its max, many of them more
    # than 2^17 (W_hs subnormal) or 2^28 (W_hs zero) below it
    w *= torch.exp2(-40.0 * torch.rand(rows, cin, k))
    w[:, 0, 0] = 1.0                                                   # each row's max, at a known place
    w[rows // 2:] *= 2.0 ** -60                                        # rows of a tiny overall scale keep their accuracy
    below = w.abs() < w.abs().amax(dim=(1, 2), keepdim=True) * 2.0 ** -17
    assert below.float().mean() > 0.5
    x = torch.randn(4, cin, 3000).cuda()
    conv = FusedConv1d(w, padding=3, precision="f16x3")
    with _lib.dispatch_log() as log:
        got = conv(x, in_slope=0.1)
    torch.cuda.synchronize()
    assert log.names == [family], log.names
    want = F.conv1d(F.leaky_relu(x.double(), 0.1), w.double().cuda(), padding=3)
    # row by row: a row's error is measured against its own scale
    for r in range(rows):
        assert _rel_rms(got[:, r], want[:, r]) <= LAYER_REL_TOL, (r, _rel_rms(got[:, r], want[:, r]))
