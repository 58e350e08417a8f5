"""The HiFiGAN decoder's default arithmetic: the 3-product fp16 split (B200TTS_PRECISION_F16X3, FusedConv1d precision
"f16x3"), against float64 and against the 3xTF32 build ("tf32x3").

  - single layers (every LAYER_CASES shape, the four upsamplers) against float64 at the fp32 layer tolerance, also with
    the input scaled by 1e-3 and 1e3: the weights are scaled per row into fp16's range and the activations split into
    two fp16 terms, so neither a small nor a large (but < 65504) input may cost accuracy;
  - an activation fp16 cannot hold is reported, once, instead of turning into inf silently;
  - whole models against the fp32 oracle: everything before the decoder is untouched, and the waveform error stays
    within 2x of the tf32x3 build's on the same inputs;
  - the dispatch is the tf32x3 build's (tc3 / tc3_grouped), and the arithmetic really differs from it.
"""
import pytest
import torch
import torch.nn.functional as F

import vits_oracle as O
from test_bench_scale_gpu import LAYER_CASES, LAYER_REL_TOL
from test_decoder_lowp_gpu import _perturb, _rel_rms, cfg2_case  # noqa: F401  (cfg2_case is a fixture)

pytestmark = pytest.mark.gpu

SCALES = [1.0, 1e-3, 1e3]
UPSAMPLERS = [(256, 128, 16, 8, 32, 1200), (512, 256, 16, 8, 32, 152), (128, 64, 4, 2, 32, 9600), (64, 32, 4, 2, 32, 19200)]


def _tc_error():
    from tts_b200 import _lib
    return _lib.lib().b200tts_debug_tc_error()


# ----------------------------------------------------------------------------- single layers vs float64
@pytest.mark.parametrize("scale", SCALES)
@pytest.mark.parametrize("c,k,dil,b,t,family", LAYER_CASES)
def test_layer_vs_float64(scale, c, k, dil, b, t, family):
    """ResBlock1's second-conv form with residual, accumulate and MRF mean, then the plain form."""
    from tts_b200 import _lib
    from tts_b200.conv import FusedConv1d
    torch.manual_seed(c * 1000 + k * 10 + dil)
    w = torch.randn(c, c, k) / (c * k) ** 0.5
    bias = torch.randn(c) * 0.1 * scale
    x = (torch.randn(b, c, t) * scale).cuda()
    res = (torch.randn(b, c, t) * scale).cuda()
    yold = (torch.randn(b, c, t) * scale).cuda()
    pad = (k * dil - dil) // 2
    conv = FusedConv1d(w, bias, dilation=dil, padding=pad, precision="f16x3")
    y = yold.clone()
    with _lib.dispatch_log() as log:
        got = conv(x, in_slope=0.1, residual=res, accumulate_into=y, post_div=3.0)
    torch.cuda.synchronize()
    assert _tc_error() == 0
    assert log.names == [family or "tc3"], log.names
    w64, b64 = w.double().cuda(), bias.double().cuda()
    ref = F.conv1d(F.leaky_relu(x.double(), 0.1), w64, b64, dilation=dil, padding=pad)
    want = (yold.double() + (ref + res.double())) / 3.0
    assert _rel_rms(got, want) <= LAYER_REL_TOL, _rel_rms(got, want)
    xs = x[:, :, : t - 76]
    got2 = conv(xs, in_slope=0.1)
    want2 = F.conv1d(F.leaky_relu(xs.double(), 0.1), w64, b64, dilation=dil, padding=pad)
    assert _rel_rms(got2, want2) <= LAYER_REL_TOL, _rel_rms(got2, want2)


@pytest.mark.parametrize("scale", SCALES)
@pytest.mark.parametrize("cin,cout,k,s,b,t", UPSAMPLERS)
def test_upsampler_vs_float64(scale, cin, cout, k, s, b, t):
    from tts_b200 import _lib
    from tts_b200.conv import FusedConv1d
    torch.manual_seed(cin + k)
    w = torch.randn(cin, cout, k) / (cin * k / s) ** 0.5
    bias = torch.randn(cout) * 0.1 * scale
    x = (torch.randn(b, cin, t) * scale).cuda()
    conv = FusedConv1d(w, bias, padding=(k - s) // 2, transposed=True, stride=s, precision="f16x3")
    with _lib.dispatch_log() as log:
        got = conv(x, in_slope=0.1)
    torch.cuda.synchronize()
    assert _tc_error() == 0
    assert log.names == ["tc3"], log.names
    want = F.conv_transpose1d(F.leaky_relu(x.double(), 0.1), w.double().cuda(), bias.double().cuda(), stride=s,
                              padding=(k - s) // 2)
    assert got.shape == want.shape
    assert _rel_rms(got, want) <= LAYER_REL_TOL, _rel_rms(got, want)


def test_rows_of_very_different_scale():
    """Each output row gets its own power-of-two scale: rows 2^-20 and 2^20 apart keep the same relative accuracy."""
    from tts_b200.conv import FusedConv1d
    torch.manual_seed(5)
    w = torch.randn(128, 64, 7) / (64 * 7) ** 0.5
    w[:32] *= 2.0 ** -20
    w[32:64] *= 2.0 ** 20
    w[64:70] = 0.0                                                 # all-zero rows
    x = torch.randn(4, 64, 3000).cuda()
    got = FusedConv1d(w, padding=3, precision="f16x3")(x, in_slope=0.1)
    want = F.conv1d(F.leaky_relu(x.double(), 0.1), w.double().cuda(), padding=3)
    for rows in (slice(0, 32), slice(32, 64), slice(70, 128)):
        assert _rel_rms(got[:, rows], want[:, rows]) <= LAYER_REL_TOL, rows
    assert torch.equal(got[:, 64:70], torch.zeros_like(got[:, 64:70]))


# ----------------------------------------------------------------------------- range guard
def test_activation_outside_fp16_range_is_reported():
    from tts_b200.conv import FusedConv1d
    torch.manual_seed(6)
    w = torch.randn(128, 64, 3) / (64 * 3) ** 0.5
    conv = FusedConv1d(w, padding=1, precision="f16x3")
    x = torch.randn(2, 64, 1000).cuda()
    below = x.clone()
    below[1, 5, 300] = 65000.0                                     # still an fp16 value: no error
    conv(below, in_slope=0.1)
    torch.cuda.synchronize()
    assert _tc_error() == 0
    for big, slope in ((65504.0, 0.1), (-1e6, 0.1)):               # the limit itself; a negative one after the leaky ReLU
        bad = x.clone()
        bad[1, 7, 500] = big
        conv(bad, in_slope=slope)
        torch.cuda.synchronize()
        assert _tc_error() == 2
        with pytest.raises(RuntimeError, match="65504"):           # the next launch reports it ...
            conv(x, in_slope=0.1)
        assert _tc_error() == 0                                    # ... once: the device is fine
        assert torch.isfinite(conv(x, in_slope=0.1)).all()
    # 3xTF32 takes the same input
    got = FusedConv1d(w, padding=1, precision="tf32x3")(bad, in_slope=0.1)
    torch.cuda.synchronize()
    assert _tc_error() == 0 and torch.isfinite(got).all()


# ----------------------------------------------------------------------------- dispatch and selection
def test_decoder_dispatch_is_pinned():
    from tts_b200 import _lib
    from tts_b200.vits import Vits, VitsConfig
    torch.manual_seed(0)
    m = Vits(VitsConfig()).eval().cuda()
    z = torch.randn(2, 192, 256).cuda()
    dec = m.waveform_decoder
    out, names = {}, {}
    for p in ("tf32x3", "fp32", "f16x3"):
        dec.precision = p
        with _lib.dispatch_log() as log:
            out[p] = dec(z)
        names[p] = log.names
        assert _lib.lib().b200tts_hifigan_precision(dec._handle) == _lib.PRECISIONS[p]
    assert names["fp32"] == names["tf32x3"] == names["f16x3"], names
    assert len(names["fp32"]) == 1 + 4 * 19 + 1 and names["fp32"][-1] == "row1", names["fp32"]
    assert set(names["fp32"][:-1]) == {"tc3", "tc3_grouped"}, names["fp32"]
    assert torch.equal(out["fp32"], out["f16x3"])                 # "fp32" is the split-fp16 arithmetic ...
    assert not torch.equal(out["fp32"], out["tf32x3"])            # ... which is not 3xTF32
    assert _rel_rms(out["fp32"], out["tf32x3"]) <= 1e-4
    with _lib.dispatch_log() as log:                               # the flow keeps 3xTF32
        m.flow(torch.randn(4, 192, 192).cuda(), torch.ones(4, 1, 192).cuda(), reverse=True)
    assert set(log.names) == {"tc3"} and len(log.names) == 4 * (2 + 2 * 4), log.names


# ----------------------------------------------------------------------------- whole models against the fp32 oracle
def test_cfg1_standalone_hifigan_vs_fp32_oracle():
    """BASELINE configs[0]: HifiganGenerator(80, 1, '1', ...) on randn(4, 80, 256), weight norm removed."""
    from tts_b200.hifigan import HifiganGenerator
    torch.manual_seed(1234)
    m = HifiganGenerator(80, 1, "1", [[1, 3, 5]] * 3, [3, 7, 11], [16, 16, 4, 4], 512, [8, 8, 2, 2]).eval()
    mel = torch.randn(4, 80, 256)
    want = O.hifigan_forward(m.state_dict(), mel)
    m.remove_weight_norm()
    m.cuda()
    rel = {}
    for p in ("tf32x3", "fp32"):
        m.precision = p
        got = m(mel.cuda())
        assert got.shape == (4, 1, 65536) and torch.isfinite(got).all()
        rel[p] = _rel_rms(got.cpu(), want)
    print(f"cfg1: waveform relative RMS vs the fp32 oracle {rel}")
    assert rel["fp32"] <= 2 * rel["tf32x3"], rel


def test_cfg2_vits_inference_vs_fp32_oracle(cfg2_case):
    """cfg2_case's run is the default (split-fp16) decoder; this adds the tf32x3 build on the same inputs."""
    c = cfg2_case
    m, rows, want = c["model"], c["rows"], c["want"]
    m.waveform_decoder.precision = "tf32x3"
    try:
        tf = m.inference(c["tok"], c["aux"], sdp_noise=c["sdp_noise"], prior_noise=c["prior_noise"])
    finally:
        m.waveform_decoder.precision = "fp32"
    torch.cuda.synchronize()
    got = c["fp32"]
    for k in ("durations", "y_lengths", "alignments", "y_mask"):
        assert torch.equal(got[k].cpu()[rows], want[k]), k
        assert torch.equal(got[k], tf[k]), k
    assert torch.isfinite(got["model_outputs"]).all()
    n = want["model_outputs"].shape[-1]
    valid = (torch.arange(n)[None, None, :] < (want["y_lengths"] * 256)[:, None, None])
    w = want["model_outputs"][valid]
    rel = _rel_rms(got["model_outputs"].cpu()[rows][valid], w)
    rel_tf = _rel_rms(tf["model_outputs"].cpu()[rows][valid], w)
    print(f"cfg2: waveform relative RMS vs the fp32 oracle: default {rel:.3e}, tf32x3 {rel_tf:.3e}")
    assert rel <= 2 * rel_tf, (rel, rel_tf)
