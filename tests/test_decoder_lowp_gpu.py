"""Opt-in 16-bit operands for the HiFiGAN decoder (``HifiganGenerator.precision = "bf16"`` / ``"fp16"``).

Three kinds of check, for both types:
  - single layers against the 16-bit reference (tests/lowp_reference.py: the same rounded operands, float64 sums): the
    only difference left is fp32 accumulation order, so the fp32 layer tolerance applies -- a wrong rounding, slab
    order or missing tap fails by orders of magnitude;
  - within one precision everything the fp32 decoder guarantees bit-for-bit still holds (ragged, windows, streaming,
    repeat runs), and the dispatch is pinned;
  - whole models against the fp32 oracle: durations and paths are untouched (the decoder comes last), the waveform
    error stays under a bound set from H100 measurements.
"""
import pytest
import torch

import lowp_reference as R
import vits_oracle as O
from test_bench_scale_gpu import LAYER_CASES, LAYER_REL_TOL

pytestmark = pytest.mark.gpu

PRECS = ["bf16", "fp16"]
TO_16 = {"tc3": "tc16", "tc3_grouped": "tc16_grouped", None: "tc16"}
# whole-model waveform relative RMS against the fp32 oracle.  Measured on an H100 80GB HBM3 (400 W limit): bf16 1.67e-3
# (cfg1) / 1.41e-3 (cfg2), fp16 2.49e-4 / 1.82e-4 -- the bounds leave about 2.4x margin (DESIGN.md section 6)
WAV_REL_BOUND = {"bf16": 4e-3, "fp16": 6e-4}
NAN = float("nan")


def _rel_rms(got, want):
    err = got.double() - want.double()
    return float(err.pow(2).mean().sqrt() / want.double().pow(2).mean().sqrt().clamp_min(1e-30))


# ----------------------------------------------------------------------------- single layers
@pytest.mark.parametrize("precision", PRECS)
@pytest.mark.parametrize("c,k,dil,b,t,family", LAYER_CASES)
def test_layer_vs_16bit_reference(precision, c, k, dil, b, t, family):
    """ResBlock1's second-conv form with residual, accumulate and MRF mean, then the plain form; 10-45 tiles per CTA."""
    from tts_b200 import _lib
    from tts_b200.conv import FusedConv1d
    torch.manual_seed(c * 1000 + k * 10 + dil)
    w = torch.randn(c, c, k) / (c * k) ** 0.5
    bias = torch.randn(c) * 0.1
    x = torch.randn(b, c, t).cuda()
    res = torch.randn(b, c, t).cuda()
    yold = torch.randn(b, c, t).cuda()
    pad = (k * dil - dil) // 2
    conv = FusedConv1d(w, bias, dilation=dil, padding=pad, precision=precision)
    y = yold.clone()
    with _lib.dispatch_log() as log:
        got = conv(x, in_slope=0.1, residual=res, accumulate_into=y, post_div=3.0)
    torch.cuda.synchronize()
    assert _lib.lib().b200tts_debug_tc_error() == 0
    assert log.names == [TO_16[family]], log.names
    ref = R.lowp_conv1d(x, w.cuda(), bias.cuda(), precision=precision, in_slope=0.1, dilation=dil, padding=pad)
    want = (yold.double() + (ref + res.double())) / 3.0
    assert _rel_rms(got, want) <= LAYER_REL_TOL, _rel_rms(got, want)
    xs = x[:, :, : t - 76]           # another tile count; rows stay 16-byte aligned (unaligned ones take the FMA kernel)
    with _lib.dispatch_log() as log:
        got2 = conv(xs, in_slope=0.1)
    assert log.names == [TO_16[family]], log.names
    want2 = R.lowp_conv1d(xs, w.cuda(), bias.cuda(), precision=precision, in_slope=0.1, dilation=dil, padding=pad)
    assert _rel_rms(got2, want2) <= LAYER_REL_TOL, _rel_rms(got2, want2)


@pytest.mark.parametrize("precision", PRECS)
@pytest.mark.parametrize("cin,cout,k,s,b,t", [(256, 128, 16, 8, 32, 1200), (512, 256, 16, 8, 32, 152),
                                              (128, 64, 4, 2, 32, 9600), (64, 32, 4, 2, 32, 19200)])
def test_upsampler_vs_16bit_reference(precision, cin, cout, k, s, b, t):
    from tts_b200 import _lib
    from tts_b200.conv import FusedConv1d
    torch.manual_seed(cin + k)
    w = torch.randn(cin, cout, k) / (cin * k / s) ** 0.5
    bias = torch.randn(cout) * 0.1
    x = torch.randn(b, cin, t).cuda()
    conv = FusedConv1d(w, bias, padding=(k - s) // 2, transposed=True, stride=s, precision=precision)
    with _lib.dispatch_log() as log:
        got = conv(x, in_slope=0.1)
    torch.cuda.synchronize()
    assert _lib.lib().b200tts_debug_tc_error() == 0
    assert log.names == ["tc16"], log.names
    want = R.lowp_conv1d(x, w.cuda(), bias.cuda(), precision=precision, in_slope=0.1, transposed=True, stride=s,
                         padding=(k - s) // 2)
    assert got.shape == want.shape
    assert _rel_rms(got, want) <= LAYER_REL_TOL, _rel_rms(got, want)


def test_layer_with_cin_not_multiple_of_16_stays_fp32():
    """Cin % 16 != 0: the layer keeps the 3xTF32 kernel (visible as tc3 in the log) and its fp32 result."""
    from tts_b200 import _lib
    from tts_b200.conv import FusedConv1d
    torch.manual_seed(3)
    w = torch.randn(128, 24, 7) / (24 * 7) ** 0.5
    x = torch.randn(2, 24, 1000).cuda()
    want = FusedConv1d(w, padding=3)(x, in_slope=0.1)
    with _lib.dispatch_log() as log:
        got = FusedConv1d(w, padding=3, precision="bf16")(x, in_slope=0.1)
    assert log.names == ["tc3"], log.names
    assert torch.equal(got, want)


# ----------------------------------------------------------------------------- dispatch
@pytest.mark.parametrize("precision", PRECS)
def test_decoder_dispatch_is_pinned(precision):
    from tts_b200 import _lib
    from tts_b200.hifigan import HifiganGenerator
    from tts_b200.vits import Vits, VitsConfig
    torch.manual_seed(0)
    m = Vits(VitsConfig()).eval().cuda()
    z = torch.randn(2, 192, 256).cuda()
    with _lib.dispatch_log() as ref:
        m.waveform_decoder(z)
    m.waveform_decoder.precision = precision
    with _lib.dispatch_log() as log:
        m.waveform_decoder(z)
    assert len(log.names) == len(ref.names) == 1 + 4 * 19 + 1, log.names
    assert log.names[-1] == "row1", log.names                       # conv_post stays fp32
    for a, b in zip(ref.names, log.names):
        assert b == TO_16.get(a, a), (ref.names, log.names)
    assert set(log.names[:-1]) == {"tc16", "tc16_grouped"}, log.names
    mask = torch.ones(4, 1, 192).cuda()                             # the flow does not follow the decoder
    with _lib.dispatch_log() as log:
        m.flow(torch.randn(4, 192, 192).cuda(), mask, reverse=True)
    assert set(log.names) == {"tc3"} and len(log.names) == 4 * (2 + 2 * 4), log.names
    # in_channels = 20: conv_pre cannot take 16-bit operands and stays on the 3xTF32 kernel, visibly
    g = HifiganGenerator(20, 1, "1", [[1, 3, 5]] * 3, [3, 7, 11], [16, 16, 4, 4], 512, [8, 8, 2, 2]).eval().cuda()
    g.precision = precision
    with _lib.dispatch_log() as log:
        g(torch.randn(2, 20, 256).cuda())
    assert log.names[0] == "tc3" and log.names[-1] == "row1", log.names
    assert set(log.names[1:-1]) == {"tc16", "tc16_grouped"}, log.names


# ----------------------------------------------------------------------------- exactness within one precision
def _decoder(precision, cond=0):
    from tts_b200.hifigan import HifiganGenerator
    m = HifiganGenerator(in_channels=192, out_channels=1, resblock_type="1", resblock_dilation_sizes=[[1, 3, 5]] * 3,
                         resblock_kernel_sizes=[3, 7, 11], upsample_kernel_sizes=[16, 16, 4, 4],
                         upsample_initial_channel=512, upsample_factors=[8, 8, 2, 2], inference_padding=0,
                         cond_channels=cond, conv_pre_weight_norm=False, conv_post_weight_norm=False,
                         conv_post_bias=False).eval().cuda()
    m.precision = precision
    return m


def _poison_workspace(m, z):
    from tts_b200 import _lib
    b, _, t = z.shape
    h = m._ensure_handle(z.device)
    _lib.workspace(z.device, _lib.lib().b200tts_hifigan_workspace_bytes(h, b, t), "hifigan").fill_(255)   # NaN


@pytest.mark.parametrize("precision", PRECS)
def test_ragged_windows_and_repeat_runs_are_exact(precision):
    torch.manual_seed(21)
    m = _decoder(precision, cond=256)
    lens = [150, 97, 33, 2]
    b, t = len(lens), 150
    mask = (torch.arange(t)[None, :] < torch.tensor(lens)[:, None]).float().unsqueeze(1)
    z = (torch.randn(b, 192, t) * mask).cuda()
    g = torch.randn(b, 256, 1).cuda()
    full = m(z, g)
    assert torch.isfinite(full).all()
    assert torch.equal(m(z, g), full)                                # two runs
    lt = torch.tensor(lens).cuda()
    ragged = m(z, g, lengths=lt)
    valid = (torch.arange(t * 256)[None, None, :] < (torch.tensor(lens) * 256)[:, None, None]).cuda()
    assert torch.equal(ragged[valid], full[valid])                  # ragged == dense on the valid samples
    for lengths, want in ((None, full), (lt, ragged)):
        out = torch.full_like(full, NAN)
        for f0 in range(0, t, 32):
            _poison_workspace(m, z)
            m.forward_window(z, g, start=f0, end=min(t, f0 + 32), lengths=lengths, out=out)
        assert torch.equal(out, want)


def _perturb(m, seed):
    gen = torch.Generator().manual_seed(seed)
    for _, p in m.named_parameters():
        if float(p.detach().abs().sum()) == 0.0:
            p.data.copy_(torch.randn(p.shape, generator=gen) * 0.05)


@pytest.mark.parametrize("precision", PRECS)
def test_inference_stream_equals_inference(precision):
    from tts_b200.vits import Vits, VitsConfig
    torch.manual_seed(8)
    m = Vits(VitsConfig()).eval()
    _perturb(m, 1)
    m = m.cuda()
    m.trim_padding = True
    m.waveform_decoder.precision = precision
    lens = torch.tensor([64, 50, 33, 20, 11, 64])
    gen = torch.Generator().manual_seed(3)
    tok = (torch.randint(0, 100, (6, 64), generator=gen) * (torch.arange(64)[None, :] < lens[:, None])).cuda()
    aux = {"x_lengths": lens.cuda()}
    noise = torch.randn(6, 2, 64, generator=gen)
    prior = torch.randn(6, 192, 4096, generator=torch.Generator().manual_seed(2)).cuda()
    full = m.inference(tok, aux, sdp_noise=noise, prior_noise=lambda s: prior[:, :, : s[-1]])
    chunks = list(m.inference_stream(tok, aux, chunk_frames=24, sdp_noise=noise,
                                     prior_noise=lambda s: prior[:, :, : s[-1]]))
    assert torch.equal(torch.cat([c["model_outputs"] for c in chunks], dim=-1), full["model_outputs"])


# ----------------------------------------------------------------------------- whole models against the fp32 oracle
@pytest.mark.parametrize("precision", PRECS)
def test_cfg1_standalone_hifigan_vs_fp32_oracle(precision):
    """BASELINE configs[0]: HifiganGenerator(80, 1, '1', ...) on randn(4, 80, 256), weight norm removed."""
    from tts_b200.hifigan import HifiganGenerator
    torch.manual_seed(1234)
    m = HifiganGenerator(80, 1, "1", [[1, 3, 5]] * 3, [3, 7, 11], [16, 16, 4, 4], 512, [8, 8, 2, 2]).eval()
    mel = torch.randn(4, 80, 256)
    want = O.hifigan_forward(m.state_dict(), mel)
    m.remove_weight_norm()
    m.cuda().precision = precision
    got = m(mel.cuda())
    assert got.shape == (4, 1, 65536)
    assert torch.isfinite(got).all()
    rel = _rel_rms(got.cpu(), want)
    print(f"cfg1 {precision}: waveform relative RMS vs the fp32 oracle {rel:.3e}")
    assert rel <= WAV_REL_BOUND[precision], rel


@pytest.fixture(scope="module")
def cfg2_case():
    """bench.py's cfg2 batch (32 x 64 tokens, VitsConfig defaults) with fixed noise, and the fp32 oracle on 8 of its rows
    (the longest utterance among them, so the padded length -- hence every row's arithmetic -- is the full batch's)."""
    from tts_b200.vits import Vits, VitsConfig
    from dataclasses import asdict
    cfg = VitsConfig()
    torch.manual_seed(1234)
    m = Vits(cfg).eval()
    _perturb(m, 1234)
    sd = {k: v.clone() for k, v in m.state_dict().items()}
    gen = torch.Generator().manual_seed(4321)
    tok = torch.randint(0, 100, (32, 64), generator=gen)
    lens = torch.full((32,), 64)
    sdp_noise = torch.randn(32, 2, 64, generator=torch.Generator().manual_seed(1235))
    store = {}

    def prior_noise(shape):
        if "n" not in store:
            store["n"] = torch.randn(shape, generator=torch.Generator().manual_seed(1236))
        return store["n"].cuda()

    m.cuda()
    aux = {"x_lengths": lens.cuda()}
    fp32 = m.inference(tok.cuda(), aux, sdp_noise=sdp_noise, prior_noise=prior_noise)
    ylen = fp32["y_lengths"].cpu()
    longest = int(ylen.argmax())
    others = [i for i in torch.randperm(32, generator=torch.Generator().manual_seed(1237)).tolist() if i != longest]
    rows = torch.tensor(sorted([longest] + others[:7]))
    a = asdict(cfg.model_args)
    want = O.vits_inference(sd, tok[rows], lens[rows], sdp_noise[rows], lambda s: store["n"][rows], args=a)
    return dict(model=m, tok=tok.cuda(), aux=aux, sdp_noise=sdp_noise, prior_noise=prior_noise, rows=rows, want=want,
                fp32=fp32)


@pytest.mark.parametrize("precision", PRECS)
def test_cfg2_vits_inference_vs_fp32_oracle(cfg2_case, precision):
    c = cfg2_case
    m, rows, want = c["model"], c["rows"], c["want"]
    m.waveform_decoder.precision = precision
    try:
        got = m.inference(c["tok"], c["aux"], sdp_noise=c["sdp_noise"], prior_noise=c["prior_noise"])
    finally:
        m.waveform_decoder.precision = "fp32"
    torch.cuda.synchronize()
    for k in ("durations", "y_lengths", "alignments", "y_mask"):      # everything before the decoder is untouched
        assert torch.equal(got[k].cpu()[rows], want[k]), k
        assert torch.equal(got[k], c["fp32"][k]), k
    wav = got["model_outputs"]
    assert torch.isfinite(wav).all()
    n = want["model_outputs"].shape[-1]
    valid = (torch.arange(n)[None, None, :] < (want["y_lengths"] * 256)[:, None, None])
    g, w = wav.cpu()[rows][valid], want["model_outputs"][valid]
    rel = _rel_rms(g, w)
    rel32 = _rel_rms(c["fp32"]["model_outputs"].cpu()[rows][valid], w)
    print(f"cfg2 {precision}: waveform relative RMS vs the fp32 oracle {rel:.3e} (fp32 decoder: {rel32:.3e})")
    assert rel <= WAV_REL_BOUND[precision], rel


@pytest.mark.parametrize("precision", PRECS)
def test_switching_back_to_fp32_is_exact(precision):
    torch.manual_seed(31)
    m = _decoder(precision)
    fresh = _decoder("fp32")
    fresh.load_state_dict(m.state_dict())
    z = torch.randn(2, 192, 130).cuda()
    low = m(z)
    m.precision = "fp32"
    back = m(z)
    want = fresh(z)
    assert torch.equal(back, want)
    assert not torch.equal(low, want)
