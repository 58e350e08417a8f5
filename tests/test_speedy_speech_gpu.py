"""SpeedySpeech on the GPU: the Conv1dBN epilogue (valid window, ReLU, per-row affine) one layer at a time against
float64 through b200tts_debug_conv1d_launch_bn, every oracle case of tests/test_speedy_speech_oracle_cpu.py against the
oracle, a ragged batch against per-row oracle calls, the bench batch with its dispatch pinned, the short-row errors,
bit-identical repeat runs and the text -> mel -> HiFiGAN chain."""
import ctypes

import pytest
import torch
import torch.nn.functional as F

import conv_check as CC
import speedy_speech_oracle as SO
import vits_oracle as O
from test_bench_scale_gpu import LAYER_REL_TOL
from test_forward_tts_gpu import check_against_oracle, gpu_inference, ragged_batch
from test_speedy_speech_oracle_cpu import CASES, round_margin, run_case, speedy_config, speedy_state
from tts_b200 import _lib
from tts_b200.forward_tts import SpeedySpeech, SpeedySpeechConfig

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
NAN = float("nan")
MARGIN = 1e-3   # pre-round durations this far from a round-half boundary cannot flip on FP32 rounding differences


# ----------------------------------------------------------------------------- one layer
def layer_ref(x, w, b, s, h, dil, lens, res, mask):
    """Conv1dBN of each row on its own (length lens[b]) in float64, + res, * mask; [B, C, T], zero past each row."""
    k = w.shape[-1]
    r = dil * (k - 1)
    out = torch.zeros(x.shape[0], w.shape[0], x.shape[2], dtype=torch.float64)
    for i, n in enumerate(lens):
        z = F.conv1d(x[i: i + 1, :, :n].double(), w.double(), b.double(), dilation=dil)
        v = F.relu(F.pad(z, (r // 2, r - r // 2))) * s.double()[:, None] + h.double()[:, None]
        if res is not None:
            v = v + res[i: i + 1, :, :n].double()
        if mask is not None:
            v = v * mask[i: i + 1, :, :n].double()
        out[i, :, :n] = v[0]
    return out


LAYERS = [(4, 1), (4, 2), (4, 4), (4, 8), (3, 1), (3, 2), (1, 1)]


@pytest.mark.parametrize("k,dil", LAYERS)
@pytest.mark.parametrize("ragged", [False, True])
@pytest.mark.parametrize("residual", [False, True])
@pytest.mark.parametrize("prec", ["fp32", "off"])
def test_conv_bn_layer_against_float64(k, dil, ragged, residual, prec):
    c, b, t = 128, 3, 300
    r = dil * (k - 1)
    g = torch.Generator().manual_seed(100 * k + dil)
    w = (torch.rand(c, c, k, generator=g) * 2 - 1) / (c * k) ** 0.5
    bias = 0.1 * torch.randn(c, generator=g)
    s = torch.randn(c, generator=g)          # negative gains too
    h = 0.1 * torch.randn(c, generator=g)
    lens = [t, r + 1, 217] if ragged else [t] * b
    x = torch.randn(b, c, t, generator=g)
    res = torch.randn(b, c, t, generator=g) if residual else None
    mask = (torch.arange(t)[None, None, :] < torch.tensor(lens)[:, None, None]).float() if residual else None
    want = layer_ref(x, w, bias, s, h, dil, lens, res, mask)
    # device tensors, NaN past every row and around every tensor; the conv is created with the front padding and sees
    # r - 2 (r // 2) more input columns than it produces, so that it produces exactly t
    tin = t + r - 2 * (r // 2)
    xp = (tin + 8 + 3) // 4 * 4                 # 16-byte rows, as the tensor-core kernels need
    xb = torch.full((b + 1, c + 4, xp), NAN, device=DEV)
    for i, n in enumerate(lens):
        xb[i, :c, :n] = x[i, :, :n].to(DEV)
    yb = torch.full((b + 1, c + 4, t + 8), NAN, device=DEV)
    cfg = _lib.Conv1dConfigC(c, c, k, dil, r // 2, 0, 1)
    hdl = ctypes.c_void_p()
    tc = prec != "off"
    _lib.check(_lib.lib().b200tts_debug_conv1d_create(ctypes.byref(cfg), _lib.ptr(w.contiguous()), _lib.ptr(bias),
                                                      int(tc), _lib.precision_id("fp32"), 0, 0, None, None,
                                                      ctypes.byref(hdl)), "debug_conv1d_create")
    keep = []
    try:
        assert _lib.lib().b200tts_conv1d_out_len(hdl, tin) == t
        io = _lib.DebugConvIOC()
        io.x, io.x_batch_stride, io.x_channel_stride, io.T = xb.data_ptr(), (c + 4) * xp, xp, tin
        io.y, io.y_batch_stride, io.y_channel_stride = yb.data_ptr(), (c + 4) * (t + 8), t + 8
        io.in_slope, io.scale, io.post_div, io.act, io.B = 1.0, 1.0, 1.0, _lib.ACT_RELU, b
        io.rate_out = io.rate_in = 1
        io.q_lo, io.q_hi, io.in_lo, io.in_hi = 0, 0x7fffffff, 0, 0x7fffffff
        io.flags = _lib.EPI_WINDOW
        if residual:
            rb = torch.full((b + 1, c, t + 4), NAN, device=DEV)
            for i, n in enumerate(lens):
                rb[i, :, :n] = res[i, :, :n].to(DEV)
            mb = torch.full((b + 1, t + 4), NAN, device=DEV)
            mb[:b, :t] = mask[:, 0].to(DEV)
            keep += [rb, mb]
            io.res, io.res_batch_stride, io.res_channel_stride = rb.data_ptr(), c * (t + 4), t + 4
            io.ymask, io.ymask_batch_stride = mb.data_ptr(), t + 4
            io.flags |= _lib.EPI_MASK_POST
        if ragged:
            lt = torch.tensor(lens, dtype=torch.int32, device=DEV)
            keep.append(lt)
            io.lens = lt.data_ptr()
        sd, hd = s.to(DEV), h.to(DEV)
        bn = _lib.DebugConvBNC(r // 2, r - r // 2, sd.data_ptr(), hd.data_ptr())
        with _lib.dispatch_log() as log:
            rc = _lib.lib().b200tts_debug_conv1d_launch_bn(hdl, ctypes.byref(io), ctypes.byref(bn),
                                                           _lib.stream_ptr(DEV))
            torch.cuda.synchronize()
        _lib.check(rc, "debug_conv1d_launch_bn")
        assert log.names == (["tc3"] if tc else ["fma"]), log.names
        got = yb[:b, :c, :t].cpu().double()
        for i, n in enumerate(lens):   # compared inside each row only
            got[i, :, n:] = 0.0
        assert torch.isfinite(got).all()
        bad, m = CC.failures(got, want, LAYER_REL_TOL)
        assert not bad, (bad, m)
        # outside the window: exactly the affine's h (times the mask)
        hv = h.to(torch.float32)
        for i, n in enumerate(lens):
            edge = list(range(r // 2)) + list(range(n - (r - r // 2), n))
            if edge and not residual:
                assert torch.equal(yb[i, :c, edge].cpu(), hv[:, None].expand(c, len(edge)))
    finally:
        _lib.lib().b200tts_conv1d_destroy(hdl)


def test_conv_bn_options_refused_where_they_would_be_ignored():
    """the Conv1dBN options with a gate, a column window or conditioning are an error, not silently dropped"""
    c, t = 64, 40
    cfg = _lib.Conv1dConfigC(c, c, 3, 1, 1, 0, 1)
    w = torch.zeros(c, c, 3)
    hdl = ctypes.c_void_p()
    _lib.check(_lib.lib().b200tts_debug_conv1d_create(ctypes.byref(cfg), _lib.ptr(w), None, 0, 0, 0, 0, None, None,
                                                      ctypes.byref(hdl)), "debug_conv1d_create")
    try:
        x = torch.zeros(1, c, t, device=DEV)
        y = torch.zeros(1, c, t, device=DEV)
        sh = torch.ones(c, device=DEV)
        cond = torch.zeros(1, c, device=DEV)
        for what in ("window", "cond", "gate", "half_affine"):
            io = _lib.DebugConvIOC()
            io.x, io.x_batch_stride, io.x_channel_stride, io.T = x.data_ptr(), c * t, t, t
            io.y, io.y_batch_stride, io.y_channel_stride = y.data_ptr(), c * t, t
            io.in_slope, io.scale, io.post_div, io.B, io.rate_out, io.rate_in = 1.0, 1.0, 1.0, 1, 1, 1
            io.q_lo, io.q_hi, io.in_lo, io.in_hi = 0, 0x7fffffff, 0, 0x7fffffff
            io.flags = _lib.EPI_WINDOW
            bn = _lib.DebugConvBNC(1, 1, sh.data_ptr(), sh.data_ptr())
            if what == "window":
                io.q_lo, io.q_hi = 8, 16
            elif what == "cond":
                io.cond, io.cond_batch_stride = cond.data_ptr(), c
            elif what == "gate":
                io.flags |= _lib.EPI_GATE
            else:
                bn.aff_h = None
            assert _lib.lib().b200tts_debug_conv1d_launch_bn(hdl, ctypes.byref(io), ctypes.byref(bn),
                                                             _lib.stream_ptr(DEV)) == 1, what
        # and the plain debug launch takes no window flag
        assert _lib.lib().b200tts_debug_conv1d_launch(hdl, ctypes.byref(io), _lib.stream_ptr(DEV)) == 1
    finally:
        _lib.lib().b200tts_conv1d_destroy(hdl)


# ----------------------------------------------------------------------------- the model
def model_for(cfg, sd, sm=None):
    m = SpeedySpeech(cfg, speaker_manager=sm).eval()
    m.load_state_dict(sd)
    return m.to(DEV)


def check(got, want, length_scale=1.0):
    assert round_margin(want, length_scale) > MARGIN
    check_against_oracle(got, want)


@pytest.mark.parametrize("case", list(CASES))
def test_speedy_speech_matches_oracle(case):
    cfg, sd, x, extra = run_case(case)
    from test_forward_tts_oracle_cpu import speaker_manager
    want = SO.inference(sd, x, cfg.model_args, **extra)
    got = gpu_inference(model_for(cfg, sd, speaker_manager(CASES[case][1])), x, None, extra)
    check(got, want, cfg.model_args.length_scale)


def test_ragged_batch_of_32_matches_per_row_oracle():
    cfg = speedy_config({}, {})
    sd = speedy_state(SpeedySpeech(cfg), 14, 5)
    x, lens = ragged_batch(cfg, 32, 40, 13, seed=3)
    want = SO.inference(sd, x, cfg.model_args, x_lengths=lens)
    got = gpu_inference(model_for(cfg, sd), x, lens)
    check(got, want)
    for i in range(32):   # padded frames exactly zero
        assert float(got["model_outputs"][i, int(got["y_lengths"][i]):].abs().sum()) == 0.0
    assert got["model_outputs"].shape[1] >= 128   # long enough for the tensor-core convs


def bench_batch(seed=0):
    """The bench workload: default SpeedySpeechConfig, 32 utterances of 40-64 tokens, duration-predictor bias log 6
    (5 frames per token)."""
    cfg = SpeedySpeechConfig(model_args=SpeedySpeechConfig().model_args)
    cfg.model_args.num_chars = 100
    sd = speedy_state(SpeedySpeech(cfg), 21, 5)
    x, lens = ragged_batch(cfg, 32, 64, 40, seed)
    return cfg, sd, x, lens


def test_bench_scale_matches_oracle_and_pins_dispatch():
    cfg, sd, x, lens = bench_batch()
    want = SO.inference(sd, x, cfg.model_args, x_lengths=lens)
    m = model_for(cfg, sd)
    with _lib.dispatch_log() as log:
        got = gpu_inference(m, x, lens)
    check(got, want)
    a = cfg.model_args
    ep, dp = a.encoder_params, a.decoder_params
    n_enc = 1 + ep["num_res_blocks"] * ep["num_conv_blocks"] + 2 + 3   # prenet, stack, postnet, duration predictor
    n_dec = dp["num_res_blocks"] * dp["num_conv_blocks"] + 1 + 2 + 1   # stack, post_conv, postnet block, postnet.1
    assert log.names == ["fma"] * n_enc + ["tc3"] * n_dec, log.names


def test_short_rows_raise_before_decoding():
    cfg, sd, x, _ = run_case("min_frames")
    m = model_for(cfg, sd)
    with pytest.raises(RuntimeError, match="12 tokens"):
        m.inference(x[:, :12].to(DEV), {})
    with pytest.raises(RuntimeError, match="24 frames"):   # 24 tokens of one frame each
        m.inference(x[:, :24].to(DEV), {})
    with pytest.raises(RuntimeError, match="12 tokens"):   # one short row in a batch
        m.inference(x.repeat(2, 1).to(DEV), {"x_lengths": torch.tensor([25, 12], device=DEV)})
    assert gpu_inference(m, x)["model_outputs"].shape[1] == 25


def test_repeat_and_poisoned_workspace_bit_identical():
    cfg, sd, x, lens = bench_batch(1)
    m = model_for(cfg, sd)
    a = gpu_inference(m, x, lens)
    b = gpu_inference(m, x, lens)
    for buf in _lib._workspaces.values():
        buf.view(torch.float32)[: buf.numel() // 4].fill_(NAN)
    c = gpu_inference(m, x, lens)
    for k in ("model_outputs", "alignments", "durations_log", "durations", "y_lengths"):
        assert torch.equal(a[k], b[k]) and torch.equal(a[k], c[k]), k


def test_wrong_weight_count_is_rejected():
    cfg, sd, _, _ = run_case("defaults")
    m = model_for(cfg, sd)
    orig = m._make

    def short(name, c, tensors):
        return orig(name, c, tensors[:-1])

    def long(name, c, tensors):
        return orig(name, c, tensors + [tensors[-1]])

    for bad, msg in ((short, "ends after"), (long, "expected")):
        m._drop_handle()
        m._make = bad
        with pytest.raises(RuntimeError, match=msg):
            m.handle(DEV)
    m._make = orig


def test_speedy_speech_to_hifigan_v2_chain():
    """SpeedySpeech -> vocoder_input -> a HiFiGAN v2-shaped generator (upsample_initial_channel 128), against the oracle
    chain."""
    from tts_b200.vocoder import GAN, AudioNorm, HifiganConfig, vocoder_input
    cfg = speedy_config(dict(out_channels=80), {})
    sd = speedy_state(SpeedySpeech(cfg), 17, 3)
    x = torch.randint(0, 40, (1, 19), generator=torch.Generator().manual_seed(9))
    want_mel = SO.inference(sd, x, cfg.model_args)["model_outputs"]
    torch.manual_seed(3)
    hc = HifiganConfig()
    hc.generator_model_params["upsample_initial_channel"] = 128
    gan = GAN(hc).eval()
    want = O.hifigan_inference(gan.model_g.state_dict(), want_mel.transpose(1, 2), 5)
    gan.to(DEV)
    mel = model_for(cfg, sd).inference(x.to(DEV), {})["model_outputs"]
    voc_in = vocoder_input(mel, AudioNorm.identity(), AudioNorm.identity(), padding=5, time_last=False, aligned=True)
    got = gan.model_g(voc_in).cpu()
    assert got.shape == want.shape
    rms = float((got - want).pow(2).mean().sqrt())
    assert rms <= 1e-4, rms
