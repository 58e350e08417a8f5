"""ForwardTTS on the GPU against the CPU oracle (tests/forward_tts_oracle.py, itself pinned to the reference): every
oracle case, the tensor-core attention kernel against float64, a ragged batch against the oracle's per-row calls, the
bench-scale batch with its dispatch pinned, bit-identical repeat runs and the text -> mel -> HiFiGAN chain."""
import math

import pytest
import torch

import forward_tts_oracle as FO
import vits_oracle as O
from test_forward_tts_oracle_cpu import CASES, SMALL, forward_state, make_config, run_case, speaker_manager
from tts_b200 import _lib
from tts_b200.forward_tts import FastPitchConfig, ForwardTTS, ForwardTTSArgs, attention

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")


def rel_rms(got, want):
    return float((got - want).pow(2).mean().sqrt() / want.pow(2).mean().sqrt().clamp_min(1e-30))


def model_for(cfg, sd, sm=None):
    m = ForwardTTS(cfg, speaker_manager=sm).eval()
    m.load_state_dict(sd)
    return m.to(DEV)


def gpu_inference(m, x, lens=None, extra=None):
    aux = {} if lens is None else {"x_lengths": lens.to(DEV)}
    aux.update({k: v.to(DEV) for k, v in (extra or {}).items()})
    out = m.inference(x.to(DEV), aux)
    return {k: (v.cpu() if torch.is_tensor(v) else v) for k, v in out.items()}


def check_against_oracle(got, want):
    assert torch.equal(got["y_lengths"], want["y_lengths"])
    assert torch.equal(got["durations"], want["durations"])
    assert torch.equal(got["alignments"], want["alignments"])
    for k in ("durations_log", "pitch", "energy"):
        if want[k] is None:
            assert got[k] is None, k
        elif float(want[k].abs().max()) == 0.0:
            assert torch.equal(got[k], want[k]), k
        else:
            assert rel_rms(got[k], want[k]) <= 1e-5, (k, rel_rms(got[k], want[k]))
    g, w = got["model_outputs"], want["model_outputs"]
    assert g.shape == w.shape
    assert rel_rms(g, w) <= 1e-4 and float((g - w).pow(2).mean().sqrt()) <= 1e-4, rel_rms(g, w)


@pytest.mark.parametrize("case", list(CASES))
def test_forward_tts_matches_oracle(case):
    cfg, sd, x, extra = run_case(case)
    want = FO.inference(sd, x, cfg.model_args, **extra)
    got = gpu_inference(model_for(cfg, sd, speaker_manager(CASES[case][2])), x, None, extra)
    check_against_oracle(got, want)


def attention_ref(qkv, lens, heads, dtype=torch.float64):
    b, c3, t = qkv.shape
    c = c3 // 3
    d = c // heads
    out = torch.zeros(b, c, t, dtype=dtype, device=qkv.device)
    for i in range(b):
        n = int(lens[i])
        q, k, v = (qkv[i, s * c:(s + 1) * c, :n].to(dtype).view(heads, d, n) for s in range(3))
        p = torch.softmax(torch.einsum("hci,hcj->hij", q * math.sqrt(1.0 / d), k), -1)
        out[i, :, :n] = torch.einsum("hij,hcj->hci", p, v).reshape(c, n)
    return out


@pytest.mark.parametrize("d,heads,t,lens", [
    (16, 4, 37, [37, 20, 1]),
    (192, 2, 1000, [1000, 777, 129]),
    (384, 1, 301, [301, 64, 65, 300]),
    (384, 1, 5000, [5000, 4999]),
])
def test_attention_kernel_against_float64(d, heads, t, lens):
    g = torch.Generator(device=DEV).manual_seed(d + t)
    b = len(lens)
    qkv = torch.randn(b, 3 * d * heads, t, generator=g, device=DEV)
    ln = torch.tensor(lens, device=DEV)
    for i, n in enumerate(lens):   # stale data past a row's end must not matter
        qkv[i, :, n:] = float("nan")
    with _lib.dispatch_log() as log:
        got = attention(qkv, ln, heads)
    assert log.names == ["attn_tc3"]
    clean = torch.nan_to_num(qkv)
    want = attention_ref(clean, ln, heads)
    f32 = attention_ref(clean, ln, heads, torch.float32)   # torch in FP32 (TF32 off): the accuracy bar
    for i, n in enumerate(lens):
        assert float(got[i, :, n:].abs().sum()) == 0.0
        err = float((got[i, :, :n].double() - want[i, :, :n]).pow(2).mean().sqrt())
        err32 = float((f32[i, :, :n].double() - want[i, :, :n]).pow(2).mean().sqrt())
        # an output row averages up to 5000 values: its relative error is set by that cancellation, so the kernel is
        # held to FP32 accuracy (within 2x of torch's FP32 result) rather than to a fixed relative bound
        assert rel_rms(got[i, :, :n].double(), want[i, :, :n]) <= 1e-5 or err <= 2 * err32, (err, err32)


def ragged_batch(cfg, n, t_max, lo, seed=0):
    g = torch.Generator().manual_seed(seed)
    lens = torch.randint(lo, t_max + 1, (n,), generator=g)
    lens[0] = t_max
    x = torch.randint(0, cfg.model_args.num_chars, (n, t_max), generator=g)
    return x, lens


def test_ragged_batch_of_32_matches_per_row_oracle():
    cfg = make_config("FastSpeech2Config", {}, {})
    sd = forward_state(ForwardTTS(cfg), 13, 5)
    x, lens = ragged_batch(cfg, 32, 40, 5, seed=3)
    want = FO.inference(sd, x, cfg.model_args, x_lengths=lens)
    got = gpu_inference(model_for(cfg, sd), x, lens)
    check_against_oracle(got, want)
    for i in range(32):   # padded frames exactly zero
        assert float(got["model_outputs"][i, int(got["y_lengths"][i]):].abs().sum()) == 0.0
    assert got["model_outputs"].shape[1] >= 128   # long enough for the tensor-core convs


def bench_batch(seed=0):
    """The bench workload: default FastPitchConfig, 32 utterances of 40-64 tokens, duration-predictor bias log 6
    (5 frames per token)."""
    cfg = FastPitchConfig(model_args=ForwardTTSArgs(num_chars=100))
    sd = forward_state(ForwardTTS(cfg), 21, 5)
    x, lens = ragged_batch(cfg, 32, 64, 40, seed)
    return cfg, sd, x, lens


def test_bench_scale_matches_oracle_and_pins_dispatch():
    cfg, sd, x, lens = bench_batch()
    want = FO.inference(sd, x, cfg.model_args, x_lengths=lens)
    m = model_for(cfg, sd)
    with _lib.dispatch_log() as log:
        got = gpu_inference(m, x, lens)
    check_against_oracle(got, want)
    a = cfg.model_args
    n_text = 4 * a.encoder_params["num_layers"] + 3 + 3 + 1   # encoder, duration / pitch predictors, pitch_emb
    per_layer = ["tc3", "attn_tc3", "tc3", "tc3", "tc3"]
    assert log.names[:n_text] == ["fma"] * n_text
    assert log.names[n_text:] == per_layer * a.decoder_params["num_layers"] + ["tc3"], log.names[n_text:]


def test_repeat_and_poisoned_workspace_bit_identical():
    cfg, sd, x, lens = bench_batch(1)
    m = model_for(cfg, sd)
    a = gpu_inference(m, x, lens)
    b = gpu_inference(m, x, lens)
    for buf in _lib._workspaces.values():
        buf.view(torch.float32)[: buf.numel() // 4].fill_(float("nan"))
    c = gpu_inference(m, x, lens)
    for k in ("model_outputs", "alignments", "durations_log", "pitch", "durations", "y_lengths"):
        assert torch.equal(a[k], b[k]) and torch.equal(a[k], c[k]), k


def test_attention_fallback_for_heads_the_tensor_cores_do_not_take():
    """d = 20 (not a multiple of 8): the decoder attention runs on the FP32-FMA kernel and says so."""
    cfg = make_config("FastPitchConfig", dict(hidden_channels=40, decoder_params={**SMALL["decoder_params"],
                                                                                  "num_heads": 2}), {})
    sd = forward_state(ForwardTTS(cfg), 5, 5)
    x, lens = ragged_batch(cfg, 4, 30, 10, seed=1)
    want = FO.inference(sd, x, cfg.model_args, x_lengths=lens)
    with _lib.dispatch_log() as log:
        got = gpu_inference(model_for(cfg, sd), x, lens)
    check_against_oracle(got, want)
    assert "attn_fma" in log.names and "attn_tc3" not in log.names


def test_forward_tts_to_hifigan_v2_chain():
    """FastPitch -> vocoder_input -> a HiFiGAN v2-shaped generator (upsample_initial_channel 128), against the oracle
    chain."""
    from tts_b200.vocoder import GAN, AudioNorm, HifiganConfig, vocoder_input
    cfg = make_config("FastPitchConfig", dict(out_channels=80), {})
    sd = forward_state(ForwardTTS(cfg), 17, 3)
    x = torch.randint(0, 40, (1, 19), generator=torch.Generator().manual_seed(9))
    want_mel = FO.inference(sd, x, cfg.model_args)["model_outputs"]
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
