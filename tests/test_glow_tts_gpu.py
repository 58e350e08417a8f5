"""GlowTTS on the GPU against the CPU oracle (tests/glow_oracle.py, itself pinned to the reference): every configuration
of the oracle tests at a small size, the bench-scale batch, bit-identical repeat runs, the dispatch of the decoder's
WaveNet convs and the text path, and the text -> mel -> HiFiGAN chain."""
import math

import pytest
import torch

import glow_oracle as GO
import vits_oracle as O
from test_glow_oracle_cpu import CASES, glow_state, run_case
from tts_b200 import _lib
from tts_b200.glow_tts import GlowTTS, GlowTTSConfig

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")


def rel_rms(got, want):
    return float((got - want).pow(2).mean().sqrt() / want.pow(2).mean().sqrt().clamp_min(1e-30))


def model_for(cfg, sd):
    m = GlowTTS(cfg).eval()
    m.load_state_dict(sd)
    return m.to(DEV)


def gpu_inference(m, x, lens, extra, noise):
    aux = {"x_lengths": lens.to(DEV)}
    aux.update({k: v.to(DEV) for k, v in extra.items()})
    out = m.inference(x.to(DEV), aux, noise=None if noise is None else noise.to(DEV))
    return {k: (v.cpu() if torch.is_tensor(v) else v) for k, v in out.items()}


def check_against_oracle(got, want):
    assert torch.equal(got["y_lengths"], want["y_lengths"])
    assert torch.equal(got["durations"], want["durations"])
    assert torch.equal(got["alignments"], want["alignments"])
    for k in ("durations_log", "y_mean", "y_log_scale", "total_durations_log"):
        if float(want[k].abs().max()) == 0.0:
            assert torch.equal(got[k], want[k]), k
        else:
            assert rel_rms(got[k], want[k]) <= 1e-5, (k, rel_rms(got[k], want[k]))
    g, w = got["model_outputs"], want["model_outputs"]
    assert g.shape == w.shape
    assert rel_rms(g, w) <= 1e-4 and float((g - w).pow(2).mean().sqrt()) <= 1e-4, rel_rms(g, w)


@pytest.mark.parametrize("case", list(CASES))
def test_glow_tts_matches_oracle(case):
    cfg, sd, x, lens, extra, noise = run_case(case)
    want = GO.inference(sd, x, lens, cfg, noise=noise, **extra)
    got = gpu_inference(model_for(cfg, sd), x, lens, extra, noise)
    check_against_oracle(got, want)


def bench_batch(seed=0):
    """bench.py's batch shape: 32 utterances of up to 64 tokens; the duration predictor's output bias is log 6, so
    random-init durations are about 5 frames per token (LJSpeech-like)."""
    cfg = GlowTTSConfig(num_chars=100)
    sd = glow_state(cfg, 21, math.log(6.0))
    g = torch.Generator().manual_seed(seed)
    lens = torch.randint(40, 65, (32,), generator=g)
    lens[0] = 64
    x = torch.randint(0, 100, (32, 64), generator=g)
    return cfg, sd, x, lens


def test_glow_tts_bench_scale_matches_oracle_and_pins_dispatch():
    cfg, sd, x, lens = bench_batch()
    want = GO.inference(sd, x, lens, cfg)
    m = model_for(cfg, sd)
    with _lib.dispatch_log() as log:
        got = gpu_inference(m, x, lens, {}, None)
    check_against_oracle(got, want)
    assert got["model_outputs"].shape[1] >= 256          # long enough for the tensor-core convs (squeezed >= 128)
    p = cfg.encoder_params
    n_text = 4 * cfg.use_encoder_prenet + 4 * p["num_layers"] + 1 + 3   # prenet, transformer, proj, duration predictor
    per_block = 2 + 2 * cfg.num_block_layers
    assert len(log.names) == n_text + cfg.num_flow_blocks_dec * per_block, len(log.names)
    assert log.names[:n_text] == ["fma"] * n_text
    for n in range(cfg.num_flow_blocks_dec):
        blk = log.names[n_text + n * per_block: n_text + (n + 1) * per_block]
        assert blk[1:-1] == ["tc3"] * (2 * cfg.num_block_layers), blk


def test_glow_tts_repeat_and_poisoned_workspace_bit_identical():
    cfg, sd, x, lens = bench_batch(1)
    cfg.inference_noise_scale = 0.33
    m = model_for(cfg, sd)
    first = gpu_inference(m, x, lens, {}, None)
    noise = torch.randn(32, cfg.out_channels, first["y_mean"].shape[1], generator=torch.Generator().manual_seed(5))
    a = gpu_inference(m, x, lens, {}, noise)
    b = gpu_inference(m, x, lens, {}, noise)
    for buf in _lib._workspaces.values():
        buf.view(torch.float32)[: buf.numel() // 4].fill_(float("nan"))
    c = gpu_inference(m, x, lens, {}, noise)
    for k in ("model_outputs", "y_mean", "y_log_scale", "alignments", "durations_log", "total_durations_log"):
        assert torch.equal(a[k], b[k]) and torch.equal(a[k], c[k]), k
    assert not torch.equal(a["model_outputs"], first["model_outputs"])   # the noise is used


def test_glow_tts_to_hifigan_chain():
    """GlowTTS -> vocoder_input (replicate padding of HifiganGenerator.inference) -> HiFiGAN v1 (80 mel), against the
    oracle chain."""
    from tts_b200.vocoder import GAN, AudioNorm, HifiganConfig, vocoder_input
    cfg, sd, x, lens, extra, noise = run_case("default")
    want_mel = GO.inference(sd, x, lens, cfg)["model_outputs"]
    torch.manual_seed(3)
    gan = GAN(HifiganConfig()).eval()
    want = O.hifigan_inference(gan.model_g.state_dict(), want_mel.transpose(1, 2), 5)
    gan.to(DEV)
    mel = model_for(cfg, sd).inference(x.to(DEV), {"x_lengths": lens.to(DEV)})["model_outputs"]
    voc_in = vocoder_input(mel, AudioNorm.identity(), AudioNorm.identity(), padding=5, time_last=False, aligned=True)
    got = gan.model_g(voc_in).cpu()
    assert got.shape == want.shape
    rms = float((got - want).pow(2).mean().sqrt())
    assert rms <= 1e-4, rms
