"""Overflow / Neural-HMM on the GPU: the BiLSTM and frame kernels against float64, full inference against the CPU oracle
(tests/overflow_oracle.py) at temperature 0 and with supplied draws, a ragged batch of 32 rows, a max_sampling_time cut
inside a chunk, repeatability over a NaN-poisoned workspace, the kernel of every launch, and Overflow -> vocoder_input
-> a HiFiGAN v2-shaped generator."""
import pytest
import torch

import overflow_oracle as OO
from ref_golden import layout, seeded_state_dict
from tts_b200 import _lib
from tts_b200 import overflow as OV

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
SMALL = dict(encoder_in_out_features=64, prenet_dim=32, memory_rnn_dim=64, outputnet_size=[64])
# one decoder block at hidden 150 (start 1x1, four WaveNet in_layers (k5, gated), four res_skip 1x1, end 1x1): below
# 128 squeezed frames the tensor-core kernels are not taken and every conv runs on the FP32 FMA tile kernel
DECODER_BLOCK_SHORT = ["fma"] * 10
DECODER_BLOCK_LONG = ["tc3"] * 10


def rel_rms(got, want):
    got, want = got.double().cpu(), want.double().cpu()
    return float((got - want).pow(2).mean().sqrt() / want.pow(2).mean().sqrt().clamp_min(1e-30))


def make(kind, seed=13, **over):
    cls, cfg_cls = (OV.Overflow, OV.OverflowConfig) if kind == "overflow" else (OV.NeuralhmmTTS, OV.NeuralhmmTTSConfig)
    cfg = cfg_cls(num_chars=40, **over)
    model = cls(cfg)
    sd = OO.seeded_weights(seeded_state_dict(layout(model.state_dict()), seed), seed + 4)
    model.load_state_dict(sd)
    model.eval()
    return cfg, model.to(DEV), sd


def tokens(lens, seed=3):
    g = torch.Generator().manual_seed(seed)
    text = torch.zeros(len(lens), max(lens), dtype=torch.long)
    for b, n in enumerate(lens):
        text[b, :n] = torch.randint(1, 40, (n,), generator=g)
    return text, torch.tensor(lens)


def check_against_oracle(model, cfg, sd, text, lens, kind, temp=0.0, draws=None, max_t=None, margin_min=5e-5,
                         mel_tol=None):
    aux = {"x_lengths": lens.to(DEV), "sampling_temp": temp}
    if max_t is not None:
        aux["max_sampling_time"] = max_t
    got = model.inference(text.to(DEV), aux, draws=None if draws is None else {k: v.to(DEV) for k, v in draws.items()})
    want = OO.inference(sd, text, lens, cfg, has_decoder=kind == "overflow", temp=temp, max_t=max_t, draws=draws)
    want64 = OO.inference(sd, text, lens, cfg, has_decoder=kind == "overflow", temp=temp, max_t=max_t, draws=draws,
                          dtype=torch.float64)
    # the trajectory must stay clear of threshold ties, or a rounding difference could flip a duration: the quantiles of
    # the GPU and the fp32 oracle differ by ~1e-6, the smallest margin of these seeds is >= 5e-5
    assert min(want["margins"]) > margin_min, want["margins"]
    # and every row has states of different lengths, so the per-row duration path is exercised
    for b in range(len(lens)):
        assert len(set(OO.state_durations(want["alignments"][b], int(want["hmm_outputs_len"][b])))) > 1, b
    assert torch.equal(want["hmm_outputs_len"], want64["hmm_outputs_len"])
    assert torch.equal(got["hmm_outputs_len"].cpu(), want["hmm_outputs_len"])
    assert torch.equal(got["alignments"].cpu(), want["alignments"])
    assert torch.equal(got["model_outputs_len"].cpu(), want["model_outputs_len"])
    assert got["model_outputs"].shape == want["model_outputs"].shape
    own = rel_rms(want["model_outputs"], want64["model_outputs"])
    err = rel_rms(got["model_outputs"], want64["model_outputs"])
    assert err <= (2 * own + 1e-6 if mel_tol is None else mel_tol), (err, own)
    assert rel_rms(got["hmm_outputs"], want64["hmm_outputs"]) <= 2 * rel_rms(want["hmm_outputs"], want64["hmm_outputs"]) + 1e-6
    return got, want


def test_bilstm_against_float64_ragged():
    """The encoder (embedding, convs, BiLSTM) on ragged rows up to T = 200 with one row of length 1, on a NaN-filled
    workspace: within 1e-5 of float64 per row and zero past every row."""
    cfg, model, sd = make("neuralhmm", prenet_dropout_at_inference=False)
    lens = [200, 1, 57, 131]
    text, lt = tokens(lens)
    states = torch.empty(len(lens), 200 * 2, 512, device=DEV)
    h = model.handle(DEV)
    L = _lib.lib()
    ws = torch.full((L.b200tts_overflow_workspace_bytes(h, len(lens), 200, 1) // 4,), float("nan"), device=DEV)
    tok, ln = text.to(DEV), lt.to(DEV)   # held: the call is asynchronous
    with _lib.dispatch_log() as log:
        _lib.check(L.b200tts_overflow_encode(h, _lib.ptr(tok), _lib.ptr(ln), len(lens), 200,
                                             _lib.ptr(states), _lib.ptr(ws), ws.numel() * 4, _lib.stream_ptr(DEV)),
                   "encode")
    torch.cuda.synchronize()
    assert log.names.count("lstm_bi") == 200 and set(log.names) <= {"fma", "lstm_bi"}
    # float64 reference of the same encoder per row
    for b, n in enumerate(lens):
        ref = OO.encoder(sd, text[b:b + 1, :n], cfg, torch.float64)[0]
        got = states[b, :n * 2].cpu()
        assert rel_rms(got, ref) <= 1e-5, (b, rel_rms(got, ref))
        assert torch.isfinite(got).all() and float(states[b, n * 2:].abs().sum()) == 0.0


@pytest.mark.parametrize("frames", [1, 8])
def test_frame_step_against_float64(frames):
    """The frame kernels on their own, at the default Neural-HMM sizes (prenet 2 x 256 with dropout at inference,
    LSTMCell 1024, output net 1024, 161 outputs): ``max_sampling_time`` = 1 runs exactly one frame (prenet with the
    supplied dropout masks, lstm_cell, hmm_linear with the gathered hoisted state column, the last layer, hmm_step's
    sample and transition); with 8 frames and a duration threshold of 0.999 the state advances on every frame, so the
    gather reads a different state column each frame.  Frame outputs within 1e-5 relative RMS of float64 and the states
    travelled equal."""
    cfg, model, sd = make("neuralhmm")
    text, lens = tokens([9, 6])
    g = torch.Generator().manual_seed(5)
    draws = {"noise": torch.randn(2, frames, 80, generator=g),
             "dropout": torch.rand(2, frames, cfg.prenet_n_layers, cfg.prenet_dim, generator=g) < 0.5}
    aux = {"x_lengths": lens.to(DEV), "sampling_temp": 0.4, "max_sampling_time": frames, "duration_threshold": 0.999}
    got = model.inference(text.to(DEV), aux, draws={k: v.to(DEV) for k, v in draws.items()})
    want = OO.inference(sd, text, lens, cfg, has_decoder=False, temp=0.4, max_t=frames, thr=0.999, draws=draws,
                        dtype=torch.float64)
    assert got["hmm_outputs"].shape == (2, frames, 80)
    assert torch.equal(got["alignments"].cpu(), want["alignments"])
    if frames > 1:
        assert want["alignments"][0].argmax(-1).tolist() == list(range(frames + 1))
    assert rel_rms(got["hmm_outputs"], want["hmm_outputs"]) <= 1e-5, rel_rms(got["hmm_outputs"], want["hmm_outputs"])


@pytest.mark.parametrize("kind", ["overflow", "neuralhmm"])
def test_inference_matches_oracle_temp0(kind):
    over = dict(sampling_temp=0.0) if kind == "overflow" else dict(prenet_dropout_at_inference=False)
    cfg, model, sd = make(kind, **over)
    text, lens = tokens([17, 9, 13])
    check_against_oracle(model, cfg, sd, text, lens, kind)


def test_ragged_batch_of_32_matches_single_rows():
    cfg, model, sd = make("overflow", **SMALL, hidden_channels_dec=48, num_flow_blocks_dec=4)
    g = torch.Generator().manual_seed(8)
    lens = torch.randint(40, 65, (32,), generator=g).tolist()
    text, lt = tokens(lens, seed=9)
    # durations, alignments and lengths are equal; the decoder's convs (3xTF32 from 128 squeezed frames on) sum in
    # another order than the CPU oracle's
    check_against_oracle(model, cfg, sd, text, lt, "overflow", mel_tol=1e-5)


@pytest.mark.parametrize("kind", ["overflow", "neuralhmm"])
def test_sampled_with_supplied_draws(kind):
    over = dict(SMALL, hidden_channels_dec=24, num_flow_blocks_dec=3) if kind == "overflow" else dict(SMALL)
    cfg, model, sd = make(kind, **over)   # Neural-HMM: prenet dropout at inference (its default) on
    text, lens = tokens([11, 7])
    g = torch.Generator().manual_seed(21)
    draws = {"noise": torch.randn(2, cfg.max_sampling_time, 80, generator=g),
             "dropout": torch.rand(2, cfg.max_sampling_time, cfg.prenet_n_layers, cfg.prenet_dim, generator=g) < 0.5}
    check_against_oracle(model, cfg, sd, text, lens, kind, temp=0.3, draws=draws)


def test_max_sampling_time_cut_mid_chunk_and_repeatable():
    cfg, model, sd = make("overflow", **SMALL, hidden_channels_dec=24, num_flow_blocks_dec=3, sampling_temp=0.0)
    text, lens = tokens([30, 4])
    got, want = check_against_oracle(model, cfg, sd, text, lens, "overflow", max_t=45)   # 45 = 32 + 13
    assert int(got["hmm_outputs_len"][0]) == 45
    ws = _lib.workspace(DEV, 1, "overflow")
    ws.fill_(255)   # NaN-poisoned workspace
    again = model.inference(text.to(DEV), {"x_lengths": lens.to(DEV), "sampling_temp": 0.0, "max_sampling_time": 45})
    for k in ("model_outputs", "hmm_outputs", "alignments", "hmm_outputs_len"):
        assert torch.equal(again[k], got[k]), k


def test_dispatch_and_launches_per_frame():
    cfg, model, sd = make("overflow", **dict(SMALL, outputnet_size=[64, 48]), hidden_channels_dec=24,
                          num_flow_blocks_dec=3, sampling_temp=0.0)
    text, lens = tokens([6, 5])
    model.inference(text.to(DEV), {"x_lengths": lens.to(DEV)})
    with _lib.dispatch_log() as log:
        model.inference(text.to(DEV), {"x_lengths": lens.to(DEV)})
    names = log.names
    # encoder: 3 convs + the input projection (fma), 6 BiLSTM steps, the hoisted conv (fma); one frame of the loop
    assert names[:4] == ["fma"] * 4 and names[4:10] == ["lstm_bi"] * 6 and names[10] == "fma"
    frame = ["hmm_linear"] * 2 + ["lstm_cell"] + ["hmm_linear"] * 3 + ["hmm_step"]
    assert names[11:11 + len(frame)] == frame
    assert all(n not in ("lstm_bi", "lstm_cell", "hmm_linear", "hmm_step") for n in names[11 + len(frame):])


def test_overflow_to_hifigan_chain():
    from tts_b200.hifigan import HifiganGenerator
    from tts_b200.vocoder import AudioNorm, vocoder_input

    cfg, model, sd = make("overflow", **SMALL, hidden_channels_dec=24, num_flow_blocks_dec=3, sampling_temp=0.0)
    text, lens = tokens([10, 6])
    out = model.inference(text.to(DEV), {"x_lengths": lens.to(DEV)})
    mel = out["model_outputs"]
    norm = AudioNorm(signal_norm=True, symmetric_norm=True, max_norm=4.0, clip_norm=True, min_level_db=-100.0,
                     ref_level_db=20.0)
    x = vocoder_input(mel, norm, norm, padding=0, time_last=False)
    gen = HifiganGenerator(in_channels=80, out_channels=1, resblock_type="1", resblock_dilation_sizes=[[1, 3, 5]] * 3,
                           resblock_kernel_sizes=[3, 7, 11], upsample_kernel_sizes=[16, 16, 4, 4],
                           upsample_initial_channel=128, upsample_factors=[8, 8, 2, 2], inference_padding=0,
                           cond_channels=0, conv_pre_weight_norm=False, conv_post_weight_norm=False,
                           conv_post_bias=False).eval().to(DEV)
    wav = gen(x)
    assert wav.shape == (2, 1, mel.shape[1] * 256) and torch.isfinite(wav).all()


@pytest.mark.parametrize("n_tokens", [6, 60])
def test_decoder_dispatch_at_default_config(n_tokens):
    """Overflow's Glow decoder at its default sizes (hidden 150, 12 blocks of 4 WaveNet layers): the kernel family of
    every decoder conv, in launch order (start, 4 x in_layer, 4 x res_skip, end per block), for a short utterance
    (fewer than 128 squeezed frames: the FMA tile kernel) and a long one."""
    cfg, model, sd = make("overflow", sampling_temp=0.0)
    text, lens = tokens([n_tokens])
    out = model.inference(text.to(DEV), {"x_lengths": lens.to(DEV)})
    with _lib.dispatch_log() as log:
        model.inference(text.to(DEV), {"x_lengths": lens.to(DEV)})
    names = log.names
    last = max(i for i, n in enumerate(names) if n == "hmm_step")
    dec = names[last + 1:]
    tq = int(out["model_outputs_len"][0]) // 2
    print("decoder dispatch:", n_tokens, tq, dec[:10])
    assert len(dec) == 12 * 10 and dec == dec[:10] * 12, dec
    assert dec[:10] == (DECODER_BLOCK_SHORT if tq < 128 else DECODER_BLOCK_LONG)
    assert (tq < 128) == (n_tokens == 6)
