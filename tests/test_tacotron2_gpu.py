"""Tacotron2 on the GPU: one decoder step against float64 at B = 1, 8, 32 and 33 (both LSTM instantiations, both
attention types, ragged rows with a one-token row), full inference against the CPU oracle (tests/tacotron2_oracle.py)
for every in-scope option, rows stopping at different steps, a 32-row ragged batch against single-row calls,
repeatability over a NaN-poisoned workspace, the kernel of every launch, and Tacotron2 -> vocoder_input -> a HiFiGAN
v2-shaped generator."""
import pytest
import torch

import tacotron2_oracle as TO
from ref_golden import layout, seeded_state_dict
from tts_b200 import _lib
from tts_b200 import tacotron2 as TC

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
NEVER = -30.0   # stopnet bias that keeps every row running to max_decoder_steps


def rel_rms(got, want):
    got, want = got.double().cpu(), want.double().cpu()
    return float((got - want).pow(2).mean().sqrt() / want.pow(2).mean().sqrt().clamp_min(1e-30))


def make(seed=13, stop_bias=NEVER, stop_gain=40.0, **over):
    cfg = TC.Tacotron2Config(num_chars=40, **over)
    model = TC.Tacotron2(cfg)
    sd = TO.seeded_weights(seeded_state_dict(layout(model.state_dict()), seed), seed + 4, stop_bias=stop_bias,
                           stop_gain=stop_gain)
    model.load_state_dict(sd)
    model.eval()
    return cfg, model.to(DEV), sd


def tokens(lens, seed=3):
    g = torch.Generator().manual_seed(seed)
    text = torch.zeros(len(lens), max(lens), dtype=torch.long)
    for b, n in enumerate(lens):
        text[b, :n] = torch.randint(1, 40, (n,), generator=g)
    return text, torch.tensor(lens)


def check(model, cfg, sd, text, lens, draws=None, margin_min=None):
    got = model.inference(text.to(DEV), {"x_lengths": lens.to(DEV)},
                          draws=None if draws is None else {k: v.to(DEV) for k, v in draws.items()})
    r = model.decoder.r
    want = TO.inference(sd, text, lens, cfg, r=r, draws=draws)
    want64 = TO.inference(sd, text, lens, cfg, r=r, draws=draws, dtype=torch.float64)
    if margin_min is not None:   # every stop decision clears 0 by more than the FP32 error of the logit
        assert min(want["margins"]) > margin_min, want["margins"]
    assert want["steps"] == want64["steps"]
    assert got["model_outputs_len"].cpu().tolist() == want["model_outputs_len"].tolist()
    assert torch.equal(got["stop_tokens"].cpu() > 0.5, want["stop_tokens"] > 0.5)
    for k in ("model_outputs", "decoder_outputs", "alignments", "stop_tokens"):
        assert got[k].shape == want[k].shape, k
        own, err = rel_rms(want[k], want64[k]), rel_rms(got[k], want64[k])
        assert err <= 2 * own + 1e-6, (k, err, own)
    for b, n in enumerate(want["model_outputs_len"].tolist()):   # zero past each row
        assert float(got["model_outputs"][b, n:].abs().sum()) == 0.0
        assert float(got["alignments"][b, :, int(lens[b]):].abs().sum()) == 0.0
    return got, want


@pytest.mark.parametrize("attention", ["original", "dynamic_convolution"])
@pytest.mark.parametrize("B", [1, 8, 32, 33])
def test_decoder_steps_against_float64(B, attention):
    """Three decoder steps (prenet, attention LSTMCell, attention, decoder LSTMCell, projection, stopnet) at B rows: the
    LSTMCell runs 8 rows per weight read up to B = 8 and 32 above; ragged rows include a one-token row.  Frames,
    alignments and stop values within 1e-5 relative RMS of float64 per row."""
    cfg, model, sd = make(max_decoder_steps=3, attention_type=attention)
    g = torch.Generator().manual_seed(B)
    lens = [1] + torch.randint(2, 30, (B - 1,), generator=g).tolist()
    text, lt = tokens(lens, seed=B)
    with _lib.dispatch_log() as log:
        got = model.inference(text.to(DEV), {"x_lengths": lt.to(DEV)})
    assert ("lstm_cell32" if B > 8 else "lstm_cell") in log.names
    want = TO.inference(sd, text, lt, cfg, dtype=torch.float64)
    for b in range(B):
        for k in ("decoder_outputs", "alignments", "stop_tokens"):
            assert rel_rms(got[k][b], want[k][b]) <= 1e-5, (b, k, rel_rms(got[k][b], want[k][b]))


CASES = {
    "ddc_default": dict(double_decoder_consistency=True),
    "softmax": dict(attention_norm="softmax"),
    "no_location": dict(location_attn=False),
    "dca": dict(attention_type="dynamic_convolution"),
    "prenet_bn": dict(prenet_type="bn"),
    "dropout_at_inference": dict(prenet_dropout_at_inference=True),
    "r_below_r_init": dict(r=3),
}


@pytest.mark.parametrize("case", list(CASES))
def test_inference_matches_oracle(case):
    """max_decoder_steps 40 (a cut 8 steps into the second chunk of 32) on ragged rows with a one-token row."""
    cfg, model, sd = make(max_decoder_steps=40, **CASES[case])
    if case == "r_below_r_init":
        model.decoder.set_r(2)
    text, lens = tokens([13, 1, 7])
    draws = None
    if case == "dropout_at_inference":
        g = torch.Generator().manual_seed(21)
        draws = {"dropout": torch.rand(3, 40, 2, 256, generator=g) < 0.5}
    got, want = check(model, cfg, sd, text, lens, draws=draws)
    assert want["steps"] == [40, 40, 40]


def test_rows_stop_at_different_steps():
    """Negative stopnet weights and a bias of -0.3: the rows' stop logits rise towards different limits, so rows 0 and 3
    stop at different steps and rows 1 and 2 (one token) run into the 45-step cap, 13 steps into the second chunk.
    Every stop decision clears 0 by more than 1e-4."""
    cfg, model, sd = make(max_decoder_steps=45, stop_bias=-0.30, stop_gain=-40.0)
    text, lens = tokens([12, 7, 1, 10])
    got, want = check(model, cfg, sd, text, lens, margin_min=1e-4)
    assert want["steps"][1] == want["steps"][2] == 45 and want["steps"][0] != want["steps"][3], want["steps"]
    assert max(want["steps"][0], want["steps"][3]) < 45


def test_no_stop_at_step_zero():
    """A stop logit above 0 from the first step on: every row stops after step 1, not step 0 (the t > 0 rule)."""
    cfg, model, sd = make(max_decoder_steps=45, stop_bias=2.0)
    text, lens = tokens([12, 7, 1, 10])
    got, want = check(model, cfg, sd, text, lens, margin_min=1e-2)
    assert all(lg[0] > 0 for lg in want["logits"]) and want["steps"] == [2, 2, 2, 2]


def test_ragged_batch_of_32_matches_single_rows():
    """32 rows of 40-64 tokens (the LSTMCells at 32 rows per weight read) whose stop logits cross 0 at different steps
    (stopnet weights scaled by -120, bias -0.96; every stop decision clears 0 by more than 1e-4 in the oracle): the step
    counts equal the oracle's and differ between rows, and every row matches its own B = 1 call (8 rows per weight read):
    the same frame count and stop decisions, and values within 1e-5 relative RMS (the encoder and postnet convs pick
    their tiles by sequence length, so a padded row and its own call may differ in the last bits)."""
    cfg, model, sd = make(max_decoder_steps=48, double_decoder_consistency=True, stop_bias=-0.96, stop_gain=-120.0)
    g = torch.Generator().manual_seed(8)
    lens = torch.randint(40, 65, (32,), generator=g).tolist()
    text, lt = tokens(lens, seed=9)
    want = TO.inference(sd, text, lt, cfg)
    assert min(want["margins"]) > 1e-4, want["margins"]
    assert len(set(want["steps"])) > 1 and max(want["steps"]) < 48, want["steps"]
    with _lib.dispatch_log() as log:
        full = model.inference(text.to(DEV), {"x_lengths": lt.to(DEV)})
    assert "lstm_cell32" in log.names
    assert (full["model_outputs_len"].cpu() // 2).tolist() == want["steps"]
    for b in range(32):
        one = model.inference(text[b:b + 1, :lens[b]].to(DEV))
        n, s = int(one["model_outputs_len"][0]), int(one["model_outputs_len"][0]) // 2
        assert int(full["model_outputs_len"][b]) == n, b
        for k, x, y in (("model_outputs", full["model_outputs"][b, :n], one["model_outputs"][0]),
                        ("decoder_outputs", full["decoder_outputs"][b, :n], one["decoder_outputs"][0]),
                        ("alignments", full["alignments"][b, :s, :lens[b]], one["alignments"][0]),
                        ("stop_tokens", full["stop_tokens"][b, :s], one["stop_tokens"][0])):
            assert x.shape == y.shape and rel_rms(x, y) <= 1e-5, (b, k, rel_rms(x, y))
        assert torch.equal(full["stop_tokens"][b, :s] > 0.5, one["stop_tokens"][0] > 0.5), b


def test_dropout_follows_train_and_eval():
    """Whether the prenet dropout runs is decided per call (train mode, or prenet_dropout_at_inference), not when the
    handle is built: a handle first used in train mode runs without dropout after eval(), and the reverse."""
    cfg, model, sd = make(max_decoder_steps=12)
    text, lens = tokens([9, 4])
    aux = {"x_lengths": lens.to(DEV)}
    keep = {"dropout": torch.ones(2, 12, 2, 256, dtype=torch.bool, device=DEV)}
    model.train()
    dropped = model.inference(text.to(DEV), aux, draws=keep)
    model.eval()
    plain = model.inference(text.to(DEV), aux, draws=keep)
    want = TO.inference(sd, text, lens, cfg)
    assert rel_rms(plain["decoder_outputs"], want["decoder_outputs"]) <= 1e-5
    assert not torch.allclose(dropped["decoder_outputs"], plain["decoder_outputs"])
    model.train()
    again = model.inference(text.to(DEV), aux, draws=keep)
    assert torch.equal(again["decoder_outputs"], dropped["decoder_outputs"])


def test_repeatable_over_poisoned_workspace_and_dispatch():
    cfg, model, sd = make(max_decoder_steps=34)
    text, lens = tokens([9, 4])
    aux = {"x_lengths": lens.to(DEV)}
    first = model.inference(text.to(DEV), aux)
    ws = _lib.workspace(DEV, 1, "tacotron2")
    ws.fill_(255)   # NaN-poisoned workspace
    with _lib.dispatch_log() as log:
        again = model.inference(text.to(DEV), aux)
    for k in ("model_outputs", "decoder_outputs", "alignments", "stop_tokens", "model_outputs_len"):
        assert torch.equal(again[k], first[k]), k
    names = log.names
    # encoder: 3 convs + the input projection (fma), 9 BiLSTM steps, inputs_layer (fma); one decoder step; postnet
    assert names[:4] == ["fma"] * 4 and names[4:13] == ["lstm_bi"] * 9 and names[13] == "fma"
    step = ["hmm_linear"] * 2 + ["lstm_cell", "taco_attn", "lstm_cell"] + ["hmm_linear"] * 2 + ["taco_step"]
    assert names[14:14 + len(step)] == step
    assert names[14 + len(step):] == ["fma"] * 5


def test_tacotron2_to_hifigan_chain():
    from tts_b200.hifigan import HifiganGenerator
    from tts_b200.vocoder import AudioNorm, vocoder_input

    cfg, model, sd = make(max_decoder_steps=20, double_decoder_consistency=True)
    text, lens = tokens([10, 6])
    mel = model.inference(text.to(DEV), {"x_lengths": lens.to(DEV)})["model_outputs"]
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
