"""Tacotron (1) on the GPU: decoder steps against float64 at B = 1, 8, 32 and 33 (both GRUCell instantiations, both
attention types, ragged rows with a one-token row), full inference against the CPU oracle (tests/tacotron_oracle.py)
for every case of the CPU suite, long ragged sequences through the persistent biGRU, a 32-row ragged batch against
single-row calls, repeatability over a NaN-poisoned workspace, the kernel of every launch, and Tacotron ->
vocoder_input -> a HiFiGAN v2-shaped generator."""
import pytest
import torch

import tacotron_oracle as TO
from ref_golden import layout, seeded_state_dict
from test_tacotron_oracle_cpu import CASES, build_case, case_r
from tts_b200 import _lib
from tts_b200 import tacotron as TC

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
NEVER = -30.0   # stopnet bias that leaves the stop to the attention test or max_decoder_steps


def rel_rms(got, want):
    got, want = got.double().cpu(), want.double().cpu()
    return float((got - want).pow(2).mean().sqrt() / want.pow(2).mean().sqrt().clamp_min(1e-30))


def make(seed=13, stop_bias=NEVER, stop_gain=40.0, **over):
    cfg = TC.TacotronConfig(num_chars=40, **over)
    model = TC.Tacotron(cfg)
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


def check(model, cfg, sd, text, lens, draws=None, margin_min=1e-4):
    got = model.inference(text.to(DEV), {"x_lengths": lens.to(DEV)},
                          draws=None if draws is None else {k: v.to(DEV) for k, v in draws.items()})
    r = model.decoder.r
    want = TO.inference(sd, text, lens, cfg, r=r, draws=draws)
    want64 = TO.inference(sd, text, lens, cfg, r=r, draws=draws, dtype=torch.float64)
    # every stop decision clears 0.6 by more than the FP32 error, in both tests
    assert min(min(m) for m in want["margins"]) > margin_min, want["margins"]
    assert want["steps"] == want64["steps"]
    assert got["model_outputs_len"].cpu().tolist() == want["model_outputs_len"].tolist()
    assert torch.equal(got["stop_tokens"].cpu() > 0.6, want["stop_tokens"] > 0.6)
    for k in ("model_outputs", "decoder_outputs", "alignments", "stop_tokens"):
        assert got[k].shape == want[k].shape, k
        own, err = rel_rms(want[k], want64[k]), rel_rms(got[k], want64[k])
        assert err <= 2 * own + 1e-6, (k, err, own)
    for b, n in enumerate(want["model_outputs_len"].tolist()):   # zero past each row
        assert float(got["model_outputs"][b, n:].abs().sum()) == 0.0
        assert float(got["decoder_outputs"][b, n:].abs().sum()) == 0.0
        assert float(got["alignments"][b, :, int(lens[b]):].abs().sum()) == 0.0
    return got, want


@pytest.mark.parametrize("attention", ["original", "dynamic_convolution"])
@pytest.mark.parametrize("B", [1, 8, 32, 33])
def test_decoder_steps_against_float64(B, attention):
    """Three decoder steps at B rows (max_decoder_steps 2): the GRUCells run 8 rows per weight read up to B = 8 and 32
    above; ragged rows include a one-token row (which stops after its first step).  Frames, alignments and stop values
    within 1e-5 relative RMS of float64 per row."""
    cfg, model, sd = make(max_decoder_steps=2, attention_type=attention)
    g = torch.Generator().manual_seed(B)
    lens = [1] + torch.randint(2, 30, (B - 1,), generator=g).tolist()
    text, lt = tokens(lens, seed=B)
    with _lib.dispatch_log() as log:
        got = model.inference(text.to(DEV), {"x_lengths": lt.to(DEV)})
    assert ("gru_cell32" if B > 8 else "gru_cell") in log.names
    want = TO.inference(sd, text, lt, cfg, dtype=torch.float64)
    assert got["model_outputs_len"].cpu().tolist() == want["model_outputs_len"].tolist()
    for b in range(B):
        for k in ("decoder_outputs", "alignments", "stop_tokens"):
            assert rel_rms(got[k][b], want[k][b]) <= 1e-5, (b, k, rel_rms(got[k][b], want[k][b]))


@pytest.mark.parametrize("case", list(CASES))
def test_inference_matches_oracle(case):
    """The CPU suite's cases (the oracle there is torch.equal to the reference) against the oracle in float32 and
    float64: equal frame counts and stop decisions, errors within twice the oracle's own FP32 error."""
    cfg, sd, text, lens = build_case(case)
    model = TC.Tacotron(cfg)
    model.load_state_dict(sd)
    model.eval().to(DEV)
    model.decoder.set_r(case_r(case, cfg))
    draws = None
    if case == "dropout_at_inference":
        g = torch.Generator().manual_seed(21)
        draws = {"dropout": torch.rand(len(lens), cfg.max_decoder_steps + 1, 2, 256, generator=g) < 0.5}
    check(model, cfg, sd, text, lens, draws=draws)


def test_long_ragged_sequences_through_the_bigru():
    """Rows of 1 to 1000 tokens: the encoder biGRU runs up to 1000 steps per direction and the postnet biGRU over every
    frame; the whole call matches the float64 oracle as above."""
    cfg, model, sd = make(max_decoder_steps=3)
    text, lens = tokens([1000, 1, 333, 17])
    check(model, cfg, sd, text, lens)


def test_ragged_batch_of_32_matches_single_rows():
    """32 rows of 40-64 tokens (the GRUCells at 32 rows per weight read) whose stop values clear 0.6 by more than 0.2
    once the len / 4 gate opens, so rows of different lengths stop at different steps: the step counts equal the
    oracle's and differ between rows, and every row matches its own B = 1 call: the same frame count and stop
    decisions, and values within 1e-5 relative RMS."""
    cfg, model, sd = make(max_decoder_steps=48, double_decoder_consistency=True, stop_bias=-2.0, stop_gain=120.0)
    g = torch.Generator().manual_seed(8)
    lens = torch.randint(40, 65, (32,), generator=g).tolist()
    text, lt = tokens(lens, seed=9)
    want = TO.inference(sd, text, lt, cfg)
    assert len(set(want["steps"])) > 1 and min(m[0] for m in want["margins"]) > 0.2, want["steps"]
    with _lib.dispatch_log() as log:
        full = model.inference(text.to(DEV), {"x_lengths": lt.to(DEV)})
    assert "gru_cell32" in log.names
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
        assert torch.equal(full["stop_tokens"][b, :s] > 0.6, one["stop_tokens"][0] > 0.6), b


def test_repeatable_over_poisoned_workspace_and_dispatch():
    cfg, model, sd = make(max_decoder_steps=34, out_channels=80)
    text, lens = tokens([9, 4])
    aux = {"x_lengths": lens.to(DEV)}
    first = model.inference(text.to(DEV), aux)
    ws = _lib.workspace(DEV, 1, "tacotron")
    ws.fill_(255)   # NaN-poisoned workspace
    with _lib.dispatch_log() as log:
        again = model.inference(text.to(DEV), aux)
    for k in ("model_outputs", "decoder_outputs", "alignments", "stop_tokens", "model_outputs_len"):
        assert torch.equal(again[k], first[k]), k
    names = log.names
    # encoder: two prenet layers, bank, two projections (fma), highways, the GRU input projection, the biGRU,
    # inputs_layer; one decoder step; postnet: bank, projections, highways, GRU input projection, biGRU, last_linear
    cbhg = ["fma"] * 3 + ["highway", "fma", "bigru"]
    enc = ["fma"] * 2 + cbhg + ["fma"]
    step = ["hmm_linear"] * 2 + ["gru_cell", "taco_attn", "hmm_linear", "gru_cell", "gru_cell"] + \
        ["hmm_linear"] * 2 + ["taco1_step"]
    assert names == enc + step + cbhg + ["fma"], names


def test_tacotron_to_hifigan_chain():
    from tts_b200.hifigan import HifiganGenerator
    from tts_b200.vocoder import AudioNorm, vocoder_input

    cfg, model, sd = make(max_decoder_steps=20, out_channels=80)
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
